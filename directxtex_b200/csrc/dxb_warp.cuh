// dxb_warp.cuh — single-source SPMD helpers: the same block-encoder source runs
//   * on sm_90a by one warp for TWO 4x4 blocks, one per 16-lane half (lane-private scalars, __shfl_sync exchanges), and
//   * in tests/emul as a loop over 32 emulated lanes (lane-private values are arrays of 32).
// Per-lane variables are declared `T v[DXB_NL]` and accessed as `v[L]`; DXB_NL is 1 on the device.
#pragma once
#include "dxb_portable.h"

#if DXB_ON_DEVICE
  #define DXB_NL 1
  #define DXB_LANES_BEGIN { const int lane = (int)(threadIdx.x & 31u); const int L = 0; (void)L; (void)lane;
  #define DXB_LANES_END }
  #define DXB_FULLMASK 0xffffffffu
#else
  #define DXB_NL 32
  #define DXB_LANES_BEGIN for (int lane = 0; lane < 32; ++lane) { const int L = lane;
  #define DXB_LANES_END }
#endif

// out[lane] = in[lane ^ m]
DXB_DEV void dxb_xchg_xor_f32(const float* in, float* out, int m)
{
#if DXB_ON_DEVICE
    out[0] = __shfl_xor_sync(DXB_FULLMASK, in[0], m);
#else
    float tmp[32];
    for (int l = 0; l < 32; ++l) tmp[l] = in[l ^ m];
    for (int l = 0; l < 32; ++l) out[l] = tmp[l];
#endif
}
DXB_DEV void dxb_xchg_xor_u32(const uint32_t* in, uint32_t* out, int m)
{
#if DXB_ON_DEVICE
    out[0] = __shfl_xor_sync(DXB_FULLMASK, in[0], m);
#else
    uint32_t tmp[32];
    for (int l = 0; l < 32; ++l) tmp[l] = in[l ^ m];
    for (int l = 0; l < 32; ++l) out[l] = tmp[l];
#endif
}
// value held by lane `src` (src uniform across the warp)
DXB_DEV uint32_t dxb_bcast_u32(const uint32_t* v, int src)
{
#if DXB_ON_DEVICE
    return __shfl_sync(DXB_FULLMASK, v[0], src);
#else
    return v[src];
#endif
}
DXB_DEV float dxb_bcast_f32(const float* v, int src)
{
#if DXB_ON_DEVICE
    return __shfl_sync(DXB_FULLMASK, v[0], src);
#else
    return v[src];
#endif
}
// warp-wide minimum / OR of unsigned keys (integer => order independent => deterministic)
DXB_DEV uint32_t dxb_warp_min_u32(const uint32_t* v)
{
#if DXB_ON_DEVICE
    return __reduce_min_sync(DXB_FULLMASK, v[0]);
#else
    uint32_t m = v[0];
    for (int l = 1; l < 32; ++l) m = (v[l] < m) ? v[l] : m;
    return m;
#endif
}
DXB_DEV uint32_t dxb_warp_or_u32(const uint32_t* v)
{
#if DXB_ON_DEVICE
    return __reduce_or_sync(DXB_FULLMASK, v[0]);
#else
    uint32_t m = 0;
    for (int l = 0; l < 32; ++l) m |= v[l];
    return m;
#endif
}
DXB_DEV uint32_t dxb_warp_max_u32(const uint32_t* v)
{
#if DXB_ON_DEVICE
    return __reduce_max_sync(DXB_FULLMASK, v[0]);
#else
    uint32_t m = v[0];
    for (int l = 1; l < 32; ++l) m = (v[l] > m) ? v[l] : m;
    return m;
#endif
}
DXB_DEV uint64_t dxb_warp_min_u64(const uint64_t* v)
{
#if DXB_ON_DEVICE
    uint64_t x = v[0];
    #pragma unroll
    for (int m = 16; m >= 1; m >>= 1)
    {
        const uint64_t y = __shfl_xor_sync(DXB_FULLMASK, x, m);
        x = (y < x) ? y : x;
    }
    return x;
#else
    uint64_t m = v[0];
    for (int l = 1; l < 32; ++l) m = (v[l] < m) ? v[l] : m;
    return m;
#endif
}
// CTA-wide phase alignment: keeps the warps of a CTA in the same code region so that they share instruction-cache
// lines (the BC7 encoder is ~75 KB of straight-line code; measured 4.0 -> 3.8 ms).  -DDXB_BC7_NO_CTA_SYNC disables it.
DXB_DEV void dxb_phase_sync()
{
#if DXB_ON_DEVICE && !defined(DXB_BC7_NO_CTA_SYNC)
    __syncthreads();
#endif
}
DXB_DEV void dxb_warp_sync()
{
#if DXB_ON_DEVICE
    __syncwarp();
#endif
}

// ---------------------------------------------------------------------------------------------------
// Half-warp (16-lane group) collectives: the BC7 encoder runs TWO blocks per warp, one per half.
// Results are lane-private (uniform inside a half, different between halves).

// out[lane] = min / OR over the 16-lane half that contains `lane`
DXB_DEV void dxb_half_min_u32(const uint32_t* v, uint32_t* out)
{
#if DXB_ON_DEVICE
    const uint32_t hm = 0xFFFFu << (threadIdx.x & 16u);
    out[0] = __reduce_min_sync(hm, v[0]);
#else
    for (int h = 0; h < 32; h += 16)
    {
        uint32_t m = v[h];
        for (int l = 1; l < 16; ++l) m = (v[h + l] < m) ? v[h + l] : m;
        for (int l = 0; l < 16; ++l) out[h + l] = m;
    }
#endif
}
DXB_DEV void dxb_half_or_u32(const uint32_t* v, uint32_t* out)
{
#if DXB_ON_DEVICE
    const uint32_t hm = 0xFFFFu << (threadIdx.x & 16u);
    out[0] = __reduce_or_sync(hm, v[0]);
#else
    for (int h = 0; h < 32; h += 16)
    {
        uint32_t m = 0;
        for (int l = 0; l < 16; ++l) m |= v[h + l];
        for (int l = 0; l < 16; ++l) out[h + l] = m;
    }
#endif
}
// out[lane] = v[lane of the same half whose index inside the half is src[lane] & 15]
DXB_DEV void dxb_half_gather_u32(const uint32_t* v, const uint32_t* src, uint32_t* out)
{
#if DXB_ON_DEVICE
    out[0] = __shfl_sync(DXB_FULLMASK, v[0], (int)(src[0] & 15u), 16);
#else
    uint32_t tmp[32];
    for (int l = 0; l < 32; ++l) tmp[l] = v[(l & 16) | (int)(src[l] & 15u)];
    for (int l = 0; l < 32; ++l) out[l] = tmp[l];
#endif
}
// four predicates per lane (bit j of flags[lane], j < 4) to one 64-bit mask per half: bit 16 j + h of out[lane] = predicate j of the
// lane whose index inside the half of `lane` is h
DXB_DEV void dxb_half_ballot4_u64(const uint32_t* flags, uint64_t* out)
{
#if DXB_ON_DEVICE
    const uint32_t sh = threadIdx.x & 16u;
    uint64_t m = 0;
    #pragma unroll
    for (int j = 0; j < 4; ++j) m |= (uint64_t)((__ballot_sync(DXB_FULLMASK, (flags[0] >> j) & 1u) >> sh) & 0xFFFFu) << (16 * j);
    out[0] = m;
#else
    for (int h = 0; h < 32; h += 16)
    {
        uint64_t m = 0;
        for (int l = 0; l < 16; ++l)
            for (int j = 0; j < 4; ++j) m |= (uint64_t)((flags[h + l] >> j) & 1u) << (16 * j + l);
        for (int l = 0; l < 16; ++l) out[h + l] = m;
    }
#endif
}

// lane-private bit arithmetic: position of the n-th (from 0) set bit of m, 64 when m has n or fewer set bits
DXB_DEV uint32_t dxb_nth_set_bit_u64(uint64_t m, uint32_t n)
{
#if DXB_ON_DEVICE
    const uint32_t clo = (uint32_t)__popc((uint32_t)m);
    const bool hi = (n >= clo);
    uint32_t w = hi ? (uint32_t)(m >> 32) : (uint32_t)m, pos = hi ? 32u : 0u;
    n = hi ? n - clo : n;
    if (n >= (uint32_t)__popc(w)) return 64u;
    // binary search: the wanted bit lies in w above `pos`, with n set bits of w below it
    #pragma unroll
    for (uint32_t s = 16; s >= 1; s >>= 1)
    {
        const uint32_t c = (uint32_t)__popc(w & ((1u << s) - 1u));
        const bool up = (n >= c);
        n = up ? n - c : n; w = up ? w >> s : w; pos = up ? pos + s : pos;
    }
    return pos;
#else
    for (uint32_t b = 0; b < 64; ++b)
        if ((m >> b) & 1u) { if (n == 0u) return b; --n; }
    return 64u;
#endif
}
