// tests/bc7_ranking/collectives.cu — TEST INFRASTRUCTURE, never shipped (tests/test_cpu_bc7_collectives.py and
// tests/test_gpu_bc7_collectives.py build it).
//
// Checks of the primitives the pruned BC7 shape ranking added, each against an independent exact reference written here:
//   arg 0  dxb_half_ballot4_u64   four predicates per lane to one 64-bit mask per half-warp
//   arg 1  dxb_nth_set_bit_u64    position of the n-th set bit (lane-private; 64 when there is none)
//   arg 2  dxb_warp_max_u32       warp-wide maximum
//   arg 3  dxb_dp4a_s8s8          s8 x s8 dot product with a 32-bit accumulator (random words with extreme bytes)
// The same source is built by nvcc for sm_90a with the library's flags (the device branches) and by g++ with the emulator's flags
// (the host branches, DXB_NL = 32 emulated lanes).  Index i = 32 c + lane: on the device the 32 indices of case c are the 32 lanes
// of one warp (count is a multiple of 32, so every warp holds one case with all lanes converged); lane values are a function of
// (c, lane), so the reference recomputes every lane's value.  One case in four draws values from 0..3 (ties, sparse masks), one in
// four keeps only the low byte and the high word.  coll_run(arg, count, out) writes out[0] = the mismatch count and
// out[1..3] = (input, got, want) of one mismatch.
#include <stdint.h>
#include <string.h>
#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_pixel.cuh"
#include "dxb_bc7.cuh"

#if DXB_ON_DEVICE
  #define COLL_API extern "C" __attribute__((visibility("default")))
#else
  #define COLL_API extern "C"
#endif

DXB_DEV uint64_t coll_mix(uint64_t x)                                  // splitmix64 finaliser
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
DXB_DEV uint64_t coll_lane_val(uint64_t c, uint32_t arg, int l)
{
    const uint64_t r = coll_mix((c << 8) ^ ((uint64_t)arg << 40) ^ (uint64_t)l);
    return (c & 3u) == 0u ? (r & 3u) : (c & 3u) == 1u ? (r & 0xFFFFFFFF000000FFull) : r;
}
DXB_DEV uint32_t coll_bytes(uint64_t r)                                // random bytes, a third of them 0, 1, 127, 128, 254, 255, 0x80, 0x7F
{
    const uint8_t ext[8] = { 0, 1, 127, 128, 255, 254, 0x80, 0x7F };
    uint32_t v = 0;
    for (int n = 0; n < 4; ++n)
    {
        const uint32_t s = (uint32_t)(r >> (8 * n + 32)) & 0xFFu;
        v |= (s < 96u ? ext[s & 7u] : (uint32_t)(r >> (8 * n)) & 0xFFu) << (8 * n);
    }
    return v;
}

struct coll_out { unsigned long long n, in, got, want; };

DXB_DEV void coll_check(uint64_t i, uint32_t arg, coll_out* o)
{
    const uint64_t c = i >> 5;
    const int lane = (int)(i & 31u);
#if DXB_ON_DEVICE
    const int L = 0;
#else
    const int L = lane;
#endif
    uint32_t u[DXB_NL];
    uint64_t ow[DXB_NL];
    for (int l = 0; l < DXB_NL; ++l) u[l] = (uint32_t)coll_lane_val(c, arg, DXB_ON_DEVICE ? lane : l);
    const int h0 = lane & 16;
    uint64_t got = 0, want = 0;
    switch (arg)
    {
    case 0:
        dxb_half_ballot4_u64(u, ow); got = ow[L];
        for (int l = 0; l < 16; ++l)
            for (int j = 0; j < 4; ++j) want |= (uint64_t)((coll_lane_val(c, arg, h0 + l) >> j) & 1u) << (16 * j + l);
        break;
    case 1:
    {
        const uint64_t mv = coll_lane_val(c, arg, lane);
        const uint32_t n = (uint32_t)(coll_mix(i) % 67u);
        got = dxb_nth_set_bit_u64(mv, n);
        want = 64u;
        for (uint32_t b = 0, k = 0; b < 64; ++b)
            if ((mv >> b) & 1u) { if (k == n) { want = b; break; } ++k; }
        break;
    }
    case 2:
        got = dxb_warp_max_u32(u);
        for (int l = 0; l < 32; ++l) { const uint32_t v = (uint32_t)coll_lane_val(c, arg, l); want = v > want ? v : want; }
        break;
    case 3:
    {
        const uint64_t r0 = coll_mix(i ^ 0x5A5A000000000000ull), r1 = coll_mix(r0), r2 = coll_mix(r1);
        const uint32_t a = coll_bytes(r0), b = coll_bytes(r1);
        const uint32_t s = (uint32_t)(r2 >> 58);
        const int32_t acc = s == 0u ? (int32_t)0x80000000u : s == 1u ? 0x7FFFFFFF : s == 2u ? 0 : s == 3u ? -1 : (int32_t)(uint32_t)r2;
        int64_t x = acc;
        for (int n = 0; n < 4; ++n) x += (int64_t)(int8_t)((a >> (8 * n)) & 0xFFu) * (int64_t)(int8_t)((b >> (8 * n)) & 0xFFu);
        got = (uint32_t)dxb_dp4a_s8s8(a, b, acc);
        want = (uint32_t)(uint64_t)x;
        break;
    }
    default: break;
    }
    if (got != want)
    {
#if DXB_ON_DEVICE
        if (atomicAdd(&o->n, 1ull) == 0ull) { o->in = i; o->got = got; o->want = want; }
#else
        #pragma omp critical
        { if (o->n++ == 0ull) { o->in = i; o->got = got; o->want = want; } }
#endif
    }
}

COLL_API int coll_on_device() { return DXB_ON_DEVICE; }

#if DXB_ON_DEVICE
__global__ void __launch_bounds__(256) k_coll(uint32_t arg, uint64_t count, coll_out* o)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < count; j += stride) coll_check(j, arg, o);
}
// 0 = ran, else the CUDA error code; count must be a multiple of 32
COLL_API int coll_run(uint32_t arg, uint64_t count, unsigned long long* out)
{
    coll_out* d = nullptr;
    cudaError_t e = cudaMalloc((void**)&d, sizeof(coll_out));
    if (e != cudaSuccess) return (int)e;
    e = cudaMemset(d, 0, sizeof(coll_out));
    if (e == cudaSuccess)
    {
        const uint64_t want = (count + 255u) / 256u;
        k_coll<<<(unsigned)(want < 2048u ? want : 2048u), 256>>>(arg, count, d);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, d, sizeof(coll_out), cudaMemcpyDeviceToHost);
    cudaFree(d);
    return (int)e;
}
#else
COLL_API int coll_run(uint32_t arg, uint64_t count, unsigned long long* out)
{
    coll_out o;
    memset(&o, 0, sizeof(o));
    #pragma omp parallel for schedule(static, 4096)
    for (long long j = 0; j < (long long)count; ++j) coll_check((uint64_t)j, arg, &o);
    memcpy(out, &o, sizeof(o));
    return 0;
}
#endif
