// tests/probe/probe.cu — TEST INFRASTRUCTURE, never shipped.
//
// Exhaustive / dense checks of the arithmetic shortcuts the kernels take on the device.  Many primitives of the shared headers have an
// `#if DXB_ON_DEVICE` branch: on sm_90a a bit trick valid on a stated domain, in the host emulator a plain cast or loop.  The host
// emulator stands in for the GPU in every quality measurement only if both branches give the same value, so every check below compares
// one primitive, evaluated exactly as the headers define it, with an independent exact reference written here (integer arithmetic and
// IEEE-exact operations only; a reference never calls the primitive it checks).
//
// The same source is built twice: by nvcc for sm_90a with the library's flags (libdxb_probe.so, the device branches) and by g++ with
// the emulator's flags (libdxb_probe_host.so, the host branches).  Device == reference and host == reference on one domain give
// device == emulator there.
//
// A check maps a 64-bit index to one input, so no input crosses PCIe.  probe_run(id, arg, begin, count, step, out) evaluates the
// indices begin + j * step for j < count and writes out[0] = the mismatch count and out[1 + 3 r .. 3 + 3 r] = (input, got, want) of
// up to 16 mismatches (the first 16 found; on the device not necessarily the 16 lowest indices).  Mismatches are data: no check
// asserts or traps.
#include <stdint.h>
#include <string.h>
#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_pixel.cuh"
#include "dxb_bc7.cuh"
#include "dxb_udiv.h"

#if DXB_ON_DEVICE
  #define PROBE_API extern "C" __attribute__((visibility("default")))
#else
  #define PROBE_API extern "C"
#endif

struct probe_out { unsigned long long n; unsigned long long rec[16][3]; };

DXB_DEV void probe_bad(probe_out* o, uint64_t in, uint64_t got, uint64_t want)
{
    unsigned long long s;
#if DXB_ON_DEVICE
    s = atomicAdd(&o->n, 1ull);
#else
    #pragma omp atomic capture
    s = o->n++;
#endif
    if (s < 16) { o->rec[s][0] = in; o->rec[s][1] = got; o->rec[s][2] = want; }
}
#define PROBE_EXPECT(in, got, want) do { const uint64_t g_ = (uint64_t)(got), w_ = (uint64_t)(want); if (g_ != w_) probe_bad(o, (in), g_, w_); } while (0)

// ---- reference helpers: integers and bit patterns only ------------------------------------------------------------------------
DXB_DEV uint64_t rmix(uint64_t x)                                      // splitmix64 finaliser: the random inputs
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
DXB_DEV uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
DXB_DEV float bitsf(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

// binary32 bits of the integer m * 2^e2 rounded to nearest even (m < 2^63); sign separately
DXB_DEV uint32_t ref_u64_to_f32(uint64_t m)
{
    if (m == 0) return 0;
    int top = 63; while (!((m >> top) & 1u)) --top;
    if (top <= 23) return ((uint32_t)(127 + top) << 23) | (uint32_t)((m << (23 - top)) & 0x7FFFFFu);
    const int sh = top - 23;
    uint64_t q = m >> sh; const uint64_t rem = m & ((1ull << sh) - 1ull), half = 1ull << (sh - 1);
    if (rem > half || (rem == half && (q & 1u))) ++q;
    int e = top; if (q >> 24) { q >>= 1; ++e; }
    return ((uint32_t)(127 + e) << 23) | (uint32_t)(q & 0x7FFFFFu);
}
DXB_DEV uint32_t ref_i32_to_f32(int32_t n) { return n < 0 ? 0x80000000u | ref_u64_to_f32((uint64_t)(-(int64_t)n)) : ref_u64_to_f32((uint64_t)n); }

// |f| split: the integer part and whether the fraction is 0, below, at or above 1/2 (finite f with |f| < 2^63)
struct ref_parts { uint64_t ip; int frac; bool neg; };                 // frac: 0 none, 1 < 1/2, 2 == 1/2, 3 > 1/2
DXB_DEV ref_parts ref_split(uint32_t b)
{
    ref_parts r; r.neg = (b >> 31) != 0u;
    const int e = (int)((b >> 23) & 0xFFu);
    const uint64_t m = (e ? 0x800000u : 0u) | (b & 0x7FFFFFu);
    const int sh = 150 - (e ? e : 1);                                  // value = m * 2^-sh
    if (sh <= 0) { r.ip = m << (-sh); r.frac = 0; return r; }
    if (sh >= 64) { r.ip = 0; r.frac = m ? 1 : 0; return r; }
    r.ip = m >> sh;
    const uint64_t rem = m & ((1ull << sh) - 1ull), half = 1ull << (sh - 1);
    r.frac = rem == 0 ? 0 : rem < half ? 1 : rem == half ? 2 : 3;
    return r;
}
DXB_DEV uint64_t ref_rne_mag(ref_parts p) { return p.ip + ((p.frac == 3 || (p.frac == 2 && (p.ip & 1u))) ? 1u : 0u); }

// BC7 interpolation weights (BC7 format specification)
DXB_CONST uint8_t ref_w2[4] = { 0, 21, 43, 64 };
DXB_CONST uint8_t ref_w3[8] = { 0, 9, 18, 27, 37, 46, 55, 64 };
DXB_CONST uint8_t ref_w4[16] = { 0, 4, 9, 13, 17, 21, 26, 30, 34, 38, 43, 47, 51, 55, 60, 64 };
DXB_DEV uint32_t ref_weight(uint32_t ib, uint32_t k) { return ib == 2u ? ref_w2[k] : ib == 3u ? ref_w3[k] : ref_w4[k]; }
DXB_DEV uint32_t ref_interp(uint32_t a, uint32_t b, uint32_t w) { return (a * (64u - w) + b * w + 32u) >> 6; }
DXB_DEV uint32_t ref_unq(uint32_t f, uint32_t B)                       // BC7 unquantise: replicate the field's high bits
{
    uint32_t v = f << (8u - B);
    return v | (v >> B);
}
DXB_DEV uint32_t ref_byte(uint32_t w, int c) { return (w >> (8 * c)) & 0xFFu; }
// the eight (bits, p-bit) endpoint field layouts of the BC7 modes: (4,1) 0, (6,1) 1, (5,0) 2/4, (7,1) 3/6, (6,0) 4a, (7,0) 5, (8,0) 5a, (5,1) 7
DXB_CONST uint8_t ref_layout_bits[8] = { 4, 6, 5, 7, 6, 7, 8, 5 };
DXB_CONST uint8_t ref_layout_p[8] = { 1, 1, 0, 1, 0, 0, 0, 1 };
// per mode: colour bits, alpha bits (0 = no alpha field), p-bits present
DXB_CONST uint8_t ref_mode_cb[8] = { 4, 6, 5, 7, 5, 7, 7, 5 };
DXB_CONST uint8_t ref_mode_ab[8] = { 0, 0, 0, 0, 6, 8, 7, 5 };
DXB_CONST uint8_t ref_mode_p[8] = { 1, 1, 0, 1, 0, 0, 1, 1 };

// ---- checks ---------------------------------------------------------------------------------------------------------------------
// dxb_i2f_small: index = n + 2^22 - 1 for every |n| < 2^22
DXB_DEV void chk_i2f_small(uint64_t i, uint32_t, probe_out* o)
{
    const int32_t n = (int32_t)i - 0x3FFFFF;
    PROBE_EXPECT(i, fbits(dxb_i2f_small(n)), ref_i32_to_f32(n));
}
// dxb_byte_to_float: byte position k = i & 3, byte value (i >> 2) & 255, the other bytes 0x00 (i >> 10 == 0), 0xFF (== 1) or random
DXB_DEV void chk_byte_to_float(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t k = (uint32_t)i & 3u, b = (uint32_t)(i >> 2) & 0xFFu, sel = (uint32_t)(i >> 10);
    const uint32_t rest = sel == 0u ? 0u : sel == 1u ? 0xFFFFFFFFu : (uint32_t)rmix(i);
    const uint32_t v = (rest & ~(0xFFu << (8u * k))) | (b << (8u * k));
    PROBE_EXPECT(((uint64_t)v << 2) | k, fbits(dxb_byte_to_float(v, k)), ref_u64_to_f32(b));
}
// dxb_f2u_trunc_small on [-0, 2^23): index = the bit pattern for [+0, 2^23), index 0x4B000000 = -0
DXB_DEV void chk_f2u_trunc_small(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = i == 0x4B000000u ? 0x80000000u : (uint32_t)i;
    PROBE_EXPECT(b, dxb_f2u_trunc_small(bitsf(b)), ref_split(b).ip);
}
// dxb_f2u_trunc_small on (-1, 0), outside its precondition: the C cast gives 0 (recorded, not required)
DXB_DEV void chk_f2u_trunc_small_neg(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = 0x80000001u + (uint32_t)i;                       // i < 0x3F7FFFFF
    PROBE_EXPECT(b, dxb_f2u_trunc_small(bitsf(b)), 0u);
}
// signed bit pattern of index i over [0, 2 * npos): i < npos -> +i, else -(i - npos)
DXB_DEV uint32_t probe_signed_bits(uint64_t i, uint32_t npos) { return i < npos ? (uint32_t)i : 0x80000000u | (uint32_t)(i - npos); }
// dxb_f2i_rn_small on (-2^22, 2^22) (0x4A800000 = 2^22)
DXB_DEV void chk_f2i_rn_small(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = probe_signed_bits(i, 0x4A800000u);
    const ref_parts p = ref_split(b); const int64_t m = (int64_t)ref_rne_mag(p);
    PROBE_EXPECT(b, (uint32_t)dxb_f2i_rn_small(bitsf(b)), (uint32_t)(p.neg ? -m : m));
}
// dxb_f2i (truncation) on every float whose truncation fits int32: |f| < 2^31 and -2^31 (0x4F000000 = 2^31)
DXB_DEV void chk_f2i(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = probe_signed_bits(i, 0x4F000000u);
    const ref_parts p = ref_split(b);
    PROBE_EXPECT(b, (uint32_t)dxb_f2i(bitsf(b)), (uint32_t)(p.neg ? -(int64_t)p.ip : (int64_t)p.ip));
}
// dxb_f2u on every float whose truncation fits uint32: [+0, 2^32) and (-1, -0] (0x4F800000 = 2^32, 0x3F800000 = 1)
DXB_DEV void chk_f2u(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = i < 0x4F800000u ? (uint32_t)i : 0x80000000u | (uint32_t)(i - 0x4F800000u);
    PROBE_EXPECT(b, dxb_f2u(bitsf(b)), ref_split(b).ip);
}
// dxb_f2i_rn on every float whose RNE fits int32: [-2^31, 2^31)
DXB_DEV void chk_f2i_rn(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = probe_signed_bits(i, 0x4F000000u);
    const ref_parts p = ref_split(b); const int64_t m = (int64_t)ref_rne_mag(p);
    PROBE_EXPECT(b, (uint32_t)dxb_f2i_rn(bitsf(b)), (uint32_t)(p.neg ? -m : m));
}
// dxb_f2i outside int32 (|f| >= 2^31 except -2^31, infinities, NaN): the device saturates (NaN -> 0), the x86 host returns
// 0x80000000.  The reference here is the saturating conversion; mismatches are recorded, not required to be zero.
DXB_DEV void chk_f2i_out_of_range(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t npos = 0x80000000u - 0x4F000000u;                   // [2^31, NaN) positive patterns
    const uint32_t b = i < npos ? 0x4F000000u + (uint32_t)i : 0xCF000001u + (uint32_t)(i - npos);
    const bool nan = (b & 0x7FFFFFFFu) > 0x7F800000u;
    PROBE_EXPECT(b, (uint32_t)dxb_f2i(bitsf(b)), nan ? 0u : (b >> 31) ? 0x80000000u : 0x7FFFFFFFu);
}
// dxb_round_even on every float (NaN: any NaN)
DXB_DEV void chk_round_even(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = (uint32_t)i, a = b & 0x7FFFFFFFu;
    const uint32_t got = fbits(dxb_round_even(bitsf(b)));
    if (a > 0x7F800000u) { if ((got & 0x7FFFFFFFu) <= 0x7F800000u) probe_bad(o, b, got, 0x7FC00000u); return; }
    const uint32_t want = a >= 0x4B000000u ? b : (b & 0x80000000u) | ref_u64_to_f32(ref_rne_mag(ref_split(b)));
    PROBE_EXPECT(b, got, want);
}
// IEEE binary16 -> binary32, all 65 536 halves (a NaN must stay a NaN; its payload is not compared)
DXB_DEV uint32_t ref_half_to_float(uint32_t h)
{
    const uint32_t s = (h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    if (e == 0x1Fu) return s | 0x7F800000u | (m << 13);
    if (e == 0u) { const uint32_t mag = ref_u64_to_f32(m); return s | (m ? mag - (24u << 23) : 0u); }    // m * 2^-24
    return s | ((e + 112u) << 23) | (m << 13);
}
DXB_DEV void chk_half_to_float(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t h = (uint32_t)i, want = ref_half_to_float(h), got = fbits(dxb_half_to_float((uint16_t)h));
    if ((want & 0x7FFFFFFFu) > 0x7F800000u) { if ((got & 0x7FFFFFFFu) <= 0x7F800000u) probe_bad(o, h, got, want); return; }
    PROBE_EXPECT(h, got, want);
}
// binary32 -> binary16 round to nearest even, every non-NaN float: the value as an integer multiple of 2^-149, rounded to the
// binary16 grid (2^-24 below 2^-14, else 2^(e - 10)), overflow to infinity
DXB_DEV uint32_t ref_float_to_half(uint32_t b)
{
    const uint32_t s = (b >> 16) & 0x8000u, a = b & 0x7FFFFFFFu;
    if (a >= 0x7F800000u) return s | 0x7C00u;                             // infinity (NaN excluded by the caller)
    const int e = (int)(a >> 23);
    const uint64_t m = (e ? 0x800000u : 0u) | (a & 0x7FFFFFu);
    const int ue = e ? e - 127 : -126;                                    // value = m * 2^(ue - 23)
    if (ue >= 16) return s | 0x7C00u;
    const int he = ue < -14 ? -14 : ue;                                   // binary16 exponent of the target grid
    const int sh = (he - 10) - (ue - 23);                                 // value / 2^(he - 10) = m / 2^sh
    uint64_t q;
    if (sh <= 0) q = m << (-sh);
    else if (sh >= 40) q = 0;
    else
    {
        q = m >> sh;
        const uint64_t rem = m & ((1ull << sh) - 1ull), half = 1ull << (sh - 1);
        if (rem > half || (rem == half && (q & 1u))) ++q;
    }
    // q counts units of 2^(he - 10): below 2^-14 it is the subnormal field; otherwise 1024 + mantissa, with carries into the exponent
    if (he == -14) return s | (uint32_t)q;                                // q <= 1024: 1024 is the smallest normal, bits 0x0400
    const uint32_t bits = (uint32_t)(he + 15) * 1024u + (uint32_t)(q - 1024u);
    return s | (bits >= 0x7C00u ? 0x7C00u : bits);
}
DXB_DEV void chk_float_to_half(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = (uint32_t)i;
    if ((b & 0x7FFFFFFFu) > 0x7F800000u) return;                          // NaN: not part of the domain
    PROBE_EXPECT(b, dxb_float_to_half(bitsf(b)), ref_float_to_half(b));
}
// dxb_unorm8_trunc and dxb_pack_unorm8x4: every float v (i & 0xFFFFFFFF, NaN included) at channel position k = i >> 32 of four,
// the other channels random in [-0.25, 1.25).  Reference floor(clamp(v + 0.5/255, 0, 1) * 255) with the headers' clamp order (NaN -> 0: SSE min/max)
DXB_DEV uint32_t ref_unorm8(float v)
{
    float b = v + (0.5f / 255.0f);
    b = (b > 0.0f) ? b : 0.0f;                                            // max(b, 0), NaN -> 0
    b = (b < 1.0f) ? b : 1.0f;
    return (uint32_t)ref_split(fbits(b * 255.0f)).ip;
}
DXB_DEV void chk_unorm8(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t b = (uint32_t)i, k = (uint32_t)(i >> 32) & 3u;
    const uint64_t r = rmix(i);
    float c[4];
    for (int n = 0; n < 4; ++n) c[n] = (float)(uint32_t)((r >> (16 * n)) & 0xFFFFu) * (1.5f / 65536.0f) - 0.25f;   // [-0.25, 1.25)
    c[k] = bitsf(b);
    uint32_t want = 0;
    for (int n = 0; n < 4; ++n) want |= ref_unorm8(c[n]) << (8 * n);
    PROBE_EXPECT(i, dxb_pack_unorm8x4(c[0], c[1], c[2], c[3]), want);
    PROBE_EXPECT(i | (1ull << 40), dxb_unorm8_trunc(c[k]), ref_unorm8(c[k]));
}
// dxb_rcp_int: 1 / x for every integer x = 1 .. 2^24 - 1, against the correctly rounded quotient (double then float is correctly
// rounded: 53 >= 2 * 24 + 2)
DXB_DEV void chk_rcp_int(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t x = (uint32_t)i;
    const double q = 1.0 / (double)x;
    PROBE_EXPECT(x, fbits(dxb_rcp_int(bitsf(ref_u64_to_f32(x)))), fbits((float)q));
}
// dxb_bc7_quant2f (and dxb_floor_mul inside it): one (bits, p-bit) layout = arg & 7, p = arg >> 3, every float e in [+0, 255]
// (index = its bit pattern; index 0x437F0001 = -0) in both halves of the pair.  Requires q an integer in [+0, qmax] and deq the BC7
// decoder's unquantised value of the field (2 q + p with a p-bit, else q).
DXB_DEV void chk_quant2f(uint64_t i, uint32_t arg, probe_out* o)
{
    const uint32_t lay = arg & 7u, p = arg >> 3, bits = ref_layout_bits[lay], hasP = ref_layout_p[lay];
    const uint32_t eb = i == 0x437F0001u ? 0x80000000u : (uint32_t)i;
    const float e = bitsf(eb), e2 = bitsf(0x437F0000u - (uint32_t)(i % 0x437F0001u));   // other half: the mirrored pattern
    const dxb_bc7_qconst k = dxb_bc7_make_qconst(bits, hasP);
    dxb_f2 deq;
    const dxb_f2 q = dxb_bc7_quant2f(dxb_mk2(e, e2), k, (int)p, &deq);
    const float qs[2] = { q.x, q.y }, ds[2] = { deq.x, deq.y };
    for (int h = 0; h < 2; ++h)
    {
        const uint32_t qb = fbits(qs[h]);
        const ref_parts qp = ref_split(qb);
        const uint32_t qmax = (1u << bits) - 1u;
        const bool ok = !qp.neg && qp.frac == 0 && qp.ip <= qmax && (qb & 0x80000000u) == 0u;
        const uint64_t in = ((uint64_t)h << 32) | (h ? fbits(e2) : eb);
        if (!ok) { probe_bad(o, in, qb, 0xFFFFFFFFu); continue; }
        const uint32_t full = hasP ? 2u * (uint32_t)qp.ip + p : (uint32_t)qp.ip;
        PROBE_EXPECT(in | (1ull << 33), fbits(ds[h]), ref_u64_to_f32(ref_unq(full, bits + hasP)));
    }
}
// BC7 weights: dxb_bc7_weightf and dxb_bc7_weight for all 28 (ib, k).  The encoder's weight bits (dxb_bc7_eval: k c64 + MAGIC, one
// product and one add), the final search's FFMA weight bits and its index recovery (w (n - 1) + 32) >> 6 == k (dxb_bc7_nearest) are
// inline expressions there, so forms 1-3 restate them: a change of those constants is seen by the nearest1 / nearest4 sweeps, not
// here.  Bits 8+ of the reported input = which form failed.
DXB_DEV void chk_bc7_weights(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t ib = i < 4 ? 2u : i < 12 ? 3u : 4u, kk = (uint32_t)(i < 4 ? i : i < 12 ? i - 4 : i - 12), n = (1u << ib) - 1u;
    const uint32_t w = ref_weight(ib, kk);
    const float nmax = (float)n, c64r = 64.0f / nmax;                      // the encoder's run-time constant
    const float c64k = (ib == 2u) ? 64.0f / 3.0f : (ib == 3u) ? 64.0f / 7.0f : 64.0f / 15.0f;   // the final search's constant
    const float kf = bitsf(ref_u64_to_f32(kk));
    PROBE_EXPECT(i, fbits(dxb_bc7_weightf(kf, c64r)), ref_u64_to_f32(w) - (w ? (6u << 23) : 0u));   // w / 64
    PROBE_EXPECT(i | (1ull << 8), fbits(kf * c64r + DXB_MAGIC), 0x4B400000u + w);
    PROBE_EXPECT(i | (2ull << 8), fbits(dxb_fma(kf, c64k, DXB_MAGIC)), 0x4B400000u + w);
    PROBE_EXPECT(i | (3ull << 8), (w * n + 32u) >> 6, kk);
    PROBE_EXPECT(i | (4ull << 8), dxb_bc7_weight(ib, kk), w);
}
// dxb_bc7_make_pal4 + dxb_bc7_pal4_entry: endpoint bytes e0, e1 of channel c at every weight 0..64 (also the ones BC7 does not use),
// the other channels' bytes 0 / 255 / random, every byte mask of channels cm.  i = e0 | e1 << 8 | w << 16 (w < 65) | c << 23 |
// cm << 25 | others << 29.
DXB_DEV void chk_pal4(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t e0 = (uint32_t)i & 0xFFu, e1 = (uint32_t)(i >> 8) & 0xFFu, w = (uint32_t)(i >> 16) & 0x7Fu;
    const uint32_t c = (uint32_t)(i >> 23) & 3u, cmb = (uint32_t)(i >> 25) & 15u, oth = (uint32_t)(i >> 29);
    if (w > 64u) return;
    const uint64_t r = rmix(i);
    uint32_t d0 = oth == 0u ? 0u : oth == 1u ? 0xFFFFFFFFu : (uint32_t)r, d1 = oth == 0u ? 0xFFFFFFFFu : oth == 1u ? 0u : (uint32_t)(r >> 32);
    d0 = (d0 & ~(0xFFu << (8 * c))) | (e0 << (8 * c)); d1 = (d1 & ~(0xFFu << (8 * c))) | (e1 << (8 * c));
    uint32_t cm = 0, want = 0;
    for (int n = 0; n < 4; ++n) if ((cmb >> n) & 1u) { cm |= 0xFFu << (8 * n); want |= ref_interp(ref_byte(d0, n), ref_byte(d1, n), w) << (8 * n); }
    PROBE_EXPECT(i, dxb_bc7_pal4_entry(dxb_bc7_make_pal4(d0, d1, cm), 0x4B400000u + w), want);
}
// naive nearest palette index: ascending k, strict <, error = sum of squared byte differences over the channels of cm
DXB_DEV uint32_t ref_nearest(uint32_t pix, uint32_t d0, uint32_t d1, uint32_t cm, uint32_t ib)
{
    uint32_t best = 0, bestErr = 0xFFFFFFFFu;
    for (uint32_t k = 0; k < (1u << ib); ++k)
    {
        uint32_t err = 0;
        for (int n = 0; n < 4; ++n)
        {
            if (!ref_byte(cm, n)) continue;
            const int32_t d = (int32_t)ref_byte(pix, n) - (int32_t)ref_interp(ref_byte(d0, n), ref_byte(d1, n), ref_weight(ib, k));
            err += (uint32_t)(d * d);
        }
        if (err < bestErr) { bestErr = err; best = k; }
    }
    return best;
}
// MAXN = 16 with ib = 2, 3, 4 and MAXN = 8 with ib = 2, 3: variant v = arg (0..4)
DXB_DEV uint32_t probe_nearest(uint32_t v, uint32_t pix, const dxb_bc7_pal4& P)
{
    return v < 3u ? dxb_bc7_nearest<16>(pix, P, v + 2u) : dxb_bc7_nearest<8>(pix, P, v - 1u);
}
DXB_DEV uint32_t probe_nearest_ib(uint32_t v) { return v < 3u ? v + 2u : v - 1u; }
// one channel exhaustively: i = pixel | e0 << 8 | e1 << 16 | c << 24; the other channels random and masked out (as the caller masks)
DXB_DEV void chk_nearest1(uint64_t i, uint32_t v, probe_out* o)
{
    const uint32_t c = (uint32_t)(i >> 24) & 3u, cm = 0xFFu << (8 * c);
    const uint64_t r = rmix(i ^ ((uint64_t)v << 40));
    const uint32_t pix = ((uint32_t)r & ~cm) | (((uint32_t)i & 0xFFu) << (8 * c));
    const uint32_t d0 = ((uint32_t)(r >> 32) & ~cm) | ((((uint32_t)i >> 8) & 0xFFu) << (8 * c));
    const uint32_t d1 = ((uint32_t)(r >> 16) & ~cm) | ((((uint32_t)i >> 16) & 0xFFu) << (8 * c));
    const uint32_t ib = probe_nearest_ib(v);
    PROBE_EXPECT(i, probe_nearest(v, pix & cm, dxb_bc7_make_pal4(d0, d1, cm)), ref_nearest(pix & cm, d0, d1, cm, ib));
}
// random four-channel cases: channel masks of the encoder (RGBA, RGB, A) and random ones; equal endpoints, pixels on a palette entry
// or halfway between two (ties) in some of the cases
DXB_DEV void chk_nearest4(uint64_t i, uint32_t v, probe_out* o)
{
    const uint64_t r = rmix(i ^ ((uint64_t)v << 40)), r2 = rmix(r);
    const uint32_t ib = probe_nearest_ib(v), kind = (uint32_t)(r2 >> 60);
    const uint32_t cms[4] = { 0xFFFFFFFFu, 0x00FFFFFFu, 0xFF000000u, 0u };
    uint32_t cm = cms[(r2 >> 56) & 3u];
    if (cm == 0u) for (int n = 0; n < 4; ++n) cm |= ((r2 >> (50 + n)) & 1u) ? 0xFFu << (8 * n) : 0u;
    uint32_t d0 = (uint32_t)r, d1 = (uint32_t)(r >> 32), pix = (uint32_t)r2;
    if (kind == 0u) d1 = d0;                                                          // equal endpoints
    else if (kind == 1u || kind == 2u)
    {
        // pixel on entry k (kind 1) or per channel halfway between entries k and k + 1, rounded either way (kind 2)
        const uint32_t k = (uint32_t)(r2 >> 32) & ((1u << ib) - 2u);
        pix = 0;
        for (int n = 0; n < 4; ++n)
        {
            const uint32_t a = ref_interp(ref_byte(d0, n), ref_byte(d1, n), ref_weight(ib, k));
            const uint32_t b = ref_interp(ref_byte(d0, n), ref_byte(d1, n), ref_weight(ib, k + 1u));
            const uint32_t m = kind == 1u ? a : (a + b + ((r2 >> (40 + n)) & 1u)) >> 1;
            pix |= m << (8 * n);
        }
    }
    else if (kind == 3u) { d0 &= 0x03030303u; d1 = d0 + 0x01010101u; }                // adjacent endpoints: many equal entries
    PROBE_EXPECT(i, probe_nearest(v, pix & cm, dxb_bc7_make_pal4(d0, d1, cm)), ref_nearest(pix & cm, d0, d1, cm, ib));
}
// dxb_bc7_deq4 for mode m = arg & 7, p-bit p = arg >> 3: every combination of the four fields (mixed radix over the field widths,
// slot order: three colour fields then alpha, absent alpha = field 0)
DXB_DEV void chk_deq4(uint64_t i, uint32_t arg, probe_out* o)
{
    const uint32_t m = arg & 7u, p = arg >> 3, cb = ref_mode_cb[m], ab = ref_mode_ab[m], hasP = ref_mode_p[m];
    const uint32_t f0 = (uint32_t)i & ((1u << cb) - 1u), f1 = (uint32_t)(i >> cb) & ((1u << cb) - 1u), f2 = (uint32_t)(i >> (2 * cb)) & ((1u << cb) - 1u);
    const uint32_t f3 = ab ? (uint32_t)(i >> (3 * cb)) & ((1u << ab) - 1u) : 0u;
    const uint32_t q = f0 | (f1 << 8) | (f2 << 16) | (f3 << 24);
    dxb_bc7_modecfg cfg = dxb_bc7_cfg((int)m);
    const uint32_t pb = hasP ? p : 0u, full = hasP ? 1u : 0u;
    uint32_t want = 0;
    const uint32_t f[3] = { f0, f1, f2 };
    for (int n = 0; n < 3; ++n) want |= ref_unq(full ? 2u * f[n] + pb : f[n], cb + full) << (8 * n);
    want |= (ab ? ref_unq(full ? 2u * f3 + pb : f3, ab + full) : 255u) << 24;
    PROBE_EXPECT(((uint64_t)q << 1) | p, dxb_bc7_deq4(q, p, dxb_bc7_make_deqk(cfg)), want);
}
// dxb_put_bits4: i = pos | nbits << 7 | value << 11 | word seed << 19, skipping pos + nbits > 128; reference = a bit-by-bit OR
DXB_DEV void chk_put_bits4(uint64_t i, uint32_t, probe_out* o)
{
    const uint32_t pos = (uint32_t)i & 127u, nbits = (uint32_t)(i >> 7) & 15u, value = (uint32_t)(i >> 11) & 0xFFu;
    if (nbits > 8u || pos + nbits > 128u) return;
    const uint64_t r = rmix(i >> 19), r2 = rmix(r);
    uint32_t w[4] = { (uint32_t)r, (uint32_t)(r >> 32), (uint32_t)r2, (uint32_t)(r2 >> 32) };
    if ((i >> 19) == 0) w[0] = w[1] = w[2] = w[3] = 0u;
    uint32_t want[4] = { w[0], w[1], w[2], w[3] };
    for (uint32_t b = 0; b < nbits; ++b)
        if ((value >> b) & 1u) want[(pos + b) >> 5] |= 1u << ((pos + b) & 31u);
    dxb_put_bits4(w, pos, nbits, value);
    for (int n = 0; n < 4; ++n) PROBE_EXPECT(i | ((uint64_t)n << 60), w[n], want[n]);
}
// a random word whose bytes / halves are drawn from the extremes or at random
DXB_DEV uint32_t probe_bytes(uint64_t r)
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
DXB_DEV int32_t probe_acc(uint64_t r)
{
    const uint32_t s = (uint32_t)(r >> 58);
    return s == 0u ? (int32_t)0x80000000u : s == 1u ? 0x7FFFFFFF : s == 2u ? 0 : s == 3u ? -1 : (int32_t)(uint32_t)r;
}
DXB_DEV int32_t ref_wrap(int64_t v) { return (int32_t)(uint32_t)(uint64_t)v; }
// the byte / pair dot products, PRMT, VABSDIFF4, three-way min / max: variant = arg
DXB_DEV void chk_simd(uint64_t i, uint32_t arg, probe_out* o)
{
    const uint64_t r0 = rmix(i ^ ((uint64_t)arg << 48)), r1 = rmix(r0), r2 = rmix(r1), r3 = rmix(r2);
    const uint32_t a = probe_bytes(r0), b = probe_bytes(r1);
    const int32_t acc = probe_acc(r2);
    switch (arg)
    {
    case 0: { int64_t s = acc; for (int n = 0; n < 4; ++n) s += (int64_t)ref_byte(a, n) * (int8_t)ref_byte(b, n);
              PROBE_EXPECT(i, (uint32_t)dxb_dp4a_u8s8(a, b, acc), (uint32_t)ref_wrap(s)); break; }
    case 1: { int64_t s = acc; for (int n = 0; n < 4; ++n) s += (int64_t)ref_byte(a, n) * ref_byte(b, n);
              PROBE_EXPECT(i, (uint32_t)dxb_dp4a_u8u8(a, b, acc), (uint32_t)ref_wrap(s)); break; }
    case 2: case 3:
    {
        // s16 pairs: halves random or extreme (0x8000, 0x7FFF, 0xFFFF, 0)
        const uint16_t ext[4] = { 0x8000u, 0x7FFFu, 0xFFFFu, 0u };
        uint32_t pair = (uint32_t)r3;
        if ((r3 >> 32) & 1u) pair = (pair & 0xFFFF0000u) | ext[(r3 >> 33) & 3u];
        if ((r3 >> 35) & 1u) pair = (pair & 0x0000FFFFu) | ((uint32_t)ext[(r3 >> 36) & 3u] << 16);
        const int c0 = arg == 2u ? 0 : 2;
        const int64_t s = (int64_t)acc + (int64_t)(int16_t)(pair & 0xFFFFu) * ref_byte(b, c0) + (int64_t)(int16_t)(pair >> 16) * ref_byte(b, c0 + 1);
        const int32_t got = arg == 2u ? dxb_dp2a_lo_s16u8(pair, b, acc) : dxb_dp2a_hi_s16u8(pair, b, acc);
        PROBE_EXPECT(i, (uint32_t)got, (uint32_t)ref_wrap(s));
        break;
    }
    case 4:
    {
        // every selector without the sign-replicate bits: i & 4095 = the four 3-bit byte selectors
        const uint32_t sel = (uint32_t)(i & 7u) | ((uint32_t)(i >> 3) & 7u) << 4 | ((uint32_t)(i >> 6) & 7u) << 8 | ((uint32_t)(i >> 9) & 7u) << 12;
        uint32_t want = 0;
        for (int n = 0; n < 4; ++n) { const uint32_t s = (sel >> (4 * n)) & 7u; want |= (s < 4u ? ref_byte(a, (int)s) : ref_byte(b, (int)s - 4)) << (8 * n); }
        PROBE_EXPECT(i, dxb_prmt(a, b, sel), want);
        break;
    }
    case 5: { uint32_t want = 0; for (int n = 0; n < 4; ++n) { const int32_t d = (int32_t)ref_byte(a, n) - (int32_t)ref_byte(b, n); want |= (uint32_t)(d < 0 ? -d : d) << (8 * n); }
              PROBE_EXPECT(i, dxb_vabsdiff4(a, b), want); break; }
    case 6: case 7:
    {
        const int32_t x = probe_acc(r0), y = probe_acc(r1 ^ (r3 << 58)), z = probe_acc(r3);
        const int32_t lo = x < y ? (x < z ? x : z) : (y < z ? y : z), hi = x > y ? (x > z ? x : z) : (y > z ? y : z);
        PROBE_EXPECT(i, (uint32_t)(arg == 6u ? dxb_min3_s32(x, y, z) : dxb_max3_s32(x, y, z)), (uint32_t)(arg == 6u ? lo : hi));
        break;
    }
    default: break;
    }
}
// dxb_udiv_make / dxb_udiv_do.  arg 0: every d = 1 .. 2^16 - 1 (i >> 6) with 64 numerators n around multiples of d, at the ends of
// the 32-bit range and at random; arg 1: random d < 2^31 and random / edge n.
DXB_DEV void chk_udiv(uint64_t i, uint32_t arg, probe_out* o)
{
    const uint64_t r = rmix(i ^ ((uint64_t)arg << 50));
    const uint32_t d = arg == 0u ? (uint32_t)(i >> 6) + 1u : (uint32_t)(r >> 33) + 1u;
    const uint32_t j = (uint32_t)i & 63u, rn = (uint32_t)rmix(r);
    uint32_t n;
    if (j < 8u) { const uint32_t e[8] = { 0u, 1u, 0x7FFFFFFFu, 0x80000000u, 0xFFFFFFFFu, 0xFFFFFFFEu, d - 1u, d }; n = e[j]; }
    else if (j < 40u)
    {
        // k d - 1 .. k d + 2 for a random multiple k d <= 2^32 - 1, clamped to the 32-bit range
        const uint64_t m = (uint64_t)d * ((uint64_t)rn % (0xFFFFFFFFull / d + 1u)) + (j & 3u);
        n = m == 0u ? 0u : (m - 1u > 0xFFFFFFFFull) ? 0xFFFFFFFFu : (uint32_t)(m - 1u);
    }
    else n = rn;
    PROBE_EXPECT(((uint64_t)d << 32) | n, dxb_udiv_do(n, dxb_udiv_make(d)), n / d);
}

// dxb_warp.cuh collectives.  Index i = 32 c + lane: the 32 indices of case c are the 32 lanes of one warp on the device (probe_run
// starts at a multiple of 32 with step 1 and a count that is a multiple of 32, so every warp of the grid-stride loop holds one case
// with all lanes converged); the host build emulates the whole warp (DXB_NL = 32 lanes) and takes lane i & 31.  Lane values are a
// function of (c, lane), so the reference recomputes every lane's value instead of exchanging them.  Variant arg: 0 xchg_xor_u32,
// 1 xchg_xor_f32, 2 bcast_u32, 3 bcast_f32, 4 warp_min_u32, 5 warp_or_u32, 6 warp_min_u64, 7 half_min_u32, 8 half_or_u32,
// 9 half_gather_u32.  One case in four draws values from 0..3 (ties); the two halves differ.
DXB_DEV uint64_t probe_lane_val(uint64_t c, uint32_t arg, int l)
{
    const uint64_t r = rmix((c << 8) ^ ((uint64_t)arg << 40) ^ (uint64_t)l);
    return (c & 3u) == 0u ? (r & 3u) : (c & 3u) == 1u ? (r & 0xFFFFFFFF000000FFull) : r;
}
DXB_DEV void chk_warp(uint64_t i, uint32_t arg, probe_out* o)
{
    const uint64_t c = i >> 5;
    const int lane = (int)(i & 31u);
    const int m = (int)(c % 31u) + 1, src = (int)((c >> 5) & 31u);
#if DXB_ON_DEVICE
    const int L = 0;
#else
    const int L = lane;
#endif
    uint32_t u[DXB_NL], s[DXB_NL], ou[DXB_NL];
    float f[DXB_NL], of[DXB_NL];
    uint64_t w[DXB_NL];
    for (int l = 0; l < DXB_NL; ++l)
    {
        const int ln = DXB_ON_DEVICE ? lane : l;
        w[l] = probe_lane_val(c, arg, ln);
        u[l] = (uint32_t)w[l];
        f[l] = bitsf(u[l]);
        s[l] = (uint32_t)(w[l] >> 32);                                      // gather source: low 4 bits used, high bits garbage
    }
    uint64_t got = 0, want = 0;
    const int h0 = lane & 16;
    switch (arg)
    {
    case 0: dxb_xchg_xor_u32(u, ou, m); got = ou[L]; want = (uint32_t)probe_lane_val(c, arg, lane ^ m); break;
    case 1: dxb_xchg_xor_f32(f, of, m); got = fbits(of[L]); want = (uint32_t)probe_lane_val(c, arg, lane ^ m); break;
    case 2: got = dxb_bcast_u32(u, src); want = (uint32_t)probe_lane_val(c, arg, src); break;
    case 3: got = fbits(dxb_bcast_f32(f, src)); want = (uint32_t)probe_lane_val(c, arg, src); break;
    case 4: case 5: case 6:
    {
        got = arg == 4u ? dxb_warp_min_u32(u) : arg == 5u ? dxb_warp_or_u32(u) : dxb_warp_min_u64(w);
        want = arg == 5u ? 0u : ~0ull;
        for (int l = 0; l < 32; ++l)
        {
            const uint64_t v = probe_lane_val(c, arg, l), v32 = (uint32_t)v;
            if (arg == 4u) want = v32 < want ? v32 : want;
            else if (arg == 5u) want |= v32;
            else want = v < want ? v : want;
        }
        if (arg == 4u) want = (uint32_t)want;
        break;
    }
    case 7: case 8:
    {
        if (arg == 7u) dxb_half_min_u32(u, ou); else dxb_half_or_u32(u, ou);
        got = ou[L];
        want = arg == 8u ? 0u : 0xFFFFFFFFu;
        for (int l = h0; l < h0 + 16; ++l)
        {
            const uint32_t v = (uint32_t)probe_lane_val(c, arg, l);
            want = arg == 7u ? (v < want ? v : want) : (want | v);
        }
        break;
    }
    case 9:
        dxb_half_gather_u32(u, s, ou); got = ou[L];
        want = (uint32_t)probe_lane_val(c, arg, h0 | (int)((probe_lane_val(c, arg, lane) >> 32) & 15u));
        break;
    default: break;
    }
    PROBE_EXPECT(i | ((uint64_t)arg << 56), got, want);
}

// ---- the table of checks and the two drivers --------------------------------------------------------------------------------------
#define PROBE_CHECKS(X) \
    X(i2f_small) X(byte_to_float) X(f2u_trunc_small) X(f2u_trunc_small_neg) X(f2i_rn_small) X(f2i) X(f2u) X(f2i_rn) \
    X(f2i_out_of_range) X(round_even) X(half_to_float) X(float_to_half) X(unorm8) X(rcp_int) X(quant2f) X(bc7_weights) X(pal4) \
    X(nearest1) X(nearest4) X(deq4) X(put_bits4) X(simd) X(udiv) X(warp)

#define PROBE_NAME(f) #f,
static const char* const probe_names[] = { PROBE_CHECKS(PROBE_NAME) };
static const int probe_count = (int)(sizeof(probe_names) / sizeof(probe_names[0]));

PROBE_API const char* probe_name(int id) { return (id >= 0 && id < probe_count) ? probe_names[id] : nullptr; }
PROBE_API int probe_on_device() { return DXB_ON_DEVICE; }

typedef void (*probe_fn)(uint64_t, uint32_t, probe_out*);

#if DXB_ON_DEVICE
template <void (*F)(uint64_t, uint32_t, probe_out*)>
__global__ void __launch_bounds__(256) k_probe(uint32_t arg, uint64_t begin, uint64_t count, uint64_t step, probe_out* o)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < count; j += stride) F(begin + j * step, arg, o);
}
#define PROBE_KERNEL(f) k_probe<chk_##f>,
typedef void (*probe_kernel)(uint32_t, uint64_t, uint64_t, uint64_t, probe_out*);
static const probe_kernel probe_kernels[] = { PROBE_CHECKS(PROBE_KERNEL) };

// 0 = ran, -1 = unknown check, else the CUDA error code
PROBE_API int probe_run(int id, uint32_t arg, uint64_t begin, uint64_t count, uint64_t step, unsigned long long* out)
{
    if (id < 0 || id >= probe_count) return -1;
    probe_out* d = nullptr;
    cudaError_t e = cudaMalloc((void**)&d, sizeof(probe_out));
    if (e != cudaSuccess) return (int)e;
    e = cudaMemset(d, 0, sizeof(probe_out));
    if (e != cudaSuccess) { cudaFree(d); return (int)e; }
    int sms = 132;
    (void)cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const uint64_t want = (count + 255u) / 256u, cap = (uint64_t)sms * 16u;
    const unsigned grid = (unsigned)(want < 1u ? 1u : want < cap ? want : cap);
    probe_kernels[id]<<<grid, 256>>>(arg, begin, count, step, d);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpy(out, d, sizeof(probe_out), cudaMemcpyDeviceToHost);
    cudaFree(d);
    return (int)e;
}
#else
#define PROBE_FN(f) chk_##f,
static const probe_fn probe_fns[] = { PROBE_CHECKS(PROBE_FN) };

PROBE_API int probe_run(int id, uint32_t arg, uint64_t begin, uint64_t count, uint64_t step, unsigned long long* out)
{
    if (id < 0 || id >= probe_count) return -1;
    probe_out o;
    memset(&o, 0, sizeof(o));
    const probe_fn f = probe_fns[id];
    #pragma omp parallel for schedule(static, 4096)
    for (long long j = 0; j < (long long)count; ++j) f(begin + (uint64_t)j * step, arg, &o);
    memcpy(out, &o, sizeof(o));
    return 0;
}
#endif
