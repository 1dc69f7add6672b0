// dxb_portable.h — compile-time switch that lets the SAME arithmetic source be built
//   * by nvcc as __device__ code for sm_90a (the product), and
//   * by g++ as plain host code for tests/emul (a test-only lock-step emulator used to
//     debug parity on machines without a GPU; it is never linked into the product library).
// Under nvcc every DXB_DEV function is __device__-only, so the shipped .so contains no
// host copy of the arithmetic (no CPU fallback exists).
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
  #include <cuda_fp16.h>
  #include <cuda_runtime.h>
  #define DXB_DEV __device__ __forceinline__
  #define DXB_DEV_NOINLINE __device__ __noinline__
  #define DXB_CONST __device__ const
  #define DXB_ON_DEVICE 1
#else
  #include <math.h>
  #include <string.h>
  #define DXB_DEV static inline
  #define DXB_DEV_NOINLINE static
  #define DXB_CONST static const
  #define DXB_ON_DEVICE 0
#endif

// ---- float <-> int, truncation toward zero (C cast semantics of the reference) ----
DXB_DEV int32_t dxb_f2i(float f)
{
#if DXB_ON_DEVICE
    return __float2int_rz(f);
#else
    return (int32_t)f;
#endif
}
DXB_DEV uint32_t dxb_f2u(float f)
{
#if DXB_ON_DEVICE
    return __float2uint_rz(f);
#else
    return (uint32_t)f;
#endif
}
// round to nearest even (cvtps_epi32 / nearbyintf)
// Exact int <-> float conversions of SMALL values on the full-rate FP32/INT pipes instead of the quarter-rate
// conversion unit (I2F / F2I); the 8/10/16-bit pixel loads and stores of the HBM-bound row kernels were XU-bound.
//   dxb_i2f_small: |n| < 2^22      (1.5*2^23 + n is exact, so is the subtraction)
//   dxb_f2u_trunc_small: 0 <= f < 2^23, truncation: 2^23 + f rounded toward zero has floor(f) in its mantissa
//   dxb_f2i_rn_small: |f| < 2^22, round to nearest even (the magic-number add)
// The host build keeps the plain casts, which give the same values.
DXB_DEV float dxb_i2f_small(int32_t n)
{
#if DXB_ON_DEVICE
    return __int_as_float(0x4B400000 + n) - 12582912.0f;
#else
    return (float)n;
#endif
}
// byte k (0..3) of a 32-bit word as float: one PRMT drops the byte into the mantissa of 1.5*2^23
DXB_DEV float dxb_byte_to_float(uint32_t v, uint32_t k)
{
#if DXB_ON_DEVICE
    return __uint_as_float(__byte_perm(v, 0x4B400000u, 0x7650u + k)) - 12582912.0f;
#else
    return (float)((v >> (8u * k)) & 0xFFu);
#endif
}
DXB_DEV uint32_t dxb_f2u_trunc_small(float f)
{
#if DXB_ON_DEVICE
    return __float_as_uint(__fadd_rz(f, 8388608.0f)) & 0x7FFFFFu;
#else
    return (uint32_t)(int32_t)f;
#endif
}
DXB_DEV int32_t dxb_f2i_rn_small(float f)
{
#if DXB_ON_DEVICE
    return __float_as_int(f + 12582912.0f) - 0x4B400000;
#else
    return (int32_t)nearbyintf(f);
#endif
}
DXB_DEV int32_t dxb_f2i_rn(float f)
{
#if DXB_ON_DEVICE
    return __float2int_rn(f);
#else
    return (int32_t)nearbyintf(f);
#endif
}
// lroundf: round half away from zero
DXB_DEV int32_t dxb_lround(float f)
{
#if DXB_ON_DEVICE
    return (int32_t)lroundf(f);
#else
    return (int32_t)lroundf(f);
#endif
}
DXB_DEV float dxb_u2f(uint32_t u) { return (float)u; }
DXB_DEV float dxb_i2f(int32_t i) { return (float)i; }

DXB_DEV uint32_t dxb_float_as_uint(float f)
{
#if DXB_ON_DEVICE
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
DXB_DEV uint32_t dxb_popc16(uint32_t v)
{
#if DXB_ON_DEVICE
    return (uint32_t)__popc(v & 0xFFFFu);
#else
    return (uint32_t)__builtin_popcount(v & 0xFFFFu);
#endif
}
DXB_DEV uint32_t dxb_popc64(uint64_t v)
{
#if DXB_ON_DEVICE
    return (uint32_t)__popcll(v);
#else
    return (uint32_t)__builtin_popcountll(v);
#endif
}
DXB_DEV float dxb_uint_as_float(uint32_t u)
{
#if DXB_ON_DEVICE
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

// SSE-style min/max: max(a,b) = a > b ? a : b ; min(a,b) = a < b ? a : b
DXB_DEV float dxb_ssemax(float a, float b) { return (a > b) ? a : b; }
DXB_DEV float dxb_ssemin(float a, float b) { return (a < b) ? a : b; }

// explicit fused multiply-add (identical on host and device by IEEE-754 definition)
DXB_DEV float dxb_fma(float a, float b, float c) { return fmaf(a, b, c); }

// ---- pairs of fp32.  The BC7 encoder runs most of its arithmetic on 4-channel vectors = two pairs.  sm_90a has no
// packed fp32 instructions, so each pair is two scalar round-to-nearest operations on host and device alike, and the
// host emulator stays bit-identical (-fmad=false keeps ptxas from contracting a product into a following add; where the
// code wants a fused operation it states it with dxb_fma2).
struct dxb_f2 { float x, y; };
DXB_DEV dxb_f2 dxb_mk2(float x, float y) { dxb_f2 r; r.x = x; r.y = y; return r; }
DXB_DEV dxb_f2 dxb_fma2(dxb_f2 a, dxb_f2 b, dxb_f2 c) { return dxb_mk2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
DXB_DEV dxb_f2 dxb_add2(dxb_f2 a, dxb_f2 b) { return dxb_mk2(a.x + b.x, a.y + b.y); }
DXB_DEV dxb_f2 dxb_mul2(dxb_f2 a, dxb_f2 b) { return dxb_mk2(a.x * b.x, a.y * b.y); }
DXB_DEV dxb_f2 dxb_sub2(dxb_f2 a, dxb_f2 b) { return dxb_add2(a, dxb_mk2(-b.x, -b.y)); }
DXB_DEV dxb_f2 dxb_bc2(float v) { return dxb_mk2(v, v); }

// ---- IEEE binary16 <-> binary32 (RNE, denormals kept, overflow -> Inf) ----
DXB_DEV float dxb_half_to_float(uint16_t h)
{
#if DXB_ON_DEVICE
    return __half2float(__ushort_as_half(h));
#else
    uint32_t mant = h & 0x03FFu;
    uint32_t exp = (h & 0x7C00u);
    if (exp == 0x7C00u) exp = 0x8Fu;
    else if (exp != 0) exp = (h >> 10) & 0x1Fu;
    else if (mant != 0)
    {
        exp = 1;
        do { exp--; mant <<= 1; } while ((mant & 0x0400u) == 0);
        mant &= 0x03FFu;
    }
    else exp = (uint32_t)-112;
    uint32_t out = ((uint32_t)(h & 0x8000u) << 16) | ((exp + 112u) << 23) | (mant << 13);
    return dxb_uint_as_float(out);
#endif
}
DXB_DEV uint16_t dxb_float_to_half(float f)
{
#if DXB_ON_DEVICE
    return __half_as_ushort(__float2half_rn(f));
#else
    uint32_t iv = dxb_float_as_uint(f);
    const uint32_t sign = (iv & 0x80000000u) >> 16;
    iv &= 0x7FFFFFFFu;
    uint32_t r;
    if (iv >= 0x47800000u) r = 0x7C00u | ((iv > 0x7F800000u) ? (0x200u | ((iv >> 13) & 0x3FFu)) : 0u);
    else if (iv <= 0x33000000u) r = 0;
    else if (iv < 0x38800000u)
    {
        const uint32_t shift = 125u - (iv >> 23);
        iv = 0x800000u | (iv & 0x7FFFFFu);
        r = iv >> (shift + 1);
        const uint32_t s = (iv & ((1u << shift) - 1)) != 0;
        r += (r | s) & ((iv >> shift) & 1u);
    }
    else
    {
        iv += 0xC8000000u;
        r = ((iv + 0x0FFFu + ((iv >> 13) & 1u)) >> 13) & 0x7FFFu;
    }
    return (uint16_t)(r | sign);
#endif
}
