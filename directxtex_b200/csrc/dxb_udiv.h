// dxb_udiv.h — unsigned division by a run-time constant (Granlund / Montgomery round-up form): q = n / d for every 32-bit n.
// dxb_udiv_make runs where the divisor is known (the host, when a launch is planned); dxb_udiv_do in the kernel.  The host build
// of dxb_udiv_do (tests/probe) takes the high word of the 64-bit product where the device has __umulhi.
#pragma once
#include "dxb_portable.h"

#if DXB_ON_DEVICE
  #define DXB_UDIV_MAKE __host__ __device__ inline
#else
  #define DXB_UDIV_MAKE static inline
#endif

struct dxb_udiv { uint32_t d, M, sh; };
DXB_UDIV_MAKE dxb_udiv dxb_udiv_make(uint32_t d)
{
    dxb_udiv r; r.d = d; r.M = 0; r.sh = 0;
    if (d > 1u)
    {
        uint32_t l = 0; while ((1ull << l) < d) ++l;                      // ceil(log2 d)
        r.M = (uint32_t)(((1ull << 32) * ((1ull << l) - d)) / d + 1ull); r.sh = l - 1u;
    }
    return r;
}
DXB_DEV uint32_t dxb_udiv_do(uint32_t n, const dxb_udiv& k)
{
    if (k.d <= 1u) return n;
#if DXB_ON_DEVICE
    const uint32_t t = __umulhi(k.M, n);
#else
    const uint32_t t = (uint32_t)(((uint64_t)k.M * n) >> 32);
#endif
    return (t + ((n - t) >> 1)) >> k.sh;
}
