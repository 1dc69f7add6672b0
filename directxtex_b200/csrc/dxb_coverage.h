// dxb_coverage.h — the rule of ScaleMipMapsAlphaForCoverage's search (DirectXTexMipmaps.cpp:300-355), stated once for the host
// planner (dxb_plan.h, the emulator) and the coverage kernels (dxb_k_rows.cu).  The search depends only on the coverage values
// it has seen, and each of them is an integer count of covered sub-samples, so the counts recorded so far are its whole state:
// a kernel can replay it per job from the counts of the earlier launches, without a host round trip.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
  #define DXB_HD __host__ __device__ __forceinline__
#else
  #define DXB_HD inline
#endif

// the coverage search runs exactly this many steps unless a step hits the target (EstimateAlphaScaleForCoverage's N)
#define DXB_COVERAGE_STEPS 10u

// CalculateAlphaCoverage's result (:300-304): `count` covered samples of the 8x8 samples in each of the (w - 1)(h - 1) cells of
// 2x2 pixels; 0 for an image without a cell
DXB_HD float alpha_coverage_fraction(uint64_t count, size_t w, size_t h)
{
    const float cscale = static_cast<float>((w - 1) * (h - 1) * 8 * 8);
    return cscale > 0.0f ? static_cast<float>(count) / cscale : 0.0f;
}

// EstimateAlphaScaleForCoverage (:310-355), a bisection on [0, 4] that starts at 1, replayed from the coverage of its steps
// 0 .. k-1 (cov(i) = the coverage step i measured).  Returns true with *scale = the scale step k evaluates (k = DXB_COVERAGE_STEPS:
// the search's result), or false when the search left its loop at an earlier step because that step's coverage equalled the
// target; *scale is then that step's scale, which is the result.
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
template <typename CoverageOfStep>
DXB_HD bool dxb_coverage_replay(float target, uint32_t k, const CoverageOfStep& cov, float* scale)
{
    float lo = 0.0f, hi = 4.0f, s = 1.0f;
    for (uint32_t i = 0; i < k; ++i)
    {
        const float c = cov(i);
        if (c < target) lo = s;
        else if (c > target) hi = s;
        else { *scale = s; return false; }
        s = (lo + hi) * 0.5f;
    }
    *scale = s;
    return true;
}

// The replay of one (item, level) image from its recorded counts: baseCount = the item's level-0 count at scale 1 (the target),
// bw x bh = level 0's size, counts[0 .. k) = this level's counts at steps 0 .. k-1, w x h = this level's size.
DXB_HD bool dxb_coverage_scale(uint64_t baseCount, size_t bw, size_t bh, const unsigned long long* counts, uint32_t k, size_t w, size_t h,
                               float* scale)
{
    struct Recorded
    {
        const unsigned long long* c; size_t w, h;
        DXB_HD float operator()(uint32_t i) const { return alpha_coverage_fraction(c[i], w, h); }
    };
    return dxb_coverage_replay(k ? alpha_coverage_fraction(baseCount, bw, bh) : 0.0f, k, Recorded{ counts, w, h }, scale);
}
