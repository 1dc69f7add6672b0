// tests/emul/coverage_batch.cpp — TEST INFRASTRUCTURE, never shipped: the host lock-step emulation of the batched
// ScaleMipMapsAlphaForCoverage that k_alpha_coverage / k_scale_alpha run (dxb_k_rows.cu).  Built with the emulator's compiler
// and flags (tests/emul/build.sh).
//
// It takes the library's own job table (plan_coverage_jobs) and replays each job's search from its recorded counts with the
// shared rule (dxb_coverage_scale), step by step for the whole batch as the device does: step 0 counts every level at scale 1,
// every later step only the levels >= 1 whose search still runs, and the scaling pass uses the result of all ten steps.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"
#include "dxb_pixel.cuh"
#include "dxb_mips.cuh"

static bool job_scale(const std::vector<dxb_coverage_job>& jobs, const std::vector<unsigned long long>& counts, size_t ji, uint32_t step, float* scale)
{
    const dxb_coverage_job& j = jobs[ji]; const dxb_coverage_job& b = jobs[j.item];
    const unsigned long long target = step ? counts[(size_t)j.item * DXB_COVERAGE_STEPS] : 0ull;
    return dxb_coverage_scale(target, b.width, b.height, counts.data() + ji * DXB_COVERAGE_STEPS, step, j.width, j.height, scale);
}

// items chains in ScratchImage layout, chain `it` at src + it * chainBytes (levels described by offsets / widths / heights /
// pitches, equal for all items); results at dst + it * chainBytes.  Level 0 is copied as the per-item call copies it.
extern "C" int32_t emul_scale_mips_alpha_batch(const uint8_t* src, uint8_t* dst, size_t chainBytes, size_t items, const size_t* offsets,
                                               const size_t* widths, const size_t* heights, const size_t* pitches, size_t levels,
                                               uint32_t fmt, float ref)
{
    std::vector<dxb200_image> s(items * levels), d(items * levels);
    for (size_t it = 0; it < items; ++it)
        for (size_t l = 0; l < levels; ++l)
        {
            dxb200_image im = { widths[l], heights[l], fmt, pitches[l], pitches[l] * heights[l], nullptr };
            im.pixels = const_cast<uint8_t*>(src) + it * chainBytes + offsets[l]; s[it * levels + l] = im;
            im.pixels = dst + it * chainBytes + offsets[l]; d[it * levels + l] = im;
        }
    for (size_t it = 0; it < items; ++it)
    {
        const int32_t hr = plan_alpha_coverage(s.data() + it * levels, levels, d.data() + it * levels);
        if (hr != DXB_S_OK) return hr;
    }
    CoveragePlan cp;
    int32_t hr = plan_coverage_jobs(s.data(), d.data(), items, levels, ref, &cp);
    if (hr != DXB_S_OK) return hr;
    const std::vector<dxb_coverage_job>& jobs = cp.jobs;
    std::vector<unsigned long long> counts(jobs.size() * DXB_COVERAGE_STEPS, 0);
    for (uint32_t step = 0; step < DXB_COVERAGE_STEPS; ++step)
        for (size_t ji = step ? items : 0; ji < jobs.size(); ++ji)
        {
            float scale = 1.0f;
            if (!job_scale(jobs, counts, ji, step, &scale)) continue;
            const dxb_coverage_job& j = jobs[ji];
            unsigned long long n = 0;
            for (uint32_t y = 0; y + 1 < j.height; ++y)
                for (uint32_t x = 0; x + 1 < j.width; ++x)
                {
                    const uint8_t* r0 = j.src + y * j.srcPitch; const uint8_t* r1 = r0 + j.srcPitch;
                    n += dxb_alpha_coverage_cell(dxb_load_pixel(fmt, r0, x).w, dxb_load_pixel(fmt, r1, x).w,
                                                 dxb_load_pixel(fmt, r0, x + 1).w, dxb_load_pixel(fmt, r1, x + 1).w, scale, ref);
                }
            counts[ji * DXB_COVERAGE_STEPS + step] = n;
        }
    for (size_t it = 0; it < items; ++it)
        memcpy(d[it * levels].pixels, s[it * levels].pixels, s[it * levels].slicePitch);
    for (size_t ji = items; ji < jobs.size(); ++ji)
    {
        float scale = 1.0f;
        (void)job_scale(jobs, counts, ji, DXB_COVERAGE_STEPS, &scale);
        const dxb_coverage_job& j = jobs[ji];
        for (uint32_t y = 0; y < j.height; ++y)
            for (uint32_t x = 0; x < j.width; ++x) dxb_scale_alpha_pixel(fmt, j.src + y * j.srcPitch, j.dst + y * j.dstPitch, x, scale);
    }
    return DXB_S_OK;
}
