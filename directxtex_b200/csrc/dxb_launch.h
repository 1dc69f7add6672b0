// dxb_launch.h — the host-callable launchers each kernel TU exports (hidden visibility; not part of the C ABI), on the job and
// parameter structs of dxb_jobs.h.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <cuda_runtime.h>
#include "dxb_jobs.h"

#ifndef DXB_BC7_WARPS
#define DXB_BC7_WARPS 8       // warps per CTA of k_compress_bc7 (two blocks per warp, 8.6 KB dynamic shared per warp)
#endif
#ifndef DXB_BC7_MINB
#define DXB_BC7_MINB 3        // __launch_bounds__ min CTAs per SM of k_compress_bc7
#endif
#ifndef DXB_BC6H_WARPS
#define DXB_BC6H_WARPS 8      // warps per CTA of k_compress_bc6h (two blocks per warp)
#endif
#ifndef DXB_BC6H_MINB
#define DXB_BC6H_MINB 2
#endif

// launchers: `grid` CTAs on `stream`; hostJobs = the njobs job records on the host, jobs = their device copy, or nullptr when
// njobs == 1 (the kernel then takes hostJobs[0] by value).  Each enqueues one kernel and returns the name of its __global__
// function without template arguments.
const char* dxb_launch_bc15(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
// RGBA32F sources of full 4x4 blocks, equal images at a constant stride: the TMA-fed persistent kernel on `residentCtas` CTAs
// (DXB200_OPT_BC7_FEED); everything else: the direct kernel on `grid` CTAs
const char* dxb_launch_bc7(unsigned grid, unsigned residentCtas, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs,
                           const dxb_compress_params& P);
int dxb_bc7_get_feed();            // 0 direct kernel, 1-3 TMA-fed variants (dxb_k_bc7.cu)
void dxb_bc7_set_feed(int mode);
const char* dxb_launch_decompress(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
const char* dxb_launch_bc6h(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
const char* dxb_launch_convert(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P);
// Levels 1 .. levels-1 of `items` chains whose items all have the same sizes (a resize is a chain of two levels), each level
// from the stored previous one.  hostJobs: the (levels - 1) x items records laid out [level - 1][item]; jobs: their device
// copy, nullptr only when there is a single record.  P: format, mode, filter and lflags.  tri: TRIANGLE's device gather
// lists, X and Y of each level (nullptr for other filters).  gridCap: most CTAs of the generic kernel.  genericOnly: every level
// on k_mip_level (DXB200_OPT_MIP_KERNELS = 1).  launched(kernel) follows every launch; a result other than S_OK stops the chain
// and is returned.
int32_t dxb_launch_mip_chain(cudaStream_t stream, const dxb_mip_job* jobs, const dxb_mip_job* hostJobs, uint32_t items, uint32_t levels,
                             dxb_mip_params P, const dxb_tri_axis* tri, unsigned gridCap, bool genericOnly,
                             int32_t (*launched)(const char* kernel));
const char* dxb_launch_convert_diffuse(cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P, void* errors, uint32_t errStride);
// ScaleMipMapsAlphaForCoverage of a batch of chains (dxb_coverage_job): `jobs` is the device table, `counts` DXB_COVERAGE_STEPS
// counters per job, zero before step 0.  dxb_launch_alpha_coverage enqueues search step `step` of every job; dxb_launch_scale_alpha,
// after the last step, scales every level >= 1 by the result of its search.
const char* dxb_launch_alpha_coverage(unsigned grid, cudaStream_t stream, const dxb_coverage_job* jobs, const dxb_coverage_params& P,
                                      unsigned long long* counts, uint32_t step);
const char* dxb_launch_scale_alpha(unsigned grid, cudaStream_t stream, const dxb_coverage_job* jobs, const dxb_coverage_params& P,
                                   const unsigned long long* counts);
// IsAlphaAllOpaque of a batch (dxb_alpha_opaque.h): P.dstFormat = DXB_SCAN_ALPHA_OPAQUE and every job's dst = its result word, zero
// before the launch.  BC1 / BC2 / BC3 / BC7 sources run on the generic k_decompress, one thread per block; uncompressed sources on
// the generic k_convert, one thread per pixel.
const char* dxb_launch_alpha_opaque_blocks(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
const char* dxb_launch_alpha_opaque_pixels(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P);
// texconv's channel steps (dxb_channel_steps.h) on the generic k_convert, one thread per pixel: P.srcFormat == P.dstFormat, P.steps
// and P.key; a job's dst may be its src (same pointer and pitch)
const char* dxb_launch_channel_steps(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P);
const char* dxb_launch_pmalpha(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P);
// resident CTAs per SM of each kernel at its block size
int dxb_occupancy_bc15();
int dxb_occupancy_bc7();
int dxb_occupancy_bc6h();

#ifdef __CUDACC__
// the job of work unit `unit`; `first` names the job's prefix sum of units when a table has more than one (dxb_coverage_job)
template <typename J>
__device__ __forceinline__ const J& dxb_find_job(const J* jobs, uint32_t njobs, const J& single, uint32_t unit, uint32_t J::*first = &J::firstUnit)
{
    if (jobs == nullptr) return single;
    uint32_t lo = 0, hi = njobs;            // last job with first <= unit
    while (hi - lo > 1)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (jobs[mid].*first <= unit) lo = mid; else hi = mid;
    }
    return jobs[lo];
}
#endif
