// dxb_launch.h — job/parameter structs shared by the kernels' translation units and the host API, plus the
// host-callable launchers each kernel TU exports (hidden visibility; not part of the C ABI).
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <cuda_runtime.h>
#include "dxb_mipjob.h"

struct dxb_job
{
    const uint8_t* src; uint8_t* dst;
    size_t srcPitch, dstPitch;
    uint32_t width, height;
    uint32_t nbx, nby;
    uint32_t firstUnit;
    uint32_t pad;
};

struct dxb_compress_params
{
    uint32_t srcFormat, dstFormat;
    uint32_t inF, outF, cflags, bcflags;
    float threshold;
    uint32_t totalUnits, njobs;
};

struct dxb_convert_params
{
    uint32_t srcFormat, dstFormat, inF, outF, flags;
    uint32_t totalUnits, njobs;
    float threshold;               // alpha threshold of 1-bit alpha destinations (B5G5R5A1)
};

struct dxb_mip_params
{
    uint32_t format, mode /*DXB_FILTER_* mode bits*/, filter, lflags;
    uint32_t totalUnits, njobs;
    dxb_tri_axis triX, triY;       // triangle filter only
};

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
// njobs == 1 (the kernel then takes hostJobs[0] by value)
void dxb_launch_bc15(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
void dxb_launch_bc7(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
// TMA-fed persistent variant (RGBA32F sources of full 4x4 blocks, equal images at a constant stride); false = not eligible, nothing launched
bool dxb_launch_bc7_tma(unsigned residentCtas, cudaStream_t stream, const dxb_job* hostJobs, const dxb_compress_params& P);
int dxb_bc7_get_feed();            // 0 direct kernel, 1-3 TMA-fed variants (dxb_k_bc7.cu)
void dxb_bc7_set_feed(int mode);
void dxb_launch_decompress(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
void dxb_launch_bc6h(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P);
void dxb_launch_convert(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P);
// Levels 1 .. levels-1 of `items` chains whose items all have the same sizes (a resize is a chain of two levels), each level
// from the stored previous one.  hostJobs: the (levels - 1) x items records laid out [level - 1][item]; jobs: their device
// copy, nullptr only when there is a single record.  P: format, mode, filter and lflags.  tri: TRIANGLE's device gather
// lists, X and Y of each level (nullptr for other filters).  gridCap: most CTAs of the generic kernel.  genericOnly: every level
// on k_mip_level (DXB200_OPT_MIP_KERNELS = 1).  launched(kernel) follows every launch; a result other than S_OK stops the chain
// and is returned.
int32_t dxb_launch_mip_chain(cudaStream_t stream, const dxb_mip_job* jobs, const dxb_mip_job* hostJobs, uint32_t items, uint32_t levels,
                             dxb_mip_params P, const dxb_tri_axis* tri, unsigned gridCap, bool genericOnly,
                             int32_t (*launched)(const char* kernel));
void dxb_launch_convert_diffuse(cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P, void* errors, uint32_t errStride);
void dxb_launch_alpha_coverage(unsigned grid, cudaStream_t stream, const dxb_job& j, uint32_t fmt, float scale, float ref, unsigned long long* count);
void dxb_launch_scale_alpha(unsigned grid, cudaStream_t stream, const dxb_job& j, uint32_t fmt, float scale);
void dxb_launch_pmalpha(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P);
// resident CTAs per SM of each kernel at its block size
int dxb_occupancy_bc15();
int dxb_occupancy_bc7();
int dxb_occupancy_bc6h();

#ifdef __CUDACC__
template <typename J>
__device__ __forceinline__ const J& dxb_find_job(const J* jobs, uint32_t njobs, const J& single, uint32_t unit)
{
    if (jobs == nullptr) return single;
    uint32_t lo = 0, hi = njobs;            // last job with firstUnit <= unit
    while (hi - lo > 1)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (jobs[mid].firstUnit <= unit) lo = mid; else hi = mid;
    }
    return jobs[lo];
}
#endif
