// dxb_k_bc15.cu — BC1/2/3/4/5: one THREAD per 4x4 block (bit-exact fp32 restatement, dxb_bc15.cuh).
//   k_compress_bc15            generic: any implemented source format, any flags (run-time switches)
//   k_compress_bc15_t<DF,SF>   hot (destination, source) pairs with the default flags: formats, conversion flags and
//                              "no dithering" are compile-time constants.  The generic kernel carries every format
//                              loader, the sRGB powf paths and all five encoders with their dither variants: 106 k SASS
//                              instructions, and it ran at 13 % issue utilisation stalled on instruction fetch.
//                              No pair names an sRGB format: an sRGB call matches its twins' pair (dxb_make_linear).
#include <algorithm>
#include "dxb_launch.h"
#include "dxb_bc15.cuh"

// Launch shape per destination format.  The encoders are thousands of instructions of mostly straight-line code per block and
// instruction fetch is their top stall, so what helps is more resident warps and warps that run the same code at the same time:
//   registers  BC3 / BC4 / BC5: 64 (32 warps/SM, spills and all).  BC1 / BC2 keep the 16 pixels of their Newton fit in registers and
//              lose at 64: compiler's choice.
//   CTA shape  BC3: 512 threads that start every block together (one barrier per block).  BC1 and BC4 lose with big CTAs.
#ifndef DXB_BC3_THREADS
#define DXB_BC3_THREADS 512u
#endif
__host__ __device__ constexpr uint32_t dxb_bc15_threads(uint32_t df) { return (df == 77u) ? DXB_BC3_THREADS : 128u; }
__host__ __device__ constexpr bool dxb_bc15_sync(uint32_t df) { return df == 77u; }
template <bool GENERIC, uint32_t DF, uint32_t SF>
__device__ __forceinline__ void bc15_body(const dxb_job* __restrict__ jobs, const dxb_job& single, const dxb_compress_params& P)
{
    const uint32_t srcFormat = GENERIC ? P.srcFormat : SF, dstFormat = GENERIC ? P.dstFormat : DF;
    const uint32_t inF = GENERIC ? P.inF : dxb_convert_flags(SF), outF = GENERIC ? P.outF : dxb_convert_flags(DF);
    const uint32_t cflags = GENERIC ? P.cflags : dxb_bc15_default_cflags(DF);
    const uint32_t bcflags = GENERIC ? P.bcflags : 0u;
    const uint32_t stride = gridDim.x * blockDim.x;
    // SYNC: every warp of the CTA starts a block together, so that the warps share their instruction fetches.  The loop bound is
    // CTA-uniform; threads past the end skip the body.
    constexpr bool SYNC = !GENERIC && dxb_bc15_sync(GENERIC ? 0u : DF);
    for (uint32_t base = blockIdx.x * blockDim.x; base < P.totalUnits; base += stride)
    {
        if (SYNC) __syncthreads();
        const uint32_t unit = base + threadIdx.x;
        if (unit >= P.totalUnits) continue;
        const dxb_job& j = dxb_find_job(jobs, P.njobs, single, unit);
        const uint32_t local = unit - j.firstUnit;
        const uint32_t by = local / j.nbx, bx = local - by * j.nbx;
        dxb_image_desc img; img.pixels = j.src; img.rowPitch = j.srcPitch; img.width = j.width; img.height = j.height; img.format = srcFormat;
        dxb_px px[16];
        if (GENERIC) dxb_gather_block(img, bx, by, inF, outF, cflags, px);
        else dxb_gather_block_t<GENERIC ? 2u : SF>(img, bx, by, inF, outF, cflags, px);
        const uint32_t bs = dxb_bc_block_bytes(dstFormat);
        uint8_t* out = j.dst + (size_t)by * j.dstPitch + (size_t)bx * bs;
        __align__(16) uint8_t blk[16];
        dxb_encode_block_bc15(dstFormat, px, bcflags, P.threshold, blk);
        if (bs == 8) *reinterpret_cast<uint2*>(out) = *reinterpret_cast<const uint2*>(blk);
        else *reinterpret_cast<uint4*>(out) = *reinterpret_cast<const uint4*>(blk);
    }
}

__global__ void __launch_bounds__(128) k_compress_bc15(const dxb_job* __restrict__ jobs, dxb_job single, dxb_compress_params P)
{
    bc15_body<true, 0, 0>(jobs, single, P);
}
#ifndef DXB_BC3_MINB
#define DXB_BC3_MINB 2
#endif
__host__ __device__ constexpr int dxb_bc15_minb(uint32_t df) { return (df == 71u || df == 74u) ? 3 : (df == 77u) ? DXB_BC3_MINB : 8; }
template <uint32_t DF, uint32_t SF>
__global__ void __launch_bounds__(dxb_bc15_threads(DF), dxb_bc15_minb(DF)) k_compress_bc15_t(const dxb_job* __restrict__ jobs, dxb_job single, dxb_compress_params P)
{
    bc15_body<false, DF, SF>(jobs, single, P);
}

// hot pairs: colour formats x {RGBA8, BGRA8, RGBA16F, RGBA32F}; BC4 x {R8, RGBA8, R32F, RGBA32F}; BC5 x {R8G8, RGBA8, R32G32F, RGBA32F}
#define DXB_BC15_PAIRS(X) \
    X(71, 28) X(71, 87) X(71, 10) X(71, 2) X(74, 28) X(74, 87) X(74, 10) X(74, 2) X(77, 28) X(77, 87) X(77, 10) X(77, 2) \
    X(80, 61) X(80, 28) X(80, 41) X(80, 2) X(81, 61) X(81, 28) X(81, 41) X(81, 2) \
    X(83, 49) X(83, 28) X(83, 16) X(83, 2) X(84, 49) X(84, 28) X(84, 16) X(84, 2)

void dxb_launch_bc15(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P)
{
    // sRGB formats run their twins' kernels: an sRGB step is resolved into P.cflags, and the specialised kernels take only
    // the default flag set
    const uint32_t df = dxb_make_linear(P.dstFormat), sf = dxb_make_linear(P.srcFormat);
    if (P.bcflags == 0 && P.cflags == dxb_bc15_default_cflags(df))
    {
#define DXB_X(DF, SF) if (df == DF && sf == SF) { k_compress_bc15_t<DF, SF><<<std::max(1u, grid * 128u / dxb_bc15_threads(DF)), dxb_bc15_threads(DF), 0, stream>>>(jobs, hostJobs[0], P); return; }
        DXB_BC15_PAIRS(DXB_X)
#undef DXB_X
    }
    k_compress_bc15<<<grid, 128, 0, stream>>>(jobs, hostJobs[0], P);
}
int dxb_occupancy_bc15()
{
    // the densest of the specialised kernels (BC4 at 64 registers, 128-thread CTAs); callers size their grids in 128-thread CTAs and
    // cap them at 4 x SMs x this
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_compress_bc15_t<80, 61>, 128, 0) != cudaSuccess) { (void)cudaGetLastError(); b = 1; }
    return b > 0 ? b : 1;
}
