// dxb_k_bc7.cu — k_compress_bc7: one HALF-WARP per 4x4 block (two blocks per warp), BC7 mode/partition search (dxb_bc7.cuh)
#include <cuda.h>            // CUtensorMap and the cuTensorMapEncodeTiled prototype only: the entry point is resolved at run time
#include <stdlib.h>
#include <algorithm>
#include <atomic>
#include "dxb_launch.h"
#include "dxb_dispatch.h"
#include "dxb_bc7.cuh"
#include "dxb_udiv.h"

template <bool THREE>
__global__ void __launch_bounds__(DXB_BC7_WARPS * 32, DXB_BC7_MINB) k_compress_bc7(const dxb_job* __restrict__ jobs, dxb_job single, dxb_compress_params P)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    dxb_bc7_scratch* scratch = (dxb_bc7_scratch*)smem_raw;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, hl = lane & 15u;
    dxb_bc7_scratch* S = &scratch[warp];
    const uint32_t stride = gridDim.x * DXB_BC7_WARPS;
    const uint32_t npairs = (P.totalUnits + 1u) >> 1;
    // every warp of the CTA runs the same number of iterations (a warp without a pair encodes dummy pixels and
    // stores nothing), so CTA-wide barriers inside the encoder are legal
    for (uint32_t base = blockIdx.x * DXB_BC7_WARPS; base < npairs; base += stride)
    {
        // lanes 0-15 stage block 2*pair, lanes 16-31 block 2*pair+1; lane = pixel
        const uint32_t unit = 2u * (base + warp) + (lane >> 4);
        uint8_t* out = nullptr;
        dxb_px ldr = dxb_make_px(0.0f, 0.0f, 0.0f, 255.0f);
        if (unit < P.totalUnits)
        {
            const dxb_job& j = dxb_find_job(jobs, P.njobs, single, unit);
            const uint32_t local = unit - j.firstUnit;
            const uint32_t by = local / j.nbx, bx = local - by * j.nbx;
            // CompressBC's partial-block replication with source map {0,0,0,1} (DirectXTexCompress.cpp:159-187)
            const uint32_t x0 = bx * 4, y0 = by * 4;
            const uint32_t pw = (j.width - x0 < 4u) ? (j.width - x0) : 4u;
            const uint32_t ph = (j.height - y0 < 4u) ? (j.height - y0) : 4u;
            const uint32_t s = hl & 3u, t = hl >> 2;
            const uint32_t sc = (s < pw) ? s : ((s == 3u && pw > 1u) ? 1u : 0u);
            const uint32_t tr = (t < ph) ? t : ((t == 3u && ph > 1u) ? 1u : 0u);
            dxb_px v = dxb_load_pixel(P.srcFormat, j.src + (size_t)(y0 + tr) * j.srcPitch, x0 + sc);
            v = dxb_convert_pixel(v, P.inF, P.outF, P.cflags);
            ldr = dxb_make_px(dxb_bc7_ldr(v.x), dxb_bc7_ldr(v.y), dxb_bc7_ldr(v.z), dxb_bc7_ldr(v.w));
            out = j.dst + (size_t)by * j.dstPitch + (size_t)bx * 16u;
        }
        S->px[lane] = ldr;
        if (hl == 0) S->out[lane >> 4] = out;
        __syncwarp();
        dxb_bc7_encode_pair<THREE>(S, P.bcflags);
        __syncwarp();
    }
}

// raises kernel K's dynamic shared memory limit to `bytes` on the current device, on the first call for K there; false when the
// runtime refused.  A function attribute belongs to the module loaded in one device's context, so every device needs its own call.
template <auto K>
static bool smem_limit(size_t bytes)
{
    constexpr int kDevices = 64;
    static std::atomic<int> state[kDevices];             // per device ordinal: 0 = not set yet, 1 = raised, -1 = refused
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); dev = -1; }
    if (dev >= 0 && dev < kDevices && state[dev].load(std::memory_order_relaxed) != 0) return state[dev].load(std::memory_order_relaxed) > 0;
    const bool ok = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess;
    if (!ok) (void)cudaGetLastError();
    if (dev >= 0 && dev < kDevices) state[dev].store(ok ? 1 : -1, std::memory_order_relaxed);
    return ok;
}

static const size_t kBC7Smem = sizeof(dxb_bc7_scratch) * DXB_BC7_WARPS;
int dxb_occupancy_bc7()
{
    // Both direct instantiations get their limit here, at initialisation.  Under lazy module loading that also loads both, and the
    // kernels loaded early decide where later ones land in device memory: with only <false> loaded here, C5's BC4 kernel ran 2 %
    // slower on an H100 with identical SASS.
    int b = 0;
    if (!smem_limit<k_compress_bc7<false>>(kBC7Smem) || !smem_limit<k_compress_bc7<true>>(kBC7Smem) ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_compress_bc7<false>, DXB_BC7_WARPS * 32, kBC7Smem) != cudaSuccess) { (void)cudaGetLastError(); b = 1; }
    return b > 0 ? b : 1;
}


// ------------------------------------------------------------------------------------------------ TMA-fed variant
// k_compress_bc7_tma: the same encoder (dxb_bc7_encode_pair) behind a persistent CTA loop whose RGBA32F source tiles arrive by
// TMA 2D tile loads (north_star; the reference's accelerator path stages blocks the same way, BCDirectCompute.cpp:395-431):
//   * one tile = 16 consecutive blocks of a block row = 64 x 4 pixels x 16 B = 4 KB = the box {256 floats, 4 rows, 1 image} of a rank-3
//     tensor map {width * 4 floats, height, images} with strides {rowPitch, image stride}; a block row whose width is not a multiple of
//     64 ends in a zero-filled partial tile whose extra blocks are simply not stored;
//   * one `cp.async.bulk.tensor.3d` per tile, issued by thread 0, completion on an mbarrier (complete_tx::bytes); every lane then
//     takes its pixel from the tile with one 128-bit shared load and converts it exactly like the direct kernel does;
//   * the 4 KB landing buffer is free again as soon as every warp has taken its pixels (the barrier at the top of the iteration), so
//     the next tile is requested right there and has the whole encode of the current tile to arrive; with it the CTA needs 76.0 KB of
//     shared memory, which still leaves 3 CTAs per SM resident within the 228 KB of an H100 SM;
//   * tiles are handed out by an atomic counter (blocks with alpha cost more than opaque ones); the counter is read one tile ahead
//     of the request, so its round trip is off the critical path too.  T.counter == nullptr: statically strided tiles.
// Eligibility (launch_bc7_tma): RGBA32F source, full 4x4 blocks only (partial blocks need CompressBC's {0,0,0,1} replication,
// which a tensor map's zero fill cannot express), 16-byte aligned rows, images of one size at a constant pointer stride.
// The tile index is split into (image, block row, tile column) with dxb_udiv (dxb_udiv.h).

struct dxb_bc7_tma_params
{
    uint8_t* dst0; size_t dstPitch, dstImageStride;
    uint32_t nbx, tilesX, tilesPerImage, totalTiles;
    dxb_udiv divImage, divRow;        // tile / tilesPerImage, (tile in image) / tilesX
    uint32_t* counter;
};

#define DXB_BC7_TILE_BYTES 4096u

__device__ __forceinline__ uint32_t dxb_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// PLAIN: no sRGB conversion flag (the default, and every BC7_UNORM call without TEX_FILTER_SRGB_*).  ConvertScanline from
// RGBA32F to BC7_UNORM is then a clamp to [0, 1]: with both formats' conversion flags as compile-time constants dxb_convert_pixel
// folds to it.  The other flag sets keep the run-time branches.
template <bool THREE, bool PLAIN>
__global__ void __launch_bounds__(DXB_BC7_WARPS * 32, DXB_BC7_MINB) k_compress_bc7_tma(const __grid_constant__ CUtensorMap tmap, dxb_bc7_tma_params T, dxb_compress_params P)
{
    static_assert(DXB_BC7_WARPS == 8, "a tile is 16 blocks = 8 warps x 2");
    extern __shared__ __align__(128) unsigned char smem_tma[];
    const float4* tileBuf = (const float4*)smem_tma;                      // [row 0..3][pixel 0..63]
    uint64_t* mbar = (uint64_t*)(smem_tma + DXB_BC7_TILE_BYTES);
    volatile uint32_t* tileOf = (volatile uint32_t*)(mbar + 1);           // {tile, image, block row, tile column} of the data the barrier's current phase delivers
    dxb_bc7_scratch* scratch = (dxb_bc7_scratch*)(smem_tma + DXB_BC7_TILE_BYTES + 128u);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, hl = lane & 15u;
    dxb_bc7_scratch* S = &scratch[warp];
    const uint32_t barAddr = dxb_smem_u32(mbar), tileAddr = dxb_smem_u32(tileBuf);

    // thread 0: request `tile` (or publish the end marker)
    auto request = [&](uint32_t tile)
    {
        tileOf[0] = tile;
        if (tile < T.totalTiles)
        {
            // everything the other 255 threads need travels with the tile, and the two divisions are multiplications: this runs on one
            // thread between two CTA barriers, so every instruction here delays all eight warps
            const uint32_t img = dxb_udiv_do(tile, T.divImage), r = tile - img * T.tilesPerImage;
            const uint32_t by = dxb_udiv_do(r, T.divRow), tx = r - by * T.tilesX;
            tileOf[1] = img; tileOf[2] = by; tileOf[3] = tx;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(barAddr), "r"(DXB_BC7_TILE_BYTES) : "memory");
            asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                         :: "r"(tileAddr), "l"(&tmap), "r"(barAddr), "r"((int)(tx * 256u)), "r"((int)(by * 4u)), "r"((int)img) : "memory");
        }
        else
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(barAddr) : "memory");
    };
    // tile sequence of this CTA: its own index first, then either the counter's hand-outs or a grid stride.  `ahead` = the tile after
    // the one being requested (thread 0 only).
    uint32_t ahead = 0;
    if (threadIdx.x == 0)
    {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(barAddr) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        request(blockIdx.x);
        ahead = T.counter ? gridDim.x + atomicAdd(T.counter, 1u) : blockIdx.x + gridDim.x;
    }
    __syncthreads();
    uint32_t parity = 0;
    for (;;)
    {
        // wait for the tile (and the tile index published with it)
        asm volatile("{\n\t.reg .pred P1;\n\tDXB_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t@P1 bra DXB_DONE;\n\tbra DXB_WAIT;\n\tDXB_DONE:\n\t}"
                     :: "r"(barAddr), "r"(parity) : "memory");
        parity ^= 1u;
        const uint32_t tile = tileOf[0];
        if (tile >= T.totalTiles) break;
        const uint32_t img = tileOf[1], by = tileOf[2], tx = tileOf[3];
        const uint32_t blk = warp * 2u + (lane >> 4), bx = tx * 16u + blk;
        uint8_t* out = nullptr;
        dxb_px ldr = dxb_make_px(0.0f, 0.0f, 0.0f, 255.0f);
        if (bx < T.nbx)
        {
            const float4 f = tileBuf[(hl >> 2) * 64u + blk * 4u + (hl & 3u)];
            const dxb_px v = PLAIN ? dxb_convert_pixel(dxb_make_px(f.x, f.y, f.z, f.w), dxb_convert_flags(DXB_FMT_R32G32B32A32_FLOAT),
                                                       dxb_convert_flags(DXB_FMT_BC7_UNORM), 0u)
                                   : dxb_convert_pixel(dxb_make_px(f.x, f.y, f.z, f.w), P.inF, P.outF, P.cflags);
            ldr = dxb_make_px(dxb_bc7_ldr(v.x), dxb_bc7_ldr(v.y), dxb_bc7_ldr(v.z), dxb_bc7_ldr(v.w));
            out = T.dst0 + (size_t)img * T.dstImageStride + (size_t)by * T.dstPitch + (size_t)bx * 16u;
        }
        S->px[lane] = ldr;
        if (hl == 0) S->out[lane >> 4] = out;
        __syncthreads();                // every warp has taken its pixels (and the tile index): the landing buffer is free
        if (threadIdx.x == 0)
        {
            const uint32_t nxt = ahead;
            request(nxt);
            // hand-out for the iteration after the next; its value is not needed before the next request, so the round trip hides
            ahead = (nxt >= T.totalTiles) ? nxt : (T.counter ? gridDim.x + atomicAdd(T.counter, 1u) : nxt + gridDim.x);
        }
        dxb_bc7_encode_pair<THREE>(S, P.bcflags);
        __syncwarp();
    }
}

typedef CUresult (*dxb_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                        const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static dxb_encode_tiled_fn encode_tiled()
{
    // the one driver-API entry point the library needs, resolved through the runtime (no link against libcuda)
    static const dxb_encode_tiled_fn fn = []() -> dxb_encode_tiled_fn
    {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { (void)cudaGetLastError(); return nullptr; }
        return (dxb_encode_tiled_fn)p;
    }();
    return fn;
}

static const size_t kBC7TmaSmem = DXB_BC7_TILE_BYTES + 128u + sizeof(dxb_bc7_scratch) * DXB_BC7_WARPS;

// mode: 0 = direct kernel only, 1 = TMA with the atomic tile counter, 2 = TMA with statically strided tiles, 3 = TMA with one CTA per
// tile, 4 = automatic (default): mode 1 for batches of images, the direct kernel for a single image.  DXB200_BC7_TMA / dxb200_set_option
// select.  Static striding loses to any dynamic hand-out (tile costs differ); for a batch one tensor map serves every image, so the
// TMA feed saves the per-block job search.  The feed is not what bounds the encoder (issue-bound); the persistent loop pays two
// CTA-wide synchronisations per tile and saves the job lookup.
static std::atomic<int> g_bc7_feed{-1};
int dxb_bc7_get_feed()
{
    int m = g_bc7_feed.load(std::memory_order_relaxed);
    if (m < 0) { const char* e = getenv("DXB200_BC7_TMA"); m = e ? atoi(e) : 4; if (m < 0 || m > 4) m = 4; g_bc7_feed.store(m, std::memory_order_relaxed); }
    return m;
}
void dxb_bc7_set_feed(int mode) { g_bc7_feed.store((mode < 0 || mode > 4) ? 4 : mode, std::memory_order_relaxed); }
static int bc7_tma_mode() { return dxb_bc7_get_feed(); }

// the TMA-fed kernel when the feed mode and the batch allow it; false = not eligible, nothing launched
static bool launch_bc7_tma(unsigned residentCtas, cudaStream_t stream, const dxb_job* hostJobs, const dxb_compress_params& P, bool three)
{
    int mode = bc7_tma_mode();
    if (mode == 4) mode = (P.njobs > 1u) ? 1 : 0;
    if (mode == 0 || P.srcFormat != DXB_FMT_R32G32B32A32_FLOAT || P.njobs == 0) return false;
    const dxb_job& j0 = hostJobs[0];
    if ((j0.width & 3u) || (j0.height & 3u) || (j0.srcPitch & 15u) || ((uintptr_t)j0.src & 15u) || j0.srcPitch >= (1ull << 40)) return false;
    ptrdiff_t srcStride = (ptrdiff_t)j0.srcPitch * j0.height, dstStride = (ptrdiff_t)j0.dstPitch * j0.nby;
    if (P.njobs > 1)
    {
        srcStride = hostJobs[1].src - j0.src; dstStride = hostJobs[1].dst - j0.dst;
        if (srcStride < (ptrdiff_t)(j0.srcPitch * (size_t)(j0.height - 1u) + (size_t)j0.width * 16u) || (srcStride & 15) || srcStride >= (ptrdiff_t)(1ll << 40) || dstStride <= 0) return false;
        for (uint32_t i = 1; i < P.njobs; ++i)
        {
            const dxb_job& j = hostJobs[i];
            if (j.width != j0.width || j.height != j0.height || j.srcPitch != j0.srcPitch || j.dstPitch != j0.dstPitch ||
                j.src != j0.src + (ptrdiff_t)i * srcStride || j.dst != j0.dst + (ptrdiff_t)i * dstStride) return false;
        }
    }
    const dxb_encode_tiled_fn enc = encode_tiled();
    if (!enc) return false;
    CUtensorMap tmap;
    const cuuint64_t dims[3] = { (cuuint64_t)j0.width * 4u, j0.height, P.njobs };
    const cuuint64_t strides[2] = { (cuuint64_t)j0.srcPitch, (cuuint64_t)srcStride };
    const cuuint32_t box[3] = { 256u, 4u, 1u }, estr[3] = { 1u, 1u, 1u };
    if (dims[0] > 0x7FFFFFFFull || dims[1] > 0x7FFFFFFFull ||          // tile coordinates travel as int32
        enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)j0.src, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return false;
    dxb_bc7_tma_params T;
    T.dst0 = j0.dst; T.dstPitch = j0.dstPitch; T.dstImageStride = (size_t)dstStride;
    T.nbx = j0.nbx; T.tilesX = (j0.nbx + 15u) / 16u; T.tilesPerImage = T.tilesX * j0.nby;
    T.divImage = dxb_udiv_make(T.tilesPerImage); T.divRow = dxb_udiv_make(T.tilesX);
    const uint64_t total = (uint64_t)T.tilesPerImage * P.njobs;
    if (total >= 0x7FFFFFFFull) return false;
    T.totalTiles = (uint32_t)total;
    // mode 3: one CTA per tile (the hardware CTA scheduler hands the tiles out)
    const unsigned grid = (mode == 3) ? (unsigned)total : (unsigned)std::min<uint64_t>(total, residentCtas ? residentCtas : 1u);
    // the source is RGBA32F and the destination BC7_UNORM(_SRGB), so P.inF / P.outF are the PLAIN kernel's constants; only the
    // resolved sRGB flags can differ
    return dxb_on_bool(three, [&](auto THREE) { return dxb_on_bool(P.cflags == 0u, [&](auto PLAIN)
    {
        constexpr bool T3 = decltype(THREE)::value, PL = decltype(PLAIN)::value;
        if (!smem_limit<k_compress_bc7_tma<T3, PL>>(kBC7TmaSmem)) return false;
        T.counter = nullptr;
        if (mode == 1)
        {
            // counts the tiles handed out after the first one of every CTA (its own index); stream-ordered allocation, released after the launch
            if (cudaMallocAsync((void**)&T.counter, sizeof(uint32_t), stream) != cudaSuccess) { (void)cudaGetLastError(); return false; }
            cudaMemsetAsync(T.counter, 0, sizeof(uint32_t), stream);
        }
        k_compress_bc7_tma<T3, PL><<<grid, DXB_BC7_WARPS * 32, kBC7TmaSmem, stream>>>(tmap, T, P);
        if (T.counter) cudaFreeAsync(T.counter, stream);
        return true;
    }); });
}

const char* dxb_launch_bc7(unsigned grid, unsigned residentCtas, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs,
                           const dxb_compress_params& P)
{
    // the three-subset pass (a non-default flag) lives in its own instantiations
    const bool three = (P.bcflags & DXB_BC_FLAGS_USE_3SUBSETS) != 0u;
    if (launch_bc7_tma(residentCtas, stream, hostJobs, P, three)) return "k_compress_bc7_tma";
    dxb_on_bool(three, [&](auto THREE)
    {
        smem_limit<k_compress_bc7<decltype(THREE)::value>>(kBC7Smem);
        k_compress_bc7<decltype(THREE)::value><<<grid, DXB_BC7_WARPS * 32, kBC7Smem, stream>>>(jobs, hostJobs[0], P);
    });
    return "k_compress_bc7";
}
