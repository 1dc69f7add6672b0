// dxb_k_rows.cu — row kernels (HBM-bound side of the path):
//   k_convert            generic: one thread per pixel, any implemented format pair, heterogeneous batches
//   k_convert_vec<SF,DF> hot pairs: compile-time formats, 16-byte vector access on the wider side, uniform batches
//   k_mip_level          generic: one thread per destination pixel, any format / filter
//   k_mip_tile<FMT,MODE,SRGB>  hot formats x {BOX,LINEAR,CUBIC}: compile-time format and filter, 2D thread tiles,
//                        grid.z = array item (all items of a level have the same size), no integer division
//   k_mip_sep<FMT,SRGB>  CUBIC levels of a chain: separable, each source row decoded and filtered once per tile
//   k_mip_tail<FMT,MODE,SRGB>  the levels from 64x64 down: one CTA per item
//   k_mip_box3<FMT,SRGB,LIN>  three BOX (or 2:1 LINEAR) levels per pass
// dxb_launch_mip_chain picks the kernel of every level.  The arithmetic is the same inline code in all variants
// (dxb_pixel.cuh / dxb_mips.cuh), so all of them are bit-exact against the oracle; only the memory access pattern differs.
// The launchers route on the caller's format but instantiate every specialised kernel on dxb_make_linear(format): an sRGB
// format runs its UNORM twin's kernel, with its sRGB steps taken from P.flags / P.lflags or the SRGB argument.
#include "dxb_launch.h"
#include "dxb_pixel.cuh"
#include "dxb_mips.cuh"

// ------------------------------------------------------------------------------------------------ generic
__global__ void __launch_bounds__(256) k_convert(const dxb_job* __restrict__ jobs, dxb_job single, dxb_convert_params P)
{
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t unit = blockIdx.x * blockDim.x + threadIdx.x; unit < P.totalUnits; unit += stride)
    {
        const dxb_job& j = dxb_find_job(jobs, P.njobs, single, unit);
        const uint32_t local = unit - j.firstUnit;
        const uint32_t y = local / j.width, x = local - y * j.width;
        dxb_px v = dxb_load_pixel(P.srcFormat, j.src + (size_t)y * j.srcPitch, x);
        v = dxb_convert_pixel(v, P.inF, P.outF, P.flags);
        if (P.flags & DXB_FILTER_DITHER) dxb_store_pixel_dither(P.dstFormat, j.dst + (size_t)y * j.dstPitch, x, y, v);     // ordered dither (:4861-4879)
        else dxb_store_pixel(P.dstFormat, j.dst + (size_t)y * j.dstPitch, x, v, P.threshold);
    }
}

// Error-diffusion dithering is serial over an image (dxb_convert_diffuse_image): one thread per image, images in parallel.
// errors: per job 2 * (width + 2) pixels of scratch.
__global__ void __launch_bounds__(32) k_convert_diffuse(const dxb_job* __restrict__ jobs, dxb_job single, dxb_convert_params P, dxb_px* errors, uint32_t errStride)
{
    if (threadIdx.x != 0) return;
    const dxb_job& j = (jobs == nullptr) ? single : jobs[blockIdx.x];
    dxb_px* E = errors + (size_t)blockIdx.x * errStride;
    dxb_convert_diffuse_image(P.srcFormat, P.dstFormat, P.inF, P.outF, P.flags, j.src, j.srcPitch, j.dst, j.dstPitch, j.width, j.height,
                              E, E + (j.width + 2u));
}
void dxb_launch_convert_diffuse(cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P, void* errors, uint32_t errStride)
{
    k_convert_diffuse<<<P.njobs, 32, 0, stream>>>(jobs, hostJobs[0], P, static_cast<dxb_px*>(errors), errStride);
}

__global__ void __launch_bounds__(256) k_mip_level(const dxb_mip_job* __restrict__ jobs, dxb_mip_job single, dxb_mip_params P)
{
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t unit = blockIdx.x * blockDim.x + threadIdx.x; unit < P.totalUnits; unit += stride)
    {
        const dxb_mip_job& j = dxb_find_job(jobs, P.njobs, single, unit);
        const uint32_t local = unit - j.firstUnit;
        const uint32_t y = local / j.dw, x = local - y * j.dw;
        dxb_mip_pixel(P.format, P.mode, j, x, y, P.filter, P.lflags, P.triX, P.triY);
    }
}

// ------------------------------------------------------------------------------------------------ batch predicates
// p and pitch are multiples of one vector access of `bytes` bytes (at most 16)
static bool vec_aligned(const void* p, size_t pitch, uint32_t bytes)
{
    const uint32_t v = bytes < 16u ? bytes : 16u;
    return ((uintptr_t)p % v) == 0 && (pitch % v) == 0;
}
static bool same_size(const dxb_job& a, const dxb_job& b) { return a.width == b.width && a.height == b.height; }
static bool same_size(const dxb_mip_job& a, const dxb_mip_job& b) { return a.sw == b.sw && a.sh == b.sh && a.dw == b.dw && a.dh == b.dh; }
// every job has the first one's size and there is one per gridDim.z slice: one grid covers the batch
template <typename J> static bool uniform_batch(const J* jobs, uint32_t n)
{
    if (n > 65535u) return false;
    for (uint32_t i = 1; i < n; ++i) if (!same_size(jobs[i], jobs[0])) return false;
    return true;
}

// ------------------------------------------------------------------------------------------------ vector convert
template <int BYTES> struct dxb_vec;
template <> struct dxb_vec<1> { typedef uint8_t T; };
template <> struct dxb_vec<2> { typedef uint16_t T; };
template <> struct dxb_vec<4> { typedef uint32_t T; };
template <> struct dxb_vec<8> { typedef uint2 T; };
template <> struct dxb_vec<16> { typedef uint4 T; };

template <int BYTES> __device__ __forceinline__ typename dxb_vec<BYTES>::T dxb_ld_stream(const void* p)
{
    return __ldcs(reinterpret_cast<const typename dxb_vec<BYTES>::T*>(p));
}
template <int BYTES> __device__ __forceinline__ void dxb_st_stream(void* p, typename dxb_vec<BYTES>::T v)
{
    __stcs(reinterpret_cast<typename dxb_vec<BYTES>::T*>(p), v);
}

// One thread converts PPT consecutive pixels of a row: PPT*max(bpp) == 16 bytes, so the wider side moves as one
// 128-bit access and a warp touches one contiguous 512-byte span on that side.
// grid = (ceil(chunksPerRow / (256*UNR)), rows, jobs): no integer division anywhere; a thread takes UNR chunks of its
// row spaced 256 chunks apart and issues all its vector loads before the first store.
#define DXB_CONV_UNR 4
template <uint32_t SF, uint32_t DF>
__global__ void __launch_bounds__(256) k_convert_vec(const dxb_job* __restrict__ jobs, dxb_job single, dxb_convert_params P)
{
    constexpr int SB = (int)dxb_bytes_per_pixel(SF), DB = (int)dxb_bytes_per_pixel(DF);
    constexpr int PPT = 16 / (SB > DB ? SB : DB);
    constexpr int SBY = SB * PPT, DBY = DB * PPT;
    constexpr uint32_t inF = dxb_convert_flags(SF), outF = dxb_convert_flags(DF);
    constexpr int UNR = DXB_CONV_UNR;
    const dxb_job& j = (jobs == nullptr) ? single : jobs[blockIdx.z];
    const uint32_t y = blockIdx.y;
    const uint8_t* srow = j.src + (size_t)y * j.srcPitch;
    uint8_t* drow = j.dst + (size_t)y * j.dstPitch;
    const uint32_t width = j.width;
    const uint32_t c0 = blockIdx.x * (UNR * 256u) + threadIdx.x;
    __align__(16) uint8_t sbuf[UNR][SBY];
    #pragma unroll
    for (int u = 0; u < UNR; ++u)
    {
        const uint32_t x0 = (c0 + u * 256u) * PPT;
        if (x0 + PPT <= width)
            *reinterpret_cast<typename dxb_vec<SBY>::T*>(sbuf[u]) = dxb_ld_stream<SBY>(srow + (size_t)x0 * SB);
    }
    #pragma unroll
    for (int u = 0; u < UNR; ++u)
    {
        const uint32_t x0 = (c0 + u * 256u) * PPT;
        if (x0 + PPT <= width)
        {
            __align__(16) uint8_t dbuf[DBY];
            #pragma unroll
            for (int p = 0; p < PPT; ++p)
            {
                dxb_px v = dxb_load_pixel(SF, sbuf[u], p);
                v = dxb_convert_pixel(v, inF, outF, P.flags);
                dxb_store_pixel(DF, dbuf, p, v);
            }
            dxb_st_stream<DBY>(drow + (size_t)x0 * DB, *reinterpret_cast<const typename dxb_vec<DBY>::T*>(dbuf));
        }
        else
        {
            for (uint32_t x = x0; x < width; ++x)        // ragged end of the row
            {
                dxb_px v = dxb_load_pixel(SF, srow, x);
                v = dxb_convert_pixel(v, inF, outF, P.flags);
                dxb_store_pixel(DF, drow, x, v);
            }
        }
    }
}

// (29, 28) and (28, 29) both run k_convert_vec<28, 28>: the direction of their sRGB step is in P.flags
#define DXB_CONVERT_PAIRS(X) \
    X(61, 41) X(41, 61) X(28, 2) X(2, 28) X(10, 2) X(2, 10) X(28, 10) X(10, 28) X(28, 87) X(87, 28) \
    X(61, 28) X(28, 61) X(11, 2) X(2, 11) X(41, 2) X(2, 41) X(29, 2) X(2, 29) X(29, 28) X(28, 29)

static bool convert_vec_ok(const dxb_job* hostJobs, uint32_t njobs, uint32_t SB, uint32_t DB)
{
    const uint32_t ppt = 16u / (SB > DB ? SB : DB);
    if (hostJobs[0].height > 65535u || !uniform_batch(hostJobs, njobs)) return false;
    for (uint32_t i = 0; i < njobs; ++i)
        if (!vec_aligned(hostJobs[i].src, hostJobs[i].srcPitch, SB * ppt) || !vec_aligned(hostJobs[i].dst, hostJobs[i].dstPitch, DB * ppt)) return false;
    return true;
}

void dxb_launch_convert(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P)
{
    const uint32_t SB = dxb_bytes_per_pixel(P.srcFormat), DB = dxb_bytes_per_pixel(P.dstFormat);
    if (!(P.flags & DXB_FILTER_DITHER) && convert_vec_ok(hostJobs, P.njobs, SB, DB))
    {
        const uint32_t ppt = 16u / (SB > DB ? SB : DB);
        const uint32_t chunksPerRow = (hostJobs[0].width + ppt - 1) / ppt;
        const dim3 g((chunksPerRow + 256u * DXB_CONV_UNR - 1) / (256u * DXB_CONV_UNR), hostJobs[0].height, P.njobs);
#define DXB_X(SF, DF) if (P.srcFormat == SF && P.dstFormat == DF) { \
            k_convert_vec<dxb_make_linear(SF), dxb_make_linear(DF)><<<g, 256, 0, stream>>>(jobs, hostJobs[0], P); return; }
        DXB_CONVERT_PAIRS(DXB_X)
#undef DXB_X
    }
    k_convert<<<grid, 256, 0, stream>>>(jobs, hostJobs[0], P);
}

// ------------------------------------------------------------------------------------------------ premultiplied alpha
// PremultiplyAlpha_ / PremultiplyAlphaLinear / DemultiplyAlpha / DemultiplyAlphaLinear (DirectXTexPMAlpha.cpp:30-208):
// load (linear), rgb *= a  or  (a > 0) rgb /= a, store (linear).  P.flags = resolved TEX_FILTER_SRGB_IN/OUT bits, bit 0 = reverse.
__device__ __forceinline__ dxb_px dxb_pmalpha_op(dxb_px v, bool reverse)
{
    if (!reverse) return dxb_make_px(v.x * v.w, v.y * v.w, v.z * v.w, v.w);
    if (v.w > 0.0f) return dxb_make_px(v.x / v.w, v.y / v.w, v.z / v.w, v.w);
    return dxb_make_px(v.w, v.w, v.w, v.w);       // alpha <= 0: the reference selects xyz from the un-divided splat of w (:139-146)
}
__global__ void __launch_bounds__(256) k_pmalpha(const dxb_job* __restrict__ jobs, dxb_job single, dxb_convert_params P)
{
    const uint32_t lflags = P.flags & (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT);
    const bool reverse = (P.flags & 1u) != 0u;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t unit = blockIdx.x * blockDim.x + threadIdx.x; unit < P.totalUnits; unit += stride)
    {
        const dxb_job& j = dxb_find_job(jobs, P.njobs, single, unit);
        const uint32_t local = unit - j.firstUnit;
        const uint32_t y = local / j.width, x = local - y * j.width;
        const dxb_px v = dxb_load_linear(P.srcFormat, j.src, j.srcPitch, x, y, lflags);
        dxb_store_linear(P.srcFormat, j.dst, j.dstPitch, x, y, dxb_pmalpha_op(v, reverse), lflags);
    }
}
// hot formats: compile-time format / direction / sRGB-ness, one 16-byte vector (16/bpp pixels) per thread,
// grid = (ceil(chunksPerRow / 256), rows, jobs)
template <uint32_t FMT, bool REVERSE, bool SRGB>
__global__ void __launch_bounds__(256) k_pmalpha_vec(const dxb_job* __restrict__ jobs, dxb_job single, dxb_convert_params P)
{
    constexpr int B = (int)dxb_bytes_per_pixel(FMT), PPT = 16 / B;
    constexpr uint32_t LF = SRGB ? (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT) : 0u;
    const dxb_job& j = (jobs == nullptr) ? single : jobs[blockIdx.z];
    const uint32_t y = blockIdx.y;
    const uint32_t x0 = (blockIdx.x * 256u + threadIdx.x) * PPT;
    if (x0 >= j.width) return;
    const uint8_t* srow = j.src + (size_t)y * j.srcPitch;
    uint8_t* drow = j.dst + (size_t)y * j.dstPitch;
    if (x0 + PPT <= j.width)
    {
        __align__(16) uint8_t buf[16];
        *reinterpret_cast<uint4*>(buf) = dxb_ld_stream<16>(srow + (size_t)x0 * B);
        #pragma unroll
        for (int k = 0; k < PPT; ++k)
        {
            dxb_px v = dxb_load_pixel(FMT, buf, k);
            if (LF & DXB_FILTER_SRGB_IN) v = dxb_srgb_to_linear(v);
            v = dxb_pmalpha_op(v, REVERSE);
            if (LF & DXB_FILTER_SRGB_OUT) v = dxb_linear_to_srgb(v);
            dxb_store_pixel(FMT, buf, k, v);
        }
        dxb_st_stream<16>(drow + (size_t)x0 * B, *reinterpret_cast<const uint4*>(buf));
    }
    else
        for (uint32_t x = x0; x < j.width; ++x)
            dxb_store_linear(FMT, drow, 0, x, 0, dxb_pmalpha_op(dxb_load_linear(FMT, srow, 0, x, 0, LF), REVERSE), LF);
}

void dxb_launch_pmalpha(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_convert_params& P)
{
    const uint32_t lf = P.flags & (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT);
    const bool srgb = (lf == (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT)), rev = (P.flags & 1u) != 0u;
    const uint32_t B = dxb_bytes_per_pixel(P.srcFormat);
    if ((srgb || lf == 0) && (B == 4 || B == 8 || B == 16) && convert_vec_ok(hostJobs, P.njobs, B, B))
    {
        const uint32_t ppt = 16u / B;
        const uint32_t chunksPerRow = (hostJobs[0].width + ppt - 1) / ppt;
        const dim3 g((chunksPerRow + 255u) / 256u, hostJobs[0].height, P.njobs);
#define DXB_X(FMT) if (P.srcFormat == FMT) { \
            if (rev && srgb) k_pmalpha_vec<dxb_make_linear(FMT), true, true><<<g, 256, 0, stream>>>(jobs, hostJobs[0], P); \
            else if (rev) k_pmalpha_vec<dxb_make_linear(FMT), true, false><<<g, 256, 0, stream>>>(jobs, hostJobs[0], P); \
            else if (srgb) k_pmalpha_vec<dxb_make_linear(FMT), false, true><<<g, 256, 0, stream>>>(jobs, hostJobs[0], P); \
            else k_pmalpha_vec<dxb_make_linear(FMT), false, false><<<g, 256, 0, stream>>>(jobs, hostJobs[0], P); \
            return; }
        DXB_X(28) DXB_X(29) DXB_X(87) DXB_X(91) DXB_X(10) DXB_X(2)
#undef DXB_X
    }
    k_pmalpha<<<grid, 256, 0, stream>>>(jobs, hostJobs[0], P);
}

// ------------------------------------------------------------------------------------------------ alpha coverage
// k_alpha_coverage: one thread per 2x2 cell of one image, integer count accumulated with one atomicAdd per warp.
__global__ void __launch_bounds__(256) k_alpha_coverage(dxb_job j, uint32_t fmt, float scale, float ref, unsigned long long* count)
{
    const uint32_t cw = j.width - 1u, ch = j.height - 1u;
    const uint32_t cells = cw * ch;
    uint32_t local = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += gridDim.x * blockDim.x)
    {
        const uint32_t y = i / cw, x = i - y * cw;
        const uint8_t* r0 = j.src + (size_t)y * j.srcPitch;
        const uint8_t* r1 = r0 + j.srcPitch;
        local += dxb_alpha_coverage_cell(dxb_load_pixel(fmt, r0, x).w, dxb_load_pixel(fmt, r1, x).w,
                                         dxb_load_pixel(fmt, r0, x + 1u).w, dxb_load_pixel(fmt, r1, x + 1u).w, scale, ref);
    }
    local = __reduce_add_sync(0xffffffffu, local);
    if ((threadIdx.x & 31u) == 0 && local) atomicAdd(count, (unsigned long long)local);
}
__global__ void __launch_bounds__(256) k_scale_alpha(dxb_job j, uint32_t fmt, float scale)
{
    const uint32_t n = j.width * j.height;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const uint32_t y = i / j.width, x = i - y * j.width;
        dxb_scale_alpha_pixel(fmt, j.src + (size_t)y * j.srcPitch, j.dst + (size_t)y * j.dstPitch, x, scale);
    }
}
void dxb_launch_alpha_coverage(unsigned grid, cudaStream_t stream, const dxb_job& j, uint32_t fmt, float scale, float ref, unsigned long long* count)
{
    k_alpha_coverage<<<grid, 256, 0, stream>>>(j, fmt, scale, ref, count);
}
void dxb_launch_scale_alpha(unsigned grid, cudaStream_t stream, const dxb_job& j, uint32_t fmt, float scale)
{
    k_scale_alpha<<<grid, 256, 0, stream>>>(j, fmt, scale);
}

// ------------------------------------------------------------------------------------------------ tiled mips
// The sRGB <-> linear steps are a COMPILE-TIME property of the specialised kernels (SRGB = both SRGB_IN and SRGB_OUT,
// the only combination a mip chain produces; anything else takes the generic kernel): with a run-time flag every
// instantiation carried the inlined powf code (26.5 k SASS instructions for the fused BOX kernel) and stalled on
// instruction fetch.
#define DXB_LF(SRGB) ((SRGB) ? (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT) : 0u)

#define DXB_CUBIC_KY 4u       // output rows per thread of the CUBIC tile kernel
// grid = (ceil(dw/32), ceil(dh/8), items) (CUBIC: ceil(dh / (8 * DXB_CUBIC_KY))); jobs[z] describes item z (all items share the level's size).
template <uint32_t FMT, uint32_t MODE, bool SRGB>
__global__ void __launch_bounds__(256) k_mip_tile(const dxb_mip_job* __restrict__ jobs, dxb_mip_job single, dxb_mip_params P)
{
    const dxb_mip_job& j = (jobs == nullptr) ? single : jobs[blockIdx.z];
    constexpr uint32_t LF = DXB_LF(SRGB);
    if (MODE == DXB_FILTER_CUBIC)
    {
        // A thread produces DXB_CUBIC_KY vertically adjacent pixels of one column.  The horizontal interpolation of a
        // source row (a function of the row and the column only) is kept from one output to the next: for the 2:1
        // step of a mip chain two of the four rows are reused, so 10 instead of 16 row interpolations per 4 outputs.
        // Same operations on the same operands as dxb_mip_cubic => bit-identical.
        const uint32_t x = blockIdx.x * 32u + threadIdx.x;
        const uint32_t y0 = (blockIdx.y * 8u + threadIdx.y) * DXB_CUBIC_KY;
        if (x >= j.dw || y0 >= j.dh) return;
        const dxb_cub tx = dxb_cubic_entry(j.sw, j.dw, (P.filter & DXB_FILTER_WRAP_U) != 0, (P.filter & DXB_FILTER_MIRROR_U) != 0, x);
        uint32_t crow[4] = { 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu };
        dxb_px cval[4];
        for (int c = 0; c < 4; ++c) cval[c] = dxb_make_px(0.0f, 0.0f, 0.0f, 0.0f);
        #pragma unroll
        for (uint32_t k = 0; k < DXB_CUBIC_KY; ++k)
        {
            const uint32_t y = y0 + k;
            if (y >= j.dh) break;
            const dxb_cub ty = dxb_cubic_entry(j.sh, j.dh, (P.filter & DXB_FILTER_WRAP_V) != 0, (P.filter & DXB_FILTER_MIRROR_V) != 0, y);
            const uint32_t rows[4] = { ty.u0, ty.u1, ty.u2, ty.u3 };
            dxb_px C[4];
            #pragma unroll
            for (int r = 0; r < 4; ++r)
            {
                bool found = false;
                dxb_px hit = cval[0];
                #pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (crow[c] == rows[r]) { found = true; hit = cval[c]; }
                if (!found)
                {
                    const dxb_px q0 = dxb_load_linear(FMT, j.src, j.srcPitch, tx.u0, rows[r], LF);
                    const dxb_px q1 = dxb_load_linear(FMT, j.src, j.srcPitch, tx.u1, rows[r], LF);
                    const dxb_px q2 = dxb_load_linear(FMT, j.src, j.srcPitch, tx.u2, rows[r], LF);
                    const dxb_px q3 = dxb_load_linear(FMT, j.src, j.srcPitch, tx.u3, rows[r], LF);
                    hit = dxb_cubic4(tx.x, q0, q1, q2, q3);
                }
                C[r] = hit;
            }
            #pragma unroll
            for (int c = 0; c < 4; ++c) { crow[c] = rows[c]; cval[c] = C[c]; }
            dxb_store_linear(FMT, j.dst, j.dstPitch, x, y, dxb_cubic4(ty.x, C[0], C[1], C[2], C[3]), LF);
        }
        return;
    }
    const uint32_t x = blockIdx.x * 32u + threadIdx.x, y = blockIdx.y * 8u + threadIdx.y;
    if (x >= j.dw || y >= j.dh) return;
    if (MODE != DXB_FILTER_BOX) { dxb_mip_pixel(FMT, MODE, j, x, y, P.filter, LF, P.triX, P.triY); return; }
    // BOX: the vector and the scalar path share one store (a second copy of the inlined sRGB store costs ~260 instructions).
    // Alignment is decided per item (uniform within the CTA: blockIdx.z selects the item).
    constexpr int B = (int)dxb_bytes_per_pixel(FMT);
    dxb_px v;
    constexpr uintptr_t VA = (B * 2 <= 16) ? B * 2 : 16;
    if ((((uintptr_t)j.src % VA) == 0) && ((j.srcPitch % VA) == 0) && j.sw > 1 && j.sh > 1)
    {
        // two horizontally adjacent source pixels per row in one vector load: ((p00 + p10) + p01) + p11) * 0.25
        constexpr int VB = (B * 2 <= 16) ? B * 2 : 16;
        __align__(16) uint8_t r0[B * 2], r1[B * 2];
        const uint8_t* s0 = j.src + (size_t)(2u * y) * j.srcPitch + (size_t)(2u * x) * B;
        #pragma unroll
        for (int k = 0; k < B * 2; k += VB)
        {
            *reinterpret_cast<typename dxb_vec<VB>::T*>(r0 + k) = __ldg(reinterpret_cast<const typename dxb_vec<VB>::T*>(s0 + k));
            *reinterpret_cast<typename dxb_vec<VB>::T*>(r1 + k) = __ldg(reinterpret_cast<const typename dxb_vec<VB>::T*>(s0 + j.srcPitch + k));
        }
        dxb_px p00 = dxb_load_pixel(FMT, r0, 0), p01 = dxb_load_pixel(FMT, r0, 1);
        dxb_px p10 = dxb_load_pixel(FMT, r1, 0), p11 = dxb_load_pixel(FMT, r1, 1);
        if (LF & DXB_FILTER_SRGB_IN) { p00 = dxb_srgb_to_linear(p00); p01 = dxb_srgb_to_linear(p01); p10 = dxb_srgb_to_linear(p10); p11 = dxb_srgb_to_linear(p11); }
        v = dxb_px_add(p00, p10);
        v = dxb_px_add(v, p01);
        v = dxb_px_add(v, p11);
        v = dxb_px_scale(v, 0.25f);
    }
    else v = dxb_mip_box(FMT, j, x, y, LF);
    dxb_store_linear(FMT, j.dst, j.dstPitch, x, y, v, LF);
}


template <int N> __device__ __forceinline__ void dxb_copy_vec(uint8_t* dst, const uint8_t* src, bool streamLoad)
{
    constexpr int V = (N >= 16) ? 16 : N;
    #pragma unroll
    for (int k = 0; k < N; k += V)
    {
        typedef typename dxb_vec<V>::T T;
        if (streamLoad) *reinterpret_cast<T*>(dst + k) = __ldcs(reinterpret_cast<const T*>(src + k));
        else *reinterpret_cast<T*>(dst + k) = *reinterpret_cast<const T*>(src + k);
    }
}

// ------------------------------------------------------------------------------------------------ separable CUBIC
// One CTA (8 warps) = a 32 x 16 tile of destination pixels.  The reference filters every source row horizontally and then
// combines 4 of those rows vertically (DirectXTexMipmaps.cpp:1204-1388); k_mip_tile redoes the horizontal pass for every
// destination pixel and decodes ~10 source pixels per output.  Here
//   stage A  a warp takes one source row of the tile at a time: its lanes decode the row's pixels ONCE into the warp's
//            shared row buffer (load + format decode + sRGB linearisation),
//   stage B  lane x filters that row horizontally for destination column x (same operands, same operation order as
//            dxb_mip_cubic) into the shared H[row][x],
//   stage C  after one barrier every thread combines the H rows of its two destination pixels vertically and stores them.
// Per destination pixel of a 2:1 level that is 4.4 pixel decodes, 2.1 horizontal and 1 vertical filter evaluations instead
// of 10 / 2.5 / 1.  Source coordinates are kept UNBOUNDED inside the tile (consecutive slots of the row buffer / of H) and
// bounded (clamp / wrap / mirror, filters.h:123-207) only when the pixel is fetched, so every addressing mode of
// the reference takes the same path.  Requires source extent <= 3 x destination extent (every level of a mip chain) and
// every source and destination extent <= DXB_SEP_MAX_EXTENT.
#define DXB_SEP_TW 32
#define DXB_SEP_TH 16
#define DXB_SEP_MAXC (DXB_SEP_TW * 3 + 4)
#define DXB_SEP_MAXR (DXB_SEP_TH * 3 + 4)
// Largest extent k_mip_sep takes.  Its fp32 coordinates srcB = (u + 0.5) * (source / dest) - 0.5 round three times, each within
// 2^-24 of a value below the source extent, so below 2^22 srcB is within 0.75 of the exact value.  That keeps (a) the tap base
// inside [0, source - 1], which dxb_cubic_entry clamps before it derives the fraction and dxb_sep_entry does not, and (b) the base
// span of one tile within 3 (TW - 1) + 2 columns (3 (TH - 1) + 2 rows), so it fits rowbuf / H.  Both fail at larger extents:
// a same-size CUBIC of 12 582 912 pixels rounds the last base to the width; 537 157 722 -> 179 052 574 needs 132 columns in a
// tile.  tests/test_cpu_mip_routes.py runs the same statements at this bound.
#define DXB_SEP_MAX_EXTENT (1u << 22)

// unbounded tap base and fraction of destination coordinate u: taps base - 1 .. base + 2.  dxb_cubic_entry bounds the base tap
// before it derives the fraction; this does not: the two agree because the base stays inside [0, source - 1] up to DXB_SEP_MAX_EXTENT.
__device__ __forceinline__ void dxb_sep_entry(uint32_t source, uint32_t dest, uint32_t u, int32_t* base, float* w)
{
    const float scale = (float)source / (float)dest;
    const float t = ((float)u + 0.5f) * scale;
    const float srcB = t - 0.5f;
    const int64_t isrcB = (int64_t)srcB;
    *w = srcB - (float)isrcB; *base = (int32_t)isrcB;
}
__device__ __forceinline__ uint32_t dxb_sep_bound(int32_t i, uint32_t source, bool wrap, bool mirror)
{
    return (uint32_t)dxb_bounduvw((int64_t)i, (int64_t)source - 1, wrap, mirror);
}

template <uint32_t FMT, bool SRGB>
__global__ void __launch_bounds__(256) k_mip_sep(const dxb_mip_job* __restrict__ jobs, dxb_mip_job single, dxb_mip_params P)
{
    constexpr uint32_t LF = DXB_LF(SRGB);
    const dxb_mip_job& j = (jobs == nullptr) ? single : jobs[blockIdx.z];
    __shared__ float4 H[DXB_SEP_MAXR][DXB_SEP_TW];
    __shared__ float4 rowbuf[8][DXB_SEP_MAXC];
    __shared__ int32_t colBase[DXB_SEP_TW], rowBase[DXB_SEP_TH];
    __shared__ float colW[DXB_SEP_TW], rowW[DXB_SEP_TH];
    const uint32_t tid = threadIdx.y * 32u + threadIdx.x, warp = threadIdx.y, lane = threadIdx.x;
    const uint32_t ox = blockIdx.x * DXB_SEP_TW, oy = blockIdx.y * DXB_SEP_TH;
    const uint32_t tw = min((uint32_t)DXB_SEP_TW, j.dw - ox), th = min((uint32_t)DXB_SEP_TH, j.dh - oy);
    if (tid < DXB_SEP_TW) { int32_t b; float w; dxb_sep_entry(j.sw, j.dw, ox + min(tid, tw - 1u), &b, &w); colBase[tid] = b; colW[tid] = w; }
    else if (tid < DXB_SEP_TW + DXB_SEP_TH) { const uint32_t r = tid - DXB_SEP_TW; int32_t b; float w; dxb_sep_entry(j.sh, j.dh, oy + min(r, th - 1u), &b, &w); rowBase[r] = b; rowW[r] = w; }
    __syncthreads();
    const bool wrapU = (P.filter & DXB_FILTER_WRAP_U) != 0, mirU = (P.filter & DXB_FILTER_MIRROR_U) != 0;
    const bool wrapV = (P.filter & DXB_FILTER_WRAP_V) != 0, mirV = (P.filter & DXB_FILTER_MIRROR_V) != 0;
    const int32_t c0 = colBase[0] - 1, ncols = colBase[tw - 1u] + 2 - c0 + 1;
    const int32_t r0 = rowBase[0] - 1, nrows = rowBase[th - 1u] + 2 - r0 + 1;
    const int32_t myc = colBase[lane] - 1 - c0;
    const float myw = colW[lane];
    // the bounded source column of every row-buffer slot this lane fills is the same for all rows: computed once
    constexpr int SPL = (DXB_SEP_MAXC + 31) / 32;
    uint32_t mycol[SPL];
    #pragma unroll
    for (int k = 0; k < SPL; ++k) mycol[k] = dxb_sep_bound(c0 + (int32_t)lane + 32 * k, j.sw, wrapU, mirU);
    // software pipeline: the raw pixels of this warp's NEXT source row are in flight while the current row is decoded and filtered
    constexpr int B = (int)dxb_bytes_per_pixel(FMT);
    __align__(16) uint8_t raw[SPL][B];
    auto fetch = [&](int32_t r)
    {
        const uint8_t* srow = j.src + (size_t)dxb_sep_bound(r0 + r, j.sh, wrapV, mirV) * j.srcPitch;
        #pragma unroll
        for (int k = 0; k < SPL; ++k)
            if ((int32_t)lane + 32 * k < ncols) dxb_copy_vec<B>(raw[k], srow + (size_t)mycol[k] * B, false);
    };
    if ((int32_t)warp < nrows) fetch((int32_t)warp);
    for (int32_t r = (int32_t)warp; r < nrows; r += 8)
    {
        #pragma unroll
        for (int k = 0; k < SPL; ++k)
            if ((int32_t)lane + 32 * k < ncols)
            {
                dxb_px v = dxb_load_pixel(FMT, raw[k], 0);
                if (LF & DXB_FILTER_SRGB_IN) v = dxb_srgb_to_linear(v);
                rowbuf[warp][lane + 32 * k] = make_float4(v.x, v.y, v.z, v.w);
            }
        if (r + 8 < nrows) fetch(r + 8);
        __syncwarp();
        if (lane < tw)
        {
            dxb_px q[4];
            #pragma unroll
            for (int k = 0; k < 4; ++k) { const float4 f = rowbuf[warp][myc + k]; q[k] = dxb_make_px(f.x, f.y, f.z, f.w); }
            const dxb_px h = dxb_cubic4(myw, q[0], q[1], q[2], q[3]);
            H[r][lane] = make_float4(h.x, h.y, h.z, h.w);
        }
        __syncwarp();
    }
    __syncthreads();
    if (lane >= tw) return;
    #pragma unroll
    for (uint32_t k = 0; k < DXB_SEP_TH / 8; ++k)
    {
        const uint32_t y = warp + 8u * k;
        if (y >= th) break;
        const int32_t rr = rowBase[y] - 1 - r0;
        const float wy = rowW[y];
        dxb_px c[4];
        #pragma unroll
        for (int t = 0; t < 4; ++t) { const float4 f = H[rr + t][lane]; c[t] = dxb_make_px(f.x, f.y, f.z, f.w); }
        dxb_store_linear(FMT, j.dst, j.dstPitch, ox + lane, oy + y, dxb_cubic4(wy, c[0], c[1], c[2], c[3]), LF);
    }
}

// Tail of the chain: one CTA per item computes levels [first, first+count) back to back (each level reads the
// previous one from global memory after a block barrier), replacing `count` tiny launches by one.
// jobs is laid out [level][item]: jobs[l * items + item].
template <uint32_t FMT, uint32_t MODE, bool SRGB>
__global__ void __launch_bounds__(256) k_mip_tail(const dxb_mip_job* __restrict__ jobs, uint32_t items, uint32_t count, dxb_mip_params P)
{
    for (uint32_t l = 0; l < count; ++l)
    {
        const dxb_mip_job& j = jobs[(size_t)l * items + blockIdx.x];
        const uint32_t n = j.dw * j.dh;
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
        {
            const uint32_t y = i / j.dw, x = i - y * j.dw;
            dxb_mip_pixel(FMT, MODE, j, x, y, P.filter, DXB_LF(SRGB), P.triX, P.triY);
        }
        __threadfence_block();
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ fused BOX levels
// Three consecutive BOX levels in one pass: a thread owns an 8x8 source patch, writes the 4x4 / 2x2 / 1 destination
// pixels of levels l, l+1, l+2.  Each level is computed from the STORED representation of the previous one (pixels are
// encoded to the format and decoded again in registers), exactly what three separate launches read back from memory,
// so the result is bit-identical; the source is read once and the two intermediate levels are never re-read from HBM
// (5.6 instead of 7.0 bytes moved per source texel-chain, one launch instead of three).
// jobs: [level][item] records of the three levels; requires source width/height multiples of 8 and vector alignment.
// LIN: the LINEAR filter at an exact 2:1 ratio.  CreateLinearFilter (filters.h:64-104) gives destination u the taps 2u and 2u + 1 with
// weights 0.5 / 0.5 (srcB = 2u + 1.5, no edge clamp, WRAP irrelevant) while the source extent is at most 2^23: above it the fp32
// srcB loses its .5 (width 8388616: u = 4194304 gives 8388610, one tap at weight 1) and launch_box3 declines LIN.  So a destination pixel reads the same 2x2 patch as BOX and only the
// arithmetic differs: ((a0 w + a1 w) w) + ((b0 w + b1 w) w) in the reference's operation order (dxb_mip_linear, DirectXTexMipmaps.cpp:1087-1197).
template <uint32_t FMT, bool LIN>
__device__ __forceinline__ dxb_px dxb_box4(const uint8_t* r0, const uint8_t* r1, int k, uint32_t lflags)
{
    dxb_px p00 = dxb_load_pixel(FMT, r0, 2 * k), p01 = dxb_load_pixel(FMT, r0, 2 * k + 1);
    dxb_px p10 = dxb_load_pixel(FMT, r1, 2 * k), p11 = dxb_load_pixel(FMT, r1, 2 * k + 1);
    if (lflags & DXB_FILTER_SRGB_IN) { p00 = dxb_srgb_to_linear(p00); p01 = dxb_srgb_to_linear(p01); p10 = dxb_srgb_to_linear(p10); p11 = dxb_srgb_to_linear(p11); }
    dxb_px v;
    if (LIN)
    {
        const dxb_px r0v = dxb_px_scale(dxb_px_add(dxb_px_scale(p00, 0.5f), dxb_px_scale(p01, 0.5f)), 0.5f);
        const dxb_px r1v = dxb_px_scale(dxb_px_add(dxb_px_scale(p10, 0.5f), dxb_px_scale(p11, 0.5f)), 0.5f);
        v = dxb_px_add(r0v, r1v);
    }
    else
    {
        v = dxb_px_add(p00, p10);
        v = dxb_px_add(v, p01);
        v = dxb_px_add(v, p11);
        v = dxb_px_scale(v, 0.25f);
    }
    if (lflags & DXB_FILTER_SRGB_OUT) v = dxb_linear_to_srgb(v);
    return v;
}
template <uint32_t FMT, bool SRGB, bool LIN>
__global__ void __launch_bounds__(256) k_mip_box3(const dxb_mip_job* __restrict__ jobs, uint32_t items, dxb_mip_params P)
{
    constexpr int B = (int)dxb_bytes_per_pixel(FMT);
    const uint32_t item = blockIdx.z;
    const dxb_mip_job& jA = jobs[item];
    const dxb_mip_job& jB = jobs[(size_t)items + item];
    const dxb_mip_job& jC = jobs[2 * (size_t)items + item];
    const uint32_t tx = blockIdx.x * 32u + threadIdx.x, ty = blockIdx.y * 8u + threadIdx.y;
    if (tx >= jC.dw || ty >= jC.dh) return;
    // all source rows of a group are loaded before the first store of that group (bytes in flight per thread =
    // PRE rows x 8 pixels; 8 rows for <= 4-byte pixels, 4 for 8-byte, 2 for 16-byte keeps it at <= 64 registers)
    constexpr int PRE = (B <= 4) ? 8 : (B == 8 ? 4 : 2);
    const uint8_t* sbase = jA.src + (size_t)(8u * ty) * jA.srcPitch + (size_t)(8u * tx) * B;
    __align__(16) uint8_t rowB[2][2 * B];
    __align__(16) uint8_t rowA[2][4 * B];
    #pragma unroll
    for (int grp = 0; grp < 8 / PRE; ++grp)
    {
        __align__(16) uint8_t s[PRE][8 * B];
        #pragma unroll
        for (int k = 0; k < PRE; ++k) dxb_copy_vec<8 * B>(s[k], sbase + (size_t)(grp * PRE + k) * jA.srcPitch, true);
        #pragma unroll
        for (int pr = 0; pr < PRE / 2; ++pr)
        {
            const int arow = grp * (PRE / 2) + pr;                   // level-A row 0..3 of this thread
            #pragma unroll
            for (int k = 0; k < 4; ++k) dxb_store_pixel(FMT, rowA[arow & 1], k, dxb_box4<FMT, LIN>(s[2 * pr], s[2 * pr + 1], k, DXB_LF(SRGB)));
            dxb_copy_vec<4 * B>(jA.dst + (size_t)(4u * ty + arow) * jA.dstPitch + (size_t)(4u * tx) * B, rowA[arow & 1], false);
            if (arow & 1)
            {
                const int half = arow >> 1;
                #pragma unroll
                for (int k = 0; k < 2; ++k) dxb_store_pixel(FMT, rowB[half], k, dxb_box4<FMT, LIN>(rowA[0], rowA[1], k, DXB_LF(SRGB)));
                dxb_copy_vec<2 * B>(jB.dst + (size_t)(2u * ty + half) * jB.dstPitch + (size_t)(2u * tx) * B, rowB[half], false);
            }
        }
    }
    __align__(16) uint8_t pc[B];
    dxb_store_pixel(FMT, pc, 0, dxb_box4<FMT, LIN>(rowB[0], rowB[1], 0, DXB_LF(SRGB)));
    dxb_copy_vec<B>(jC.dst + (size_t)ty * jC.dstPitch + (size_t)tx * B, pc, false);
}

// ------------------------------------------------------------------------------------------------ chain launcher
#define DXB_MIP_FORMATS(X, MODE) X(28, MODE) X(29, MODE) X(10, MODE) X(2, MODE) X(61, MODE) X(41, MODE) X(87, MODE)

// hj: [3][items] records of levels l, l+1, l+2.  Returns false when the fused kernel does not apply (nothing launched).
static bool launch_box3(cudaStream_t stream, const dxb_mip_job* jobs, const dxb_mip_job* hj, uint32_t items, const dxb_mip_params& P, bool srgb)
{
    const uint32_t B = dxb_bytes_per_pixel(P.format);
    const dxb_mip_job& a0 = hj[0];
    if ((a0.sw & 7u) || (a0.sh & 7u) || a0.sw < 8u || a0.sh < 8u || !uniform_batch(hj, items)) return false;
    for (uint32_t i = 0; i < items; ++i)
    {
        const dxb_mip_job& a = hj[i]; const dxb_mip_job& b = hj[items + i]; const dxb_mip_job& c = hj[2 * (size_t)items + i];
        if (a.dw != a.sw / 2 || a.dh != a.sh / 2 || b.dw != a.sw / 4 || b.dh != a.sh / 4 || c.dw != a.sw / 8 || c.dh != a.sh / 8) return false;
        if (b.src != a.dst || c.src != b.dst || b.srcPitch != a.dstPitch || c.srcPitch != b.dstPitch) return false;
        if (!vec_aligned(a.src, a.srcPitch, 8 * B) || !vec_aligned(a.dst, a.dstPitch, 4 * B) || !vec_aligned(b.dst, b.dstPitch, 2 * B) ||
            !vec_aligned(c.dst, c.dstPitch, B)) return false;
    }
    const bool lin = (P.mode == DXB_FILTER_LINEAR);
    if (lin && (a0.sw > (1u << 23) || a0.sh > (1u << 23))) return false;        // CreateLinearFilter is 2u, 2u + 1 at 0.5 only up to 2^23
    const dim3 blk(32, 8, 1);
    const dim3 g((a0.sw / 8 + 31) / 32, (a0.sh / 8 + 7) / 8, items);
    if (g.y > 65535u) return false;
#define DXB_X(FMT, MODE) if (P.format == FMT) { \
        if (lin) { if (srgb) k_mip_box3<dxb_make_linear(FMT), true, true><<<g, blk, 0, stream>>>(jobs, items, P); \
                   else k_mip_box3<dxb_make_linear(FMT), false, true><<<g, blk, 0, stream>>>(jobs, items, P); } \
        else { if (srgb) k_mip_box3<dxb_make_linear(FMT), true, false><<<g, blk, 0, stream>>>(jobs, items, P); \
               else k_mip_box3<dxb_make_linear(FMT), false, false><<<g, blk, 0, stream>>>(jobs, items, P); } \
        return true; }
    DXB_MIP_FORMATS(DXB_X, 0)
#undef DXB_X
    return false;
}

// levels l .. l + count - 1 of every item in one launch; jobs: their [level][item] records
static void launch_tail(cudaStream_t stream, const dxb_mip_job* jobs, uint32_t items, uint32_t count, const dxb_mip_params& P, bool srgb)
{
#define DXB_X(FMT, MODE) if (P.format == FMT && P.mode == MODE) { \
        if (srgb) k_mip_tail<dxb_make_linear(FMT), MODE, true><<<items, 256, 0, stream>>>(jobs, items, count, P); \
        else k_mip_tail<dxb_make_linear(FMT), MODE, false><<<items, 256, 0, stream>>>(jobs, items, count, P); \
        return; }
    DXB_MIP_FORMATS(DXB_X, DXB_FILTER_BOX)
    DXB_MIP_FORMATS(DXB_X, DXB_FILTER_LINEAR)
    DXB_MIP_FORMATS(DXB_X, DXB_FILTER_CUBIC)
#undef DXB_X
}

// one level: hj = its records, jobs = their device copy (nullptr for a single item).  Returns the launched kernel's name.
static const char* launch_level(cudaStream_t stream, const dxb_mip_job* jobs, const dxb_mip_job* hj, const dxb_mip_params& P, bool special, bool srgb,
                                unsigned gridCap)
{
    const dxb_mip_job& j0 = hj[0];
    if (special && uniform_batch(hj, P.njobs))
    {
        const dim3 blk(32, 8, 1);
        // CUBIC of a chain level (source <= 3 x destination per axis): separable shared-memory kernel
        // (LINEAR at 2:1 has no tap shared between neighbouring outputs: the plain tile kernel is faster there, 0.24 vs 0.43 ms per 64 x 1024^2 chain)
        bool pixAligned = true;                     // k_mip_sep fetches whole pixels with one vector load each
        for (uint32_t i = 0; i < P.njobs; ++i) pixAligned = pixAligned && vec_aligned(hj[i].src, hj[i].srcPitch, dxb_bytes_per_pixel(P.format));
        const dim3 gs((j0.dw + DXB_SEP_TW - 1) / DXB_SEP_TW, (j0.dh + DXB_SEP_TH - 1) / DXB_SEP_TH, P.njobs);
        const bool sepExtent = j0.sw <= DXB_SEP_MAX_EXTENT && j0.dw <= DXB_SEP_MAX_EXTENT && j0.sh <= DXB_SEP_MAX_EXTENT && j0.dh <= DXB_SEP_MAX_EXTENT;
        if (P.mode == DXB_FILTER_CUBIC && pixAligned && sepExtent && j0.sw <= 3u * j0.dw && j0.sh <= 3u * j0.dh && gs.y <= 65535u)
        {
#define DXB_X(FMT, MODE) if (P.format == FMT) { \
                if (srgb) k_mip_sep<dxb_make_linear(FMT), true><<<gs, blk, 0, stream>>>(jobs, j0, P); \
                else k_mip_sep<dxb_make_linear(FMT), false><<<gs, blk, 0, stream>>>(jobs, j0, P); \
                return "k_mip_sep"; }
            DXB_MIP_FORMATS(DXB_X, 0)
#undef DXB_X
        }
        const uint32_t rowsPerCta = (P.mode == DXB_FILTER_CUBIC) ? 8u * DXB_CUBIC_KY : 8u;
        const dim3 g((j0.dw + 31) / 32, (j0.dh + rowsPerCta - 1) / rowsPerCta, P.njobs);
        if (g.y <= 65535u)
        {
#define DXB_X(FMT, MODE) if (P.format == FMT && P.mode == MODE) { \
                if (srgb) k_mip_tile<dxb_make_linear(FMT), MODE, true><<<g, blk, 0, stream>>>(jobs, j0, P); \
                else k_mip_tile<dxb_make_linear(FMT), MODE, false><<<g, blk, 0, stream>>>(jobs, j0, P); \
                return "k_mip_tile"; }
            DXB_MIP_FORMATS(DXB_X, DXB_FILTER_BOX)
            DXB_MIP_FORMATS(DXB_X, DXB_FILTER_LINEAR)
            DXB_MIP_FORMATS(DXB_X, DXB_FILTER_CUBIC)
#undef DXB_X
        }
    }
    const uint32_t need = (uint32_t)(((uint64_t)P.totalUnits + 255) / 256);
    k_mip_level<<<need < 1u ? 1u : (need < gridCap ? need : gridCap), 256, 0, stream>>>(jobs, j0, P);
    return "k_mip_level";
}

int32_t dxb_launch_mip_chain(cudaStream_t stream, const dxb_mip_job* jobs, const dxb_mip_job* hostJobs, uint32_t items, uint32_t levels,
                             dxb_mip_params P, const dxb_tri_axis* tri, unsigned gridCap, bool genericOnly,
                             int32_t (*launched)(const char* kernel))
{
    // The specialised kernels take BOX / LINEAR / CUBIC on the hot formats with both sRGB steps or none (the only combinations
    // a chain produces); anything else runs the generic k_mip_level.
    const bool srgb = (P.lflags == (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT));
    bool special = false;
#define DXB_X(FMT, MODE) special = special || P.format == FMT;
    DXB_MIP_FORMATS(DXB_X, 0)
#undef DXB_X
    special = special && !genericOnly && (srgb || P.lflags == 0) &&
              (P.mode == DXB_FILTER_BOX || P.mode == DXB_FILTER_LINEAR || P.mode == DXB_FILTER_CUBIC);
    // first level whose SOURCE is at most 64x64: from there on one CTA per item finishes the chain in one launch
    uint32_t tailStart = levels;
    for (uint32_t l = 1; l < levels; ++l)
        if (hostJobs[(size_t)(l - 1) * items].sw <= 64 && hostJobs[(size_t)(l - 1) * items].sh <= 64) { tailStart = l; break; }
    const bool tail = special && levels - tailStart >= 2 && items <= 0x7FFFFFFFu;
    const bool fused = special && P.mode != DXB_FILTER_CUBIC && levels >= 4;       // LINEAR at 2:1 reads the same 2x2 patches as BOX
    P.njobs = items;
    for (uint32_t l = 1; l < levels;)
    {
        const size_t at = (size_t)(l - 1) * items;
        const dxb_mip_job* hj = hostJobs + at;
        int32_t hr;
        // three levels per launch while the source is larger than the tail kernel's 64x64 and divides by 8
        if (fused && l + 2 < levels && (hj[0].sw > 64 || hj[0].sh > 64) && launch_box3(stream, jobs + at, hj, items, P, srgb))
        {
            hr = launched("k_mip_box3");
            l += 3;
        }
        else if (tail && l >= tailStart)
        {
            launch_tail(stream, jobs + at, items, levels - l, P, srgb);
            return launched("k_mip_tail");
        }
        else
        {
            const dxb_mip_job& last = hj[items - 1];
            P.totalUnits = last.firstUnit + last.dw * last.dh;
            if (tri) { P.triX = tri[2 * (l - 1)]; P.triY = tri[2 * (l - 1) + 1]; }
            hr = launched(launch_level(stream, items > 1 ? jobs + at : nullptr, hj, P, special, srgb, gridCap));
            l += 1;
        }
        if (hr != DXB_S_OK) return hr;
    }
    return DXB_S_OK;
}

