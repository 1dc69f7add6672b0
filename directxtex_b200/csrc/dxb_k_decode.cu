// dxb_k_decode.cu — DecompressBC (DirectXTexCompress.cpp:425-535) for a batch of images: one THREAD per 4x4 block:
// decode (dxb_decode.cuh) -> ConvertScanline -> StoreScanline.
//   k_decompress            generic: any BC source, any implemented target format
//   k_decompress_t<SF,DF>   the default (source, target) pairs with no sRGB step: compile-time formats (one decoder, one
//                           store path per kernel) and one vector store per block row.  No pair names an sRGB format:
//                           an sRGB call matches its twins' pair (dxb_make_linear).
#include "dxb_launch.h"
#include "dxb_decode.cuh"

// ---- table-driven fast paths -------------------------------------------------------------------------------------------
// BC1 / BC3 / BC4 / BC5 blocks hold at most 4 colours and 8 values per channel; ConvertScanline + StoreScanline of the default target
// formats (same class, no flags) map every channel of a pixel independently, so a block's distinct values go through them ONCE (4 or
// 8 conversions instead of 16 x channels) and the 16 pixels pick their bytes by index.  Same bytes as the per-pixel path (the GPU
// parity tests compare both with the reference decoder); ~250 instead of ~1200 instructions per BC1 block, which moves the
// kernel from issue-bound to the memory system.
template <uint32_t SF, uint32_t DF>
__device__ __forceinline__ uint32_t dec_bytes(const dxb_px v)          // one pixel -> its stored bytes (up to 4, little endian)
{
    __align__(4) uint8_t b[4] = { 0, 0, 0, 0 };
    dxb_store_pixel(DF, b, 0, dxb_convert_pixel(v, dxb_convert_flags(SF), dxb_convert_flags(DF), 0u));
    return *reinterpret_cast<const uint32_t*>(b);
}
// eight values -> eight stored bytes (byte k = value k); the value sits in channel x of an (x, 0, 0, 1) pixel
template <uint32_t SF, uint32_t DF>
__device__ __forceinline__ uint64_t dec_table8(const float* t)
{
    uint64_t tab = 0;
    #pragma unroll
    for (int k = 0; k < 8; ++k) tab |= (uint64_t)(dec_bytes<SF, DF>(dxb_make_px(t[k], 0.0f, 0.0f, 1.0f)) & 0xFFu) << (8 * k);
    return tab;
}
template <uint32_t SF, uint32_t DF> struct dec_fast { static constexpr bool value =
    ((SF == 71u || SF == 77u) && DF == 28u) || (SF == 80u && DF == 61u) || (SF == 81u && DF == 63u) || (SF == 83u && DF == 49u) || (SF == 84u && DF == 51u); };

// full, aligned block at d0: true when the fast path wrote it
template <uint32_t SF, uint32_t DF>
__device__ __forceinline__ bool decode_block_fast(const uint8_t* blk, uint8_t* d0, size_t dstPitch)
{
    if (SF == 71u || SF == 77u)
    {
        // colours: BC1 block (BC3: its second half, never in the 3-colour mode), RGBA8 words of the four palette entries
        const uint8_t* cb = (SF == 77u) ? blk + 8 : blk;
        dxb_px clr[4];
        dxb_bc1_palette(cb, SF == 71u, clr);
        const uint32_t p0 = dec_bytes<SF, DF>(clr[0]), p1 = dec_bytes<SF, DF>(clr[1]), p2 = dec_bytes<SF, DF>(clr[2]), p3 = dec_bytes<SF, DF>(clr[3]);
        uint32_t dw = reinterpret_cast<const uint32_t*>(cb)[1];
        uint64_t atab = 0, abits = 0;
        if (SF == 77u)
        {
            float fa[8];
            dxb_bc3_alpha_table(blk, fa);
            #pragma unroll
            for (int k = 0; k < 8; ++k) atab |= (uint64_t)(dec_bytes<SF, DF>(dxb_make_px(0.0f, 0.0f, 0.0f, fa[k])) >> 24) << (8 * k);
            abits = *reinterpret_cast<const uint64_t*>(blk) >> 16;                 // 16 x 3 index bits
        }
        #pragma unroll
        for (uint32_t t = 0; t < 4; ++t)
        {
            uint32_t w[4];
            #pragma unroll
            for (uint32_t s2 = 0; s2 < 4; ++s2, dw >>= 2)
            {
                const uint32_t k = dw & 3u;
                uint32_t c = (k == 0u) ? p0 : (k == 1u) ? p1 : (k == 2u) ? p2 : p3;
                if (SF == 77u)
                {
                    const uint32_t a = (uint32_t)(atab >> (8u * (uint32_t)(abits & 7ull))) & 0xFFu;
                    abits >>= 3;
                    c = (c & 0x00FFFFFFu) | (a << 24);
                }
                w[s2] = c;
            }
            *reinterpret_cast<uint4*>(d0 + (size_t)t * dstPitch) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        return true;
    }
    if (SF == 80u || SF == 81u)
    {
        float g[8];
        dxb_bc4_table(blk, SF == 81u, g);
        const uint64_t tab = dec_table8<SF, DF>(g);
        uint64_t bits = *reinterpret_cast<const uint64_t*>(blk) >> 16;
        #pragma unroll
        for (uint32_t t = 0; t < 4; ++t)
        {
            uint32_t w = 0;
            #pragma unroll
            for (uint32_t s2 = 0; s2 < 4; ++s2, bits >>= 3) w |= ((uint32_t)(tab >> (8u * (uint32_t)(bits & 7ull))) & 0xFFu) << (8u * s2);
            *reinterpret_cast<uint32_t*>(d0 + (size_t)t * dstPitch) = w;
        }
        return true;
    }
    if (SF == 83u || SF == 84u)
    {
        float g[8];
        dxb_bc4_table(blk, SF == 84u, g);
        const uint64_t tabU = dec_table8<SF, DF>(g);
        dxb_bc4_table(blk + 8, SF == 84u, g);
        uint64_t tabV = 0;                                                        // second channel: byte 1 of an (0, v, 0, 1) pixel
        #pragma unroll
        for (int k = 0; k < 8; ++k) tabV |= (uint64_t)((dec_bytes<SF, DF>(dxb_make_px(0.0f, g[k], 0.0f, 1.0f)) >> 8) & 0xFFu) << (8 * k);
        uint64_t bu = *reinterpret_cast<const uint64_t*>(blk) >> 16, bv = *reinterpret_cast<const uint64_t*>(blk + 8) >> 16;
        #pragma unroll
        for (uint32_t t = 0; t < 4; ++t)
        {
            uint32_t w[2] = { 0u, 0u };
            #pragma unroll
            for (uint32_t s2 = 0; s2 < 4; ++s2, bu >>= 3, bv >>= 3)
            {
                const uint32_t u = (uint32_t)(tabU >> (8u * (uint32_t)(bu & 7ull))) & 0xFFu, v = (uint32_t)(tabV >> (8u * (uint32_t)(bv & 7ull))) & 0xFFu;
                w[s2 >> 1] |= (u | (v << 8)) << (16u * (s2 & 1u));
            }
            *reinterpret_cast<uint2*>(d0 + (size_t)t * dstPitch) = make_uint2(w[0], w[1]);
        }
        return true;
    }
    return false;
}

template <bool GENERIC, uint32_t SF, uint32_t DF>
__device__ __forceinline__ void decode_body(const dxb_job* __restrict__ jobs, const dxb_job& single, const dxb_compress_params& P)
{
    const uint32_t srcFormat = GENERIC ? P.srcFormat : SF, dstFormat = GENERIC ? P.dstFormat : DF;
    const uint32_t inF = GENERIC ? P.inF : dxb_convert_flags(SF), outF = GENERIC ? P.outF : dxb_convert_flags(DF);
    const uint32_t cflags = GENERIC ? P.cflags : 0u;
    const uint32_t stride = gridDim.x * blockDim.x;
    const uint32_t bs = dxb_bc_block_bytes(srcFormat);
    for (uint32_t unit = blockIdx.x * blockDim.x + threadIdx.x; unit < P.totalUnits; unit += stride)
    {
        const dxb_job& j = dxb_find_job(jobs, P.njobs, single, unit);
        const uint32_t local = unit - j.firstUnit;
        const uint32_t by = local / j.nbx, bx = local - by * j.nbx;
        __align__(16) uint8_t blk[16];
        const uint8_t* src = j.src + (size_t)by * j.srcPitch + (size_t)bx * bs;
        if (bs == 8) *reinterpret_cast<uint2*>(blk) = *reinterpret_cast<const uint2*>(src);
        else *reinterpret_cast<uint4*>(blk) = *reinterpret_cast<const uint4*>(src);
        const uint32_t x0 = bx * 4, y0 = by * 4;
        const uint32_t pw = (j.width - x0 < 4u) ? (j.width - x0) : 4u;
        const uint32_t ph = (j.height - y0 < 4u) ? (j.height - y0) : 4u;
        if (!GENERIC && dec_fast<GENERIC ? 0u : SF, GENERIC ? 0u : DF>::value)
        {
            constexpr uint32_t B = dxb_bytes_per_pixel(GENERIC ? 2u : DF), ROWB = 4u * B;
            uint8_t* d0 = j.dst + (size_t)y0 * j.dstPitch + (size_t)x0 * B;
            if (pw == 4u && ph == 4u && ((((uintptr_t)d0 | j.dstPitch) & (ROWB - 1u)) == 0u) &&
                decode_block_fast<GENERIC ? 71u : SF, GENERIC ? 28u : DF>(blk, d0, j.dstPitch))
                continue;
        }
        dxb_px px[16];
        dxb_decode_block(srcFormat, blk, px);
        if (!GENERIC)
        {
            constexpr uint32_t B = dxb_bytes_per_pixel(GENERIC ? 2u : DF), ROWB = 4u * B, V = (ROWB >= 16u) ? 16u : ROWB;
            uint8_t* d0 = j.dst + (size_t)y0 * j.dstPitch + (size_t)x0 * B;
            if (pw == 4u && ph == 4u && ((((uintptr_t)d0 | j.dstPitch) & (V - 1u)) == 0u))
            {
                #pragma unroll
                for (uint32_t t = 0; t < 4; ++t)
                {
                    __align__(16) uint8_t row[ROWB];
                    #pragma unroll
                    for (uint32_t s2 = 0; s2 < 4; ++s2) dxb_store_pixel(dstFormat, row, s2, dxb_convert_pixel(px[(t << 2) | s2], inF, outF, cflags));
                    uint8_t* d = d0 + (size_t)t * j.dstPitch;
                    #pragma unroll
                    for (uint32_t k = 0; k < ROWB; k += V)
                    {
                        if (V == 16u) *reinterpret_cast<uint4*>(d + k) = *reinterpret_cast<const uint4*>(row + k);
                        else if (V == 8u) *reinterpret_cast<uint2*>(d + k) = *reinterpret_cast<const uint2*>(row + k);
                        else *reinterpret_cast<uint32_t*>(d + k) = *reinterpret_cast<const uint32_t*>(row + k);
                    }
                }
                continue;
            }
        }
        for (uint32_t t = 0; t < ph; ++t)
        {
            uint8_t* row = j.dst + (size_t)(y0 + t) * j.dstPitch;
            for (uint32_t s2 = 0; s2 < pw; ++s2)
                dxb_store_pixel(dstFormat, row, x0 + s2, dxb_convert_pixel(px[(t << 2) | s2], inF, outF, cflags));
        }
    }
}

__global__ void __launch_bounds__(128) k_decompress(const dxb_job* __restrict__ jobs, dxb_job single, dxb_compress_params P)
{
    decode_body<true, 0, 0>(jobs, single, P);
}
template <uint32_t SF, uint32_t DF>
__global__ void __launch_bounds__(128) k_decompress_t(const dxb_job* __restrict__ jobs, dxb_job single, dxb_compress_params P)
{
    decode_body<false, SF, DF>(jobs, single, P);
}

// default targets (DirectXTexCompress.cpp:552-579): BC1/2/3/7 -> RGBA8, BC4 -> R8, BC5 -> R8G8, BC6H -> RGBA32F
#define DXB_DEC_PAIRS(X) X(71, 28) X(74, 28) X(77, 28) X(98, 28) X(80, 61) X(81, 63) X(83, 49) X(84, 51) X(95, 2) X(96, 2)

void dxb_launch_decompress(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P)
{
    // sRGB formats run their twins' kernels; the specialised kernels take only calls without an sRGB step (P.cflags == 0)
    const uint32_t sf = dxb_make_linear(P.srcFormat), df = dxb_make_linear(P.dstFormat);
#ifndef DXB_DEC_GENERIC_ONLY
    if (P.cflags == 0)
    {
#define DXB_X(SF, DF) if (sf == SF && df == DF) { k_decompress_t<SF, DF><<<grid, 128, 0, stream>>>(jobs, hostJobs[0], P); return; }
        DXB_DEC_PAIRS(DXB_X)
#undef DXB_X
    }
#endif
    k_decompress<<<grid, 128, 0, stream>>>(jobs, hostJobs[0], P);
}
