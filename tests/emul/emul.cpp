// tests/emul/emul.cpp — TEST INFRASTRUCTURE, never shipped.
//
// Lock-step HOST build of the exact arithmetic sources the CUDA kernels are compiled from
// (directxtex_b200/csrc/*.cuh with DXB_DEV = plain inline).  It exists so that parity against the
// oracle can be debugged in this GPU-less container; the GPU tests then check the sm_90a build
// against the oracle AND against this emulator.  The product library never contains, loads or
// calls any of this: there is no CPU fallback.
//
// Build flags mirror the device build's numeric contract: -ffp-contract=off (== nvcc -fmad=false),
// IEEE division/sqrt, -mfma only so that explicit fmaf() is one instruction (fmaf is exact either way).
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <cmath>
#include <vector>
#include <algorithm>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_pixel.cuh"
#include "dxb_block.cuh"
#include "dxb_bc15.cuh"
#ifdef DXB_EMUL_BC7
#include "dxb_bc7.cuh"
#include "dxb_bc6h.cuh"
#endif

extern "C" {

#ifdef DXB_EMUL_BC7
// experiment hook (tools/bc_quality.py): per-block forced first candidate shape for BC7, nullptr = off
static const int8_t* g_force_shapes = nullptr;
void emul_bc7_force_shapes(const int8_t* shapes) { g_force_shapes = shapes; }
#endif

int32_t emul_compress(const uint8_t* src, size_t w, size_t h, uint32_t srcFmt, size_t rowPitch,
                      uint32_t dstFmt, uint32_t flags, float threshold, uint8_t* dst)
{
    const uint32_t inF = dxb_convert_flags(srcFmt), outF = dxb_convert_flags(dstFmt);
    const uint32_t bs = dxb_bc_block_bytes(dstFmt);
    if (!inF || !outF || !bs || (inF & DXB_CONVF_BC)) return DXB_E_NOT_SUPPORTED;
    if (rowPitch == 0) rowPitch = w * dxb_bytes_per_pixel(srcFmt);
    uint32_t cflags = 0;
    if (dstFmt == DXB_FMT_BC4_UNORM || dstFmt == DXB_FMT_BC4_SNORM) cflags = DXB_FILTER_RGB_COPY_RED;
    if (dstFmt == DXB_FMT_BC5_UNORM || dstFmt == DXB_FMT_BC5_SNORM) cflags = DXB_FILTER_RGB_COPY_RED | DXB_FILTER_RGB_COPY_GREEN;
    cflags |= (flags & DXB_FILTER_SRGB_MASK);
    cflags = dxb_resolve_srgb_convert(cflags, srcFmt, dstFmt);
    const uint32_t bcflags = flags & (DXB_BC_FLAGS_DITHER_RGB | DXB_BC_FLAGS_DITHER_A | DXB_BC_FLAGS_UNIFORM | DXB_BC_FLAGS_USE_3SUBSETS | DXB_BC_FLAGS_FORCE_BC7_MODE6);
    dxb_image_desc img; img.pixels = src; img.rowPitch = rowPitch; img.width = (uint32_t)w; img.height = (uint32_t)h; img.format = srcFmt;
    const uint32_t nbx = (uint32_t)((w + 3) / 4), nby = (uint32_t)((h + 3) / 4);
#ifdef DXB_EMUL_BC7
    if (dstFmt == DXB_FMT_BC7_UNORM || dstFmt == DXB_FMT_BC7_UNORM_SRGB)
    {
        // the device kernel encodes two consecutive blocks (raster order) per warp; so does the emulator
        const long total = (long)nbx * (long)nby;
        #pragma omp parallel for schedule(dynamic, 32)
        for (long pair = 0; pair < (total + 1) / 2; ++pair)
        {
            dxb_px px[2][16];
            alignas(16) uint8_t blk[2][16];
            const long u0 = 2 * pair, u1 = u0 + 1;
            dxb_gather_block(img, (uint32_t)(u0 % nbx), (uint32_t)(u0 / nbx), inF, outF, cflags, px[0]);
            if (u1 < total) dxb_gather_block(img, (uint32_t)(u1 % nbx), (uint32_t)(u1 / nbx), inF, outF, cflags, px[1]);
            dxb_bc7_dbg_force_shape[0] = g_force_shapes ? g_force_shapes[u0] : -1;
            dxb_bc7_dbg_force_shape[1] = (g_force_shapes && u1 < total) ? g_force_shapes[u1] : -1;
            dxb_bc7_encode_pair_emul(px[0], (u1 < total) ? px[1] : nullptr, bcflags, blk[0], blk[1]);
            memcpy(dst + (size_t)u0 * bs, blk[0], bs);
            if (u1 < total) memcpy(dst + (size_t)u1 * bs, blk[1], bs);
        }
        return DXB_S_OK;
    }
#endif
#ifdef DXB_EMUL_BC7
    if (dstFmt == DXB_FMT_BC6H_UF16 || dstFmt == DXB_FMT_BC6H_SF16)
    {
        const long total = (long)nbx * (long)nby;
        #pragma omp parallel for schedule(dynamic, 32)
        for (long pair = 0; pair < (total + 1) / 2; ++pair)
        {
            dxb_px px[2][16];
            alignas(16) uint8_t blk[2][16];
            const long u0 = 2 * pair, u1 = u0 + 1;
            dxb_gather_block(img, (uint32_t)(u0 % nbx), (uint32_t)(u0 / nbx), inF, outF, cflags, px[0]);
            if (u1 < total) dxb_gather_block(img, (uint32_t)(u1 % nbx), (uint32_t)(u1 / nbx), inF, outF, cflags, px[1]);
            dxb_bc6h_encode_pair_emul(px[0], (u1 < total) ? px[1] : nullptr, dstFmt == DXB_FMT_BC6H_SF16, blk[0], blk[1]);
            memcpy(dst + (size_t)u0 * bs, blk[0], bs);
            if (u1 < total) memcpy(dst + (size_t)u1 * bs, blk[1], bs);
        }
        return DXB_S_OK;
    }
#endif
    #pragma omp parallel for schedule(dynamic, 8)
    for (long by = 0; by < (long)nby; ++by)
        for (uint32_t bx = 0; bx < nbx; ++bx)
        {
            dxb_px px[16];
            dxb_gather_block(img, bx, (uint32_t)by, inF, outF, cflags, px);
            alignas(16) uint8_t blk[16];
            dxb_encode_block_bc15(dstFmt, px, bcflags, threshold, blk);
            memcpy(dst + ((size_t)by * nbx + bx) * bs, blk, bs);
        }
    return DXB_S_OK;
}

// Row-wise format conversion (ConvertCustom no-dither path, DirectXTexConvert.cpp:4888-4908)
int32_t emul_convert(const uint8_t* src, size_t w, size_t h, uint32_t srcFmt, size_t srcPitch,
                     uint32_t dstFmt, size_t dstPitch, uint32_t filter, uint8_t* dst)
{
    const uint32_t inF = dxb_convert_flags(srcFmt), outF = dxb_convert_flags(dstFmt);
    if (!inF || !outF || ((inF | outF) & DXB_CONVF_BC)) return DXB_E_NOT_SUPPORTED;
    if (srcPitch == 0) srcPitch = w * dxb_bytes_per_pixel(srcFmt);
    if (dstPitch == 0) dstPitch = w * dxb_bytes_per_pixel(dstFmt);
    const uint32_t flags = dxb_resolve_srgb_convert(filter, srcFmt, dstFmt);
    if (flags & DXB_FILTER_DITHER_DIFFUSION)
    {
        std::vector<dxb_px> E(2 * (w + 2));
        dxb_convert_diffuse_image(srcFmt, dstFmt, inF, outF, flags, src, srcPitch, dst, dstPitch, (uint32_t)w, (uint32_t)h, E.data(), E.data() + w + 2);
        return DXB_S_OK;
    }
    for (size_t y = 0; y < h; ++y)
        for (size_t x = 0; x < w; ++x)
        {
            dxb_px v = dxb_load_pixel(srcFmt, src + y * srcPitch, x);
            v = dxb_convert_pixel(v, inF, outF, flags);
            if (flags & DXB_FILTER_DITHER) dxb_store_pixel_dither(dstFmt, dst + y * dstPitch, x, (uint32_t)y, v);
            else dxb_store_pixel(dstFmt, dst + y * dstPitch, x, v, 0.5f);       // TEX_THRESHOLD_DEFAULT (B5G5R5A1 alpha bit)
        }
    return DXB_S_OK;
}

} // extern "C"

// ---- mip chain emulation: same per-pixel functions as k_mip_level ---------------------------------
#include "dxb_mips.cuh"
#include "dxb_host_tri.h"

// ScaleMipMapsAlphaForCoverage for one chain held in `src` (ScratchImage layout); result chain in `dst`
extern "C" int32_t emul_scale_mips_alpha(const uint8_t* src, uint8_t* dst, const size_t* offsets, const size_t* widths, const size_t* heights,
                                         const size_t* pitches, size_t levels, uint32_t fmt, float ref);

extern "C" int32_t emul_generate_mipmaps(uint8_t* chainBase, const size_t* offsets, const size_t* widths, const size_t* heights,
                                         const size_t* pitches, size_t levels, uint32_t fmt, uint32_t filter)
{
    if (!dxb_bytes_per_pixel(fmt)) return DXB_E_NOT_SUPPORTED;
    uint32_t mode = filter & DXB_FILTER_MODE_MASK;
    auto ispow2 = [](size_t x) { return x && !(x & (x - 1)); };
    if (!mode) mode = (ispow2(widths[0]) && ispow2(heights[0])) ? DXB_FILTER_BOX : DXB_FILTER_LINEAR;
    if (mode == DXB_FILTER_BOX && (!ispow2(widths[0]) || !ispow2(heights[0]))) return DXB_E_FAIL;
    const uint32_t lflags = dxb_resolve_srgb_linear(filter & DXB_FILTER_SRGB_MASK, fmt);
    const uint8_t* stale = nullptr; size_t stalePitch = 0;
    for (size_t l = 1; l < levels; ++l)
    {
        dxb_mip_job j;
        j.src = chainBase + offsets[l - 1]; j.dst = chainBase + offsets[l];
        j.srcPitch = pitches[l - 1]; j.dstPitch = pitches[l];
        j.sw = (uint32_t)widths[l - 1]; j.sh = (uint32_t)heights[l - 1]; j.dw = (uint32_t)widths[l]; j.dh = (uint32_t)heights[l];
        j.firstUnit = 0;
        if (j.sh == 2) { stale = j.src + j.srcPitch; stalePitch = j.srcPitch; }
        j.stale = nullptr; j.stalePitch = 0;
        if (mode == DXB_FILTER_BOX && j.sh <= 1 && j.sw > 1 && stale) { j.stale = stale; j.stalePitch = stalePitch; }
        TriLists tx, ty; dxb_tri_axis ax{}, ay{};
        if (mode == DXB_FILTER_TRIANGLE)
        {
            build_triangle_axis(j.sw, j.dw, (filter & DXB_FILTER_WRAP_U) != 0, tx);
            build_triangle_axis(j.sh, j.dh, (filter & DXB_FILTER_WRAP_V) != 0, ty);
            ax.off = tx.off.data(); ax.src = tx.src.data(); ax.w = tx.w.data();
            ay.off = ty.off.data(); ay.src = ty.src.data(); ay.w = ty.w.data();
        }
        for (uint32_t y = 0; y < j.dh; ++y)
            for (uint32_t x = 0; x < j.dw; ++x)
            {
                dxb_px v;
                switch (mode)
                {
                case DXB_FILTER_POINT:
                    v = dxb_mip_point(fmt, j, x, y);
                    dxb_store_pixel(fmt, j.dst + (size_t)y * j.dstPitch, x, v);
                    continue;
                case DXB_FILTER_BOX: v = dxb_mip_box(fmt, j, x, y, lflags); break;
                case DXB_FILTER_LINEAR: v = dxb_mip_linear(fmt, j, x, y, filter, lflags); break;
                case DXB_FILTER_CUBIC: v = dxb_mip_cubic(fmt, j, x, y, filter, lflags); break;
                default: v = dxb_mip_triangle(fmt, j, x, y, lflags, ax, ay); break;
                }
                dxb_store_linear(fmt, j.dst, j.dstPitch, x, y, v, lflags);
            }
    }
    return DXB_S_OK;
}

// ---- Decompress emulation (DecompressBC, DirectXTexCompress.cpp:425-535) -----------------------------------
#include "dxb_decode.cuh"
extern "C" int32_t emul_decompress(const uint8_t* blocks, size_t w, size_t h, uint32_t bcFmt, uint32_t dstFmt, uint8_t* dst)
{
    const uint32_t bs = dxb_bc_block_bytes(bcFmt), bpp = dxb_bytes_per_pixel(dstFmt);
    if (!bs || !bpp) return DXB_E_NOT_SUPPORTED;
    const uint32_t inF = dxb_convert_flags(bcFmt), outF = dxb_convert_flags(dstFmt);
    const uint32_t cflags = dxb_resolve_srgb_convert(0, bcFmt, dstFmt);
    const size_t nbx = (w + 3) / 4, nby = (h + 3) / 4, dpitch = w * bpp;
    for (size_t by = 0; by < nby; ++by)
        for (size_t bx = 0; bx < nbx; ++bx)
        {
            dxb_px px[16];
            alignas(16) uint8_t blk[16];
            memcpy(blk, blocks + (by * nbx + bx) * bs, bs);
            dxb_decode_block(bcFmt, blk, px);
            for (size_t t = 0; t < 4 && by * 4 + t < h; ++t)
                for (size_t s2 = 0; s2 < 4 && bx * 4 + s2 < w; ++s2)
                    dxb_store_pixel(dstFmt, dst + (by * 4 + t) * dpitch, bx * 4 + s2, dxb_convert_pixel(px[(t << 2) | s2], inF, outF, cflags));
        }
    return DXB_S_OK;
}

static float emul_alpha_coverage(const uint8_t* img, size_t w, size_t h, size_t pitch, uint32_t fmt, float ref, float scale)
{
    if (w < 2 || h < 2) return 0.0f;
    unsigned long long count = 0;
    for (size_t y = 0; y + 1 < h; ++y)
        for (size_t x = 0; x + 1 < w; ++x)
        {
            const uint8_t* r0 = img + y * pitch; const uint8_t* r1 = r0 + pitch;
            count += dxb_alpha_coverage_cell(dxb_load_pixel(fmt, r0, x).w, dxb_load_pixel(fmt, r1, x).w,
                                             dxb_load_pixel(fmt, r0, x + 1).w, dxb_load_pixel(fmt, r1, x + 1).w, scale, ref);
        }
    const float cscale = static_cast<float>((w - 1) * (h - 1) * 8 * 8);
    return cscale > 0.0f ? static_cast<float>(count) / cscale : 0.0f;
}
int32_t emul_scale_mips_alpha(const uint8_t* src, uint8_t* dst, const size_t* offsets, const size_t* widths, const size_t* heights,
                              const size_t* pitches, size_t levels, uint32_t fmt, float ref)
{
    if (!dxb_bytes_per_pixel(fmt)) return DXB_E_NOT_SUPPORTED;
    const float target = emul_alpha_coverage(src + offsets[0], widths[0], heights[0], pitches[0], fmt, ref, 1.0f);
    memcpy(dst + offsets[0], src + offsets[0], pitches[0] * heights[0]);
    for (size_t l = 1; l < levels; ++l)
    {
        float lo = 0.0f, hi = 4.0f, scale = 1.0f;
        for (int it = 0; it < 10; ++it)
        {
            const float cov = emul_alpha_coverage(src + offsets[l], widths[l], heights[l], pitches[l], fmt, ref, scale);
            if (cov < target) lo = scale;
            else if (cov > target) hi = scale;
            else break;
            scale = (lo + hi) * 0.5f;
        }
        for (size_t y = 0; y < heights[l]; ++y)
            for (size_t x = 0; x < widths[l]; ++x)
                dxb_scale_alpha_pixel(fmt, src + offsets[l] + y * pitches[l], dst + offsets[l] + y * pitches[l], (uint32_t)x, scale);
    }
    return DXB_S_OK;
}

#ifdef DXB_EMUL_BC7
// experiment hook: stage-1 estimates of every two-subset shape for one block (ldr = 16 RGBA pixels as floats 0..255)
extern "C" void emul_bc7_shape_estimates(const float* ldr, float nl, int opaque, float* out64)
{
    static thread_local dxb_bc7_scratch S;
    for (int i = 0; i < 16; ++i) { S.px[i] = dxb_make_px(ldr[4 * i], ldr[4 * i + 1], ldr[4 * i + 2], ldr[4 * i + 3]); S.px[16 + i] = S.px[i]; }
    dxb_bc7_build_moments(&S);
    float tot[14];
    dxb_bc7_mt_load(S.mt[0], 64, tot);
    for (uint32_t s = 0; s < 64; ++s) out64[s] = dxb_bc7_shape_h1(S.pq, S.mt[0], s, tot, opaque != 0);
}
#endif
