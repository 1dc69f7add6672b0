// tests/emul/emul.cpp — TEST INFRASTRUCTURE, never shipped.
//
// Lock-step HOST build of the exact arithmetic sources the CUDA kernels are compiled from
// (directxtex_b200/csrc/*.cuh with DXB_DEV = plain inline).  It exists so that parity against the
// oracle can be debugged in this GPU-less container; the GPU tests then check the sm_90a build
// against the oracle AND against this emulator.  The product library never contains, loads or
// calls any of this: there is no CPU fallback.
//
// Every entry point plans its call with the library's own planners (csrc/dxb_plan.h): argument checks and HRESULTs, flag
// resolution, the filter mode and a chain's job records.  Only the per-pixel and per-block walk is restated here.
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
#include "dxb_plan.h"
#include "dxb_pixel.cuh"
#include "dxb_block.cuh"
#include "dxb_bc15.cuh"
#ifdef DXB_EMUL_BC7
#include "dxb_bc7.cuh"
#include "dxb_bc6h.cuh"
#endif

// The dxb200_image the library's planners see for one w x h image at `pixels` (rowPitch 0: the tight pitch).  An unimplemented
// format keeps pitches of 0: every planner refuses it before a pitch is read.
static dxb200_image emul_image(const uint8_t* pixels, size_t w, size_t h, uint32_t fmt, size_t rowPitch)
{
    dxb200_image im = { w, h, fmt, 0, 0, const_cast<uint8_t*>(pixels) };
    (void)compute_pitch(fmt, w, h, &im.rowPitch, &im.slicePitch);
    if (rowPitch) { im.rowPitch = rowPitch; im.slicePitch = rowPitch * h; }
    return im;
}

extern "C" {

#ifdef DXB_EMUL_BC7
// experiment hook (tools/bc_quality.py): per-block forced first candidate shape for BC7, nullptr = off
static const int8_t* g_force_shapes = nullptr;
void emul_bc7_force_shapes(const int8_t* shapes) { g_force_shapes = shapes; }
#endif

int32_t emul_compress(const uint8_t* src, size_t w, size_t h, uint32_t srcFmt, size_t rowPitch,
                      uint32_t dstFmt, uint32_t flags, float threshold, uint8_t* dst)
{
    const dxb200_image s = emul_image(src, w, h, srcFmt, rowPitch), d = emul_image(dst, w, h, dstFmt, 0);
    CompressPlan plan;
    const int32_t hr = plan_compress(&s, 1, dstFmt, flags, threshold, &d, &plan);
    if (hr != DXB_S_OK) return hr;
    const uint32_t inF = plan.P.inF, outF = plan.P.outF, cflags = plan.P.cflags, bcflags = plan.P.bcflags;
    const uint32_t bs = dxb_bc_block_bytes(dstFmt);
    dxb_image_desc img; img.pixels = src; img.rowPitch = s.rowPitch; img.width = (uint32_t)w; img.height = (uint32_t)h; img.format = srcFmt;
    const uint32_t nbx = (uint32_t)((w + 3) / 4), nby = (uint32_t)((h + 3) / 4);
#ifdef DXB_EMUL_BC7
    if (plan.bc7)
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
    if (plan.bc6h)
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
            dxb_encode_block_bc15(dstFmt, px, bcflags, plan.P.threshold, blk);
            memcpy(dst + ((size_t)by * nbx + bx) * bs, blk, bs);
        }
    return DXB_S_OK;
}

// Row-wise format conversion (ConvertCustom no-dither path, DirectXTexConvert.cpp:4888-4908)
int32_t emul_convert(const uint8_t* src, size_t w, size_t h, uint32_t srcFmt, size_t srcPitch,
                     uint32_t dstFmt, size_t dstPitch, uint32_t filter, uint8_t* dst)
{
    const dxb200_image s = emul_image(src, w, h, srcFmt, srcPitch), d = emul_image(dst, w, h, dstFmt, dstPitch);
    dxb_convert_params P;
    const int32_t hr = plan_convert(&s, 1, dstFmt, filter, &d, &P);
    if (hr != DXB_S_OK) return hr;
    const uint32_t inF = P.inF, outF = P.outF, flags = P.flags;
    if (flags & DXB_FILTER_DITHER_DIFFUSION)
    {
        std::vector<dxb_px> E(2 * (w + 2));
        dxb_convert_diffuse_image(srcFmt, dstFmt, inF, outF, flags, src, s.rowPitch, dst, d.rowPitch, (uint32_t)w, (uint32_t)h, E.data(), E.data() + w + 2);
        return DXB_S_OK;
    }
    for (size_t y = 0; y < h; ++y)
        for (size_t x = 0; x < w; ++x)
        {
            dxb_px v = dxb_load_pixel(srcFmt, src + y * s.rowPitch, x);
            v = dxb_convert_pixel(v, inF, outF, flags);
            if (flags & DXB_FILTER_DITHER) dxb_store_pixel_dither(dstFmt, dst + y * d.rowPitch, x, (uint32_t)y, v);
            else dxb_store_pixel(dstFmt, dst + y * d.rowPitch, x, v, P.threshold);
        }
    return DXB_S_OK;
}

} // extern "C"

// ---- mip chain emulation: dxb_mip_pixel, the same function k_mip_level and k_mip_tail run per pixel --------------------
#include "dxb_mips.cuh"

// the dxb200_image records of one chain held in ScratchImage layout at `base`
static std::vector<dxb200_image> emul_chain(const uint8_t* base, const size_t* offsets, const size_t* widths, const size_t* heights,
                                            const size_t* pitches, size_t levels, uint32_t fmt)
{
    std::vector<dxb200_image> chain(levels);
    for (size_t l = 0; l < levels; ++l) chain[l] = emul_image(base + offsets[l], widths[l], heights[l], fmt, pitches[l]);
    return chain;
}

// levels 1 .. levels-1 of one chain planned by build_mip_plan, every pixel through dxb_mip_pixel
static void emul_run_mip_plan(const std::vector<dxb200_image>& chain, size_t levels, uint32_t filter, uint32_t mode)
{
    const MipPlan mp = build_mip_plan(chain.data(), 1, levels, filter, mode);
    for (size_t l = 1; l < levels; ++l)
    {
        const dxb_mip_job& j = mp.jobs[l - 1];
        dxb_tri_axis ax{}, ay{};
        if (!mp.tri.empty())
        {
            const TriLists& tx = mp.tri[2 * (l - 1)]; const TriLists& ty = mp.tri[2 * (l - 1) + 1];
            ax = { tx.off.data(), tx.src.data(), tx.w.data() };
            ay = { ty.off.data(), ty.src.data(), ty.w.data() };
        }
        for (uint32_t y = 0; y < j.dh; ++y)
            for (uint32_t x = 0; x < j.dw; ++x) dxb_mip_pixel(mp.P.format, mp.P.mode, j, x, y, mp.P.filter, mp.P.lflags, ax, ay);
    }
}

extern "C" int32_t emul_generate_mipmaps(uint8_t* chainBase, const size_t* offsets, const size_t* widths, const size_t* heights,
                                         const size_t* pitches, size_t levels, uint32_t fmt, uint32_t filter)
{
    const std::vector<dxb200_image> chain = emul_chain(chainBase, offsets, widths, heights, pitches, levels, fmt);
    uint32_t mode = 0;
    const int32_t hr = plan_mips(chain.data(), 1, levels, filter, &mode);
    if (hr != DXB_S_OK) return hr;
    emul_run_mip_plan(chain, levels, filter, mode);
    return DXB_S_OK;
}

// Resize of one tight w x h image to width x height: the library plans it as a chain of two levels (plan_resize)
extern "C" int32_t emul_resize(const uint8_t* src, size_t w, size_t h, uint32_t fmt, size_t width, size_t height, uint32_t filter, uint8_t* dst)
{
    const std::vector<dxb200_image> chain = { emul_image(src, w, h, fmt, 0), emul_image(dst, width, height, fmt, 0) };
    uint32_t mode = 0;
    const int32_t hr = plan_resize(&chain[0], 1, filter, &chain[1], &mode);
    if (hr != DXB_S_OK) return hr;
    emul_run_mip_plan(chain, 2, filter, mode);
    return DXB_S_OK;
}

// ---- Decompress emulation (DecompressBC, DirectXTexCompress.cpp:425-535) -----------------------------------
#include "dxb_decode.cuh"
extern "C" int32_t emul_decompress(const uint8_t* blocks, size_t w, size_t h, uint32_t bcFmt, uint32_t dstFmt, uint8_t* dst)
{
    const dxb200_image s = emul_image(blocks, w, h, bcFmt, 0), d = emul_image(dst, w, h, dstFmt, 0);
    dxb_compress_params P;
    const int32_t hr = plan_decompress(&s, 1, dstFmt, &d, &P);
    if (hr != DXB_S_OK) return hr;
    const uint32_t bs = dxb_bc_block_bytes(bcFmt), inF = P.inF, outF = P.outF, cflags = P.cflags;
    const size_t nbx = (w + 3) / 4, nby = (h + 3) / 4, dpitch = d.rowPitch;
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

static float emul_alpha_coverage(const dxb200_image& im, float ref, float scale)
{
    unsigned long long count = 0;
    for (size_t y = 0; y + 1 < im.height; ++y)
        for (size_t x = 0; x + 1 < im.width; ++x)
        {
            const uint8_t* r0 = im.pixels + y * im.rowPitch; const uint8_t* r1 = r0 + im.rowPitch;
            count += dxb_alpha_coverage_cell(dxb_load_pixel(im.format, r0, x).w, dxb_load_pixel(im.format, r1, x).w,
                                             dxb_load_pixel(im.format, r0, x + 1).w, dxb_load_pixel(im.format, r1, x + 1).w, scale, ref);
        }
    return alpha_coverage_fraction(count, im.width, im.height);
}

// ScaleMipMapsAlphaForCoverage for one chain held in `src` (ScratchImage layout); result chain in `dst`
extern "C" int32_t emul_scale_mips_alpha(const uint8_t* src, uint8_t* dst, const size_t* offsets, const size_t* widths, const size_t* heights,
                                         const size_t* pitches, size_t levels, uint32_t fmt, float ref)
{
    const std::vector<dxb200_image> s = emul_chain(src, offsets, widths, heights, pitches, levels, fmt);
    const std::vector<dxb200_image> d = emul_chain(dst, offsets, widths, heights, pitches, levels, fmt);
    const int32_t hr = plan_alpha_coverage(s.data(), levels, d.data());
    if (hr != DXB_S_OK) return hr;
    const float target = emul_alpha_coverage(s[0], ref, 1.0f);
    memcpy(d[0].pixels, s[0].pixels, s[0].rowPitch * s[0].height);
    for (size_t l = 1; l < levels; ++l)
    {
        float scale = 1.0f;
        (void)estimate_alpha_scale(target, [&](float sc, float* cov) { *cov = emul_alpha_coverage(s[l], ref, sc); return DXB_S_OK; }, &scale);
        for (size_t y = 0; y < s[l].height; ++y)
            for (size_t x = 0; x < s[l].width; ++x)
                dxb_scale_alpha_pixel(fmt, s[l].pixels + y * s[l].rowPitch, d[l].pixels + y * d[l].rowPitch, (uint32_t)x, scale);
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
