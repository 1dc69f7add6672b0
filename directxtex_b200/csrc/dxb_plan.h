// dxb_plan.h — HOST-side planning of every library call (shared by dxb_api.cu and tests/emul): argument checks with the
// reference's HRESULTs, flag resolution, the filter mode, the job records of a mip chain and the alpha-coverage bisection.
// Plain C++, no CUDA: the records only carry the caller's pointers, host or device.
#pragma once
#include <vector>
#include <cstring>
#include <cstdint>
#include <cstddef>
#include <algorithm>

#include "../../include/dxtex_b200.h"
#include "dxb_formats.h"
#include "dxb_jobs.h"
#include "dxb_host_tri.h"

namespace {

// ---- format predicates (DirectXTex.inl:57-130 / DirectXTexUtil.cpp), implemented subset ----------
bool is_compressed(uint32_t f) { return dxb_bc_block_bytes(f) != 0; }
bool is_supported_pixel_format(uint32_t f) { return dxb_bytes_per_pixel(f) != 0; }

int32_t compute_pitch(uint32_t fmt, size_t w, size_t h, size_t* row, size_t* slice)
{
    if (const uint32_t bs = dxb_bc_block_bytes(fmt))
    {
        const size_t nbw = std::max<size_t>(1, (w + 3) / 4), nbh = std::max<size_t>(1, (h + 3) / 4);
        *row = nbw * bs; *slice = *row * nbh;
        return DXB_S_OK;
    }
    if (const uint32_t bpp = dxb_bytes_per_pixel(fmt))
    {
        *row = w * bpp; *slice = *row * h;
        return DXB_S_OK;
    }
    return DXB_E_NOT_SUPPORTED;
}

size_t count_mips(size_t w, size_t h)
{
    size_t n = 1;
    while (h > 1 || w > 1) { if (h > 1) h >>= 1; if (w > 1) w >>= 1; ++n; }
    return n;
}

// ---- Compress ---------------------------------------------------------------------------------
struct CompressPlan { dxb_compress_params P; bool bc7, bc6h; };

// validation + flag resolution shared by host and device variants (DirectXTexCompress.cpp:664-676, 732-749, 72-107)
int32_t plan_compress(const dxb200_image* src, size_t n, uint32_t dstFormat, uint32_t flags, float threshold,
                      const dxb200_image* dst, CompressPlan* plan)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t srcFormat = src[0].format;
    if (is_compressed(srcFormat) || !is_compressed(dstFormat)) return DXB_E_INVALIDARG;
    if (!is_supported_pixel_format(srcFormat)) return DXB_E_NOT_SUPPORTED;        // no CPU fallback for other formats
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != srcFormat || dst[i].format != dstFormat) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height) return DXB_E_FAIL;
        if (!src[i].width || !src[i].height || src[i].width > 0xFFFFFFFFull || src[i].height > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    }
    dxb_compress_params& P = plan->P;
    P.srcFormat = srcFormat; P.dstFormat = dstFormat;
    P.inF = dxb_convert_flags(srcFormat); P.outF = dxb_convert_flags(dstFormat);
    const uint32_t cflags = dxb_bc15_default_cflags(dstFormat) | (flags & DXB_FILTER_SRGB_MASK);      // DetermineEncoderSettings :46-68, GetSRGBFlags :37-44
    P.cflags = dxb_resolve_srgb_convert(cflags, srcFormat, dstFormat);
    P.bcflags = flags & (DXB_BC_FLAGS_DITHER_RGB | DXB_BC_FLAGS_DITHER_A | DXB_BC_FLAGS_UNIFORM |
                         DXB_BC_FLAGS_USE_3SUBSETS | DXB_BC_FLAGS_FORCE_BC7_MODE6);                 // GetBCFlags :26-35
    P.threshold = threshold;
    plan->bc7 = (dxb_make_linear(dstFormat) == DXB_FMT_BC7_UNORM);
    plan->bc6h = (dstFormat == DXB_FMT_BC6H_UF16 || dstFormat == DXB_FMT_BC6H_SF16);
    return DXB_S_OK;
}

// ---- Decompress (DirectXTexCompress.cpp:852-979; DecompressBC :425-535) ---------------------------------
int32_t plan_decompress(const dxb200_image* src, size_t n, uint32_t dstFormat, const dxb200_image* dst, dxb_compress_params* P)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t srcFormat = src[0].format;
    if (!is_compressed(srcFormat) || is_compressed(dstFormat)) return DXB_E_INVALIDARG;
    if (!is_supported_pixel_format(dstFormat)) return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != srcFormat || dst[i].format != dstFormat) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height) return DXB_E_FAIL;
        if (!src[i].width || !src[i].height || src[i].width > 0xFFFFFFFFull || src[i].height > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    }
    memset(P, 0, sizeof(*P));
    P->srcFormat = srcFormat; P->dstFormat = dstFormat;
    P->inF = dxb_convert_flags(srcFormat); P->outF = dxb_convert_flags(dstFormat);
    P->cflags = dxb_resolve_srgb_convert(0, srcFormat, dstFormat);          // ConvertScanline(..., TEX_FILTER_DEFAULT) (:500)
    return DXB_S_OK;
}

// ---- Convert ----------------------------------------------------------------------------------
int32_t plan_convert(const dxb200_image* src, size_t n, uint32_t dstFormat, uint32_t filter, const dxb200_image* dst, dxb_convert_params* P)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t srcFormat = src[0].format;
    // Convert/ConvertEx argument checks (DirectXTexConvert.cpp:5113-5125): same format, BC formats -> E_INVALIDARG
    if (srcFormat == dstFormat) return DXB_E_INVALIDARG;
    if (is_compressed(srcFormat) || is_compressed(dstFormat)) return DXB_E_INVALIDARG;
    if (!is_supported_pixel_format(srcFormat) || !is_supported_pixel_format(dstFormat)) return DXB_E_NOT_SUPPORTED;
    // TEX_FILTER_DITHER = ordered 4x4 dithering; TEX_FILTER_DITHER_DIFFUSION = Floyd-Steinberg (serial per image, :4815-4858)
    if (filter & (DXB_FILTER_DITHER_MASK & ~(DXB_FILTER_DITHER | DXB_FILTER_DITHER_DIFFUSION))) return DXB_E_NOT_SUPPORTED;
    // the 16-bit packed destinations have dithered stores in the reference (:4302-4500) that this backend does not restate yet
    if ((filter & DXB_FILTER_DITHER_MASK) && (dstFormat == DXB_FMT_B5G6R5_UNORM || dstFormat == DXB_FMT_B5G5R5A1_UNORM || dstFormat == DXB_FMT_B4G4R4A4_UNORM))
        return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != srcFormat || dst[i].format != dstFormat) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height) return DXB_E_FAIL;
        if ((uint64_t)src[i].width * src[i].height > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    }
    P->srcFormat = srcFormat; P->dstFormat = dstFormat;
    P->inF = dxb_convert_flags(srcFormat); P->outF = dxb_convert_flags(dstFormat);
    P->flags = dxb_resolve_srgb_convert(filter, srcFormat, dstFormat);
    P->threshold = 0.5f;
    return DXB_S_OK;
}

// ---- PremultiplyAlpha ---------------------------------------------------------------------------
int32_t plan_pmalpha(const dxb200_image* src, size_t n, uint32_t flags, const dxb200_image* dst, dxb_convert_params* P)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = src[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                                 // :224-229
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    if (!(dxb_convert_flags(fmt) & DXB_CONVF_A)) return DXB_E_NOT_SUPPORTED;            // !HasAlpha
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != fmt || dst[i].format != fmt) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height || !src[i].width || !src[i].height) return DXB_E_INVALIDARG;
    }
    memset(P, 0, sizeof(*P));
    P->srcFormat = fmt; P->dstFormat = fmt; P->inF = P->outF = dxb_convert_flags(fmt);
    // TEX_PMALPHA_IGNORE_SRGB = 0x1, TEX_PMALPHA_REVERSE = 0x2; the SRGB bits equal TEX_FILTER_SRGB_IN/OUT (:21-26)
    const uint32_t lflags = (flags & 0x1u) ? 0u : dxb_resolve_srgb_linear(flags & DXB_FILTER_SRGB_MASK, fmt);
    P->flags = (lflags & (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT)) | ((flags & 0x2u) ? 1u : 0u);
    return DXB_S_OK;
}

// ---- GenerateMipMaps ----------------------------------------------------------------------------
bool ispow2(size_t x) { return ((x != 0) && !(x & (x - 1))); }

int32_t plan_mips(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter, uint32_t* mode)
{
    if (!chain || !items || levels < 2) return DXB_E_INVALIDARG;
    const uint32_t fmt = chain[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                         // GenerateMipMaps :2852-2856
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    const size_t w = chain[0].width, h = chain[0].height;
    if (levels > count_mips(w, h)) return DXB_E_INVALIDARG;
    for (size_t it = 0; it < items; ++it)
    {
        size_t lw = w, lh = h;
        for (size_t l = 0; l < levels; ++l)
        {
            const dxb200_image& im = chain[it * levels + l];
            if (!im.pixels) return DXB_E_POINTER;
            if (im.format != fmt || im.width != lw || im.height != lh) return DXB_E_INVALIDARG;
            if (lh > 1) lh >>= 1;
            if (lw > 1) lw >>= 1;
        }
    }
    uint32_t m = filter & DXB_FILTER_MODE_MASK;
    if (!m) m = (ispow2(w) && ispow2(h)) ? DXB_FILTER_BOX : DXB_FILTER_LINEAR;   // :3169-3174
    switch (m)
    {
    case DXB_FILTER_BOX: if (!ispow2(w) || !ispow2(h)) return DXB_E_FAIL; break;     // :1005-1006
    case DXB_FILTER_POINT: case DXB_FILTER_LINEAR: case DXB_FILTER_CUBIC: case DXB_FILTER_TRIANGLE: break;
    default: return DXB_E_NOT_SUPPORTED;
    }
    if ((uint64_t)w * h * items > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    *mode = m;
    return DXB_S_OK;
}

// Resize = one filter pass from src[i] to dst[i] (PerformResizeUsingCustomFilters, DirectXTexResize.cpp:805-837)
int32_t plan_resize(const dxb200_image* src, size_t n, uint32_t filter, const dxb200_image* dst, uint32_t* mode)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = src[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                         // Resize :875-879
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    const size_t sw = src[0].width, sh = src[0].height, dw = dst[0].width, dh = dst[0].height;
    if (!sw || !sh || !dw || !dh) return DXB_E_INVALIDARG;
    if (sw > 0xFFFFFFFFull || sh > 0xFFFFFFFFull || dw > 0xFFFFFFFFull || dh > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != fmt || dst[i].format != fmt) return DXB_E_INVALIDARG;
        if (src[i].width != sw || src[i].height != sh || dst[i].width != dw || dst[i].height != dh) return DXB_E_INVALIDARG;
    }
    uint32_t m = filter & DXB_FILTER_MODE_MASK;
    if (!m) m = ((dw << 1) == sw && (dh << 1) == sh) ? DXB_FILTER_BOX : DXB_FILTER_LINEAR;      // :812-817
    switch (m)
    {
    case DXB_FILTER_BOX: if ((dw << 1) != sw || (dh << 1) != sh) return DXB_E_FAIL; break;      // :318-319
    case DXB_FILTER_POINT: case DXB_FILTER_LINEAR: case DXB_FILTER_CUBIC: case DXB_FILTER_TRIANGLE: break;
    default: return DXB_E_NOT_SUPPORTED;
    }
    if ((uint64_t)dw * dh * n > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    *mode = m;
    return DXB_S_OK;
}

// What levels 1 .. levels-1 of `items` chains run (a resize is a chain of two levels per item): P with format, mode, filter and
// lflags; the [level - 1][item] job records; TRIANGLE's gather lists, X and Y of every level (shared by all items).
struct MipPlan { dxb_mip_params P; std::vector<dxb_mip_job> jobs; std::vector<TriLists> tri; };

// chain[it * levels + l] = level l of item it, validated by plan_mips / plan_resize; its pointers are only copied into the records
MipPlan build_mip_plan(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter, uint32_t mode)
{
    MipPlan mp;
    const uint32_t fmt = chain[0].format;
    dxb_mip_params& P = mp.P; memset(&P, 0, sizeof(P));
    P.format = fmt; P.mode = mode; P.filter = filter;
    P.lflags = dxb_resolve_srgb_linear(filter & DXB_FILTER_SRGB_MASK, fmt);
    std::vector<const dxb200_image*> stale(items, nullptr);
    std::vector<dxb_mip_job>& all = mp.jobs;
    all.resize(items * (levels - 1));
    for (size_t l = 1; l < levels; ++l)
    {
        uint64_t total = 0;
        for (size_t it = 0; it < items; ++it)
        {
            const dxb200_image& s = chain[it * levels + l - 1]; const dxb200_image& d = chain[it * levels + l];
            dxb_mip_job& j = all[(l - 1) * items + it];
            j.src = s.pixels; j.dst = d.pixels; j.srcPitch = s.rowPitch; j.dstPitch = d.rowPitch;
            j.sw = (uint32_t)s.width; j.sh = (uint32_t)s.height; j.dw = (uint32_t)d.width; j.dh = (uint32_t)d.height;
            j.firstUnit = (uint32_t)total; total += (uint64_t)j.dw * j.dh;
            if (s.height == 2) stale[it] = &s;          // box filter quirk, see dxb_mip_box
            j.stale = nullptr; j.stalePitch = 0;
            if (mode == DXB_FILTER_BOX && s.height <= 1 && s.width > 1 && stale[it])
            {
                j.stale = stale[it]->pixels + stale[it]->rowPitch;      // row 1 of that level
                j.stalePitch = stale[it]->rowPitch;
            }
        }
    }
    mp.tri.resize(mode == DXB_FILTER_TRIANGLE ? 2 * (levels - 1) : 0);
    for (size_t l = 1; l <= mp.tri.size() / 2; ++l)
    {
        build_triangle_axis(chain[l - 1].width, chain[l].width, (filter & DXB_FILTER_WRAP_U) != 0, mp.tri[2 * (l - 1)]);
        build_triangle_axis(chain[l - 1].height, chain[l].height, (filter & DXB_FILTER_WRAP_V) != 0, mp.tri[2 * (l - 1) + 1]);
    }
    return mp;
}

// ---- ScaleMipMapsAlphaForCoverage ----------------------------------------------------------------
int32_t plan_alpha_coverage(const dxb200_image* src, size_t n, const dxb200_image* dst)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = src[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                         // :3495-3497
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != fmt || dst[i].format != fmt) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height || !src[i].width || !src[i].height) return DXB_E_INVALIDARG;
        if ((uint64_t)src[i].width * src[i].height > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    }
    return DXB_S_OK;
}

// CalculateAlphaCoverage's result (DirectXTexMipmaps.cpp:300-304): `count` covered samples of the 8x8 samples in each of the
// (w - 1)(h - 1) cells of 2x2 pixels; 0 for an image without a cell
float alpha_coverage_fraction(uint64_t count, size_t w, size_t h)
{
    const float cscale = static_cast<float>((w - 1) * (h - 1) * 8 * 8);
    return cscale > 0.0f ? static_cast<float>(count) / cscale : 0.0f;
}

// EstimateAlphaScaleForCoverage (:310-355): bisection on [0, 4], at most 10 coverage evaluations.  coverage(scale, &cov)
// returns an HRESULT; anything but S_OK stops the search and is returned.
template <typename CoverageFn>
int32_t estimate_alpha_scale(float target, CoverageFn coverage, float* scale)
{
    float lo = 0.0f, hi = 4.0f, s = 1.0f;
    for (int it = 0; it < 10; ++it)
    {
        float cov = 0.0f;
        const int32_t hr = coverage(s, &cov);
        if (hr != DXB_S_OK) return hr;
        if (cov < target) lo = s;
        else if (cov > target) hi = s;
        else break;
        s = (lo + hi) * 0.5f;
    }
    *scale = s;
    return DXB_S_OK;
}

} // namespace
