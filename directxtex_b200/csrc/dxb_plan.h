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
#include "dxb_coverage.h"
#include "dxb_alpha_opaque.h"
#include "dxb_channel_steps.h"

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

// The kernels move whole blocks with 8- or 16-byte loads and stores, so every block row of a BC image they touch must start on a
// multiple of the block size.  Host images are staged into 256-byte aligned device buffers at the caller's row pitch, so for them
// only the row pitch matters (bc_pitch_ok, checked by every plan); a _device call also passes its pixel pointer straight to the
// kernel (bc_pointers_ok).  A layout that breaks the rule would fault the kernel; the call is refused with E_INVALIDARG instead.
bool bc_pitch_ok(const dxb200_image& im)
{
    const size_t bs = dxb_bc_block_bytes(im.format);
    return bs == 0 || im.rowPitch % bs == 0;
}

bool bc_pointers_ok(const dxb200_image* im, size_t n)
{
    for (size_t i = 0; i < n; ++i)
        if (const size_t bs = dxb_bc_block_bytes(im[i].format))
            if (reinterpret_cast<uintptr_t>(im[i].pixels) % bs) return false;
    return true;
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
        if (!bc_pitch_ok(dst[i])) return DXB_E_INVALIDARG;
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
        if (!bc_pitch_ok(src[i])) return DXB_E_INVALIDARG;
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

// EstimateAlphaScaleForCoverage (:310-355) driven step by step: coverage(scale, &cov) measures one step and returns an HRESULT;
// anything but S_OK stops the search and is returned.  The rule is dxb_coverage_replay's.
template <typename CoverageFn>
int32_t estimate_alpha_scale(float target, CoverageFn coverage, float* scale)
{
    float cov[DXB_COVERAGE_STEPS];
    const auto seen = [&](uint32_t i) { return cov[i]; };
    float s = 1.0f;
    for (uint32_t k = 0; k < DXB_COVERAGE_STEPS; ++k)
    {
        if (!dxb_coverage_replay(target, k, seen, &s)) break;
        const int32_t hr = coverage(s, &cov[k]);
        if (hr != DXB_S_OK) return hr;
        if (k + 1 == DXB_COVERAGE_STEPS) (void)dxb_coverage_replay(target, DXB_COVERAGE_STEPS, seen, &s);
    }
    *scale = s;
    return DXB_S_OK;
}

// The job table of a batched ScaleMipMapsAlphaForCoverage: chains[it * levels + l] = level l of item it (source), out[...] = where
// its result goes (the same images in a chain that is scaled in place).  Level 0 of every item comes first (job it), then the
// other levels item by item.  Every cell and scaled pixel of the batch must have a 32-bit index: E_INVALIDARG otherwise.
struct CoveragePlan { dxb_coverage_params P; std::vector<dxb_coverage_job> jobs; };

int32_t plan_coverage_jobs(const dxb200_image* chains, const dxb200_image* out, size_t items, size_t levels, float ref, CoveragePlan* cp)
{
    dxb_coverage_params& P = cp->P; memset(&P, 0, sizeof(P));
    P.format = chains[0].format; P.items = (uint32_t)items; P.njobs = (uint32_t)(items * levels); P.ref = ref;
    cp->jobs.assign(items * levels, dxb_coverage_job());
    uint64_t cells = 0, pixels = 0;
    for (size_t n = 0; n < items * levels; ++n)
    {
        const size_t it = n < items ? n : (n - items) / (levels - 1), l = n < items ? 0 : 1 + (n - items) % (levels - 1);
        const dxb200_image& s = chains[it * levels + l]; const dxb200_image& d = out[it * levels + l];
        dxb_coverage_job& j = cp->jobs[n];
        j.src = s.pixels; j.dst = d.pixels; j.srcPitch = s.rowPitch; j.dstPitch = d.rowPitch;
        j.width = (uint32_t)s.width; j.height = (uint32_t)s.height; j.item = (uint32_t)it; j.pad = 0;
        j.firstUnit = (uint32_t)cells; j.firstPixel = (uint32_t)pixels;
        cells += (uint64_t)(s.width - 1) * (s.height - 1);
        if (l) pixels += (uint64_t)s.width * s.height;
        if (cells > 0xFFFFFFFFull || pixels > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
        if (n + 1 == items) P.baseCells = (uint32_t)cells;
    }
    P.totalCells = (uint32_t)cells; P.scaledPixels = (uint32_t)pixels;
    return DXB_S_OK;
}

// ---- GenerateMipMaps -> ScaleMipMapsAlphaForCoverage -> PremultiplyAlpha -> [Compress] in one call (mipmaps_compress) ------------
// chain = the chain every item will have on the device: for a compressed output, the ScratchImage layout of the source format (level
// 0 at the caller's pitch, its pixels the upload source; the other levels carry base[i].pixels only for validation); for an
// uncompressed output (compressed == false), the caller's dst itself.  generate == false (levels_from): the items keep the levels
// they came with, so GenerateMipMaps and coverage do not run and every level goes through the steps in front of them.
struct ChainPlan
{
    std::vector<dxb200_image> chain;
    bool generate = true; uint32_t mode;
    bool coverage; float ref;
    bool premultiply; dxb_convert_params pm;
    bool layout; dxb_convert_params lp;         // texconv's BC3n / RXGB layout, after premultiply
    bool compressed; CompressPlan compress;
};

// ---- texconv's -alpha and BC3n / RXGB steps (dxb200_texconv_steps) --------------------------------------------------------------
// The _ex calls' own rules, checked before any other: a layout other than 1 or 2, or a layout into anything but BC3_UNORM (texconv
// asserts it, :3556) or from a call with no BC target, is E_INVALIDARG.
int32_t check_texconv_steps(const dxb200_texconv_steps* ts, uint32_t dstFormat, bool bcTarget)
{
    if (!ts) return DXB_S_OK;
    if (ts->bc3Layout > 2) return DXB_E_INVALIDARG;
    if (ts->bc3Layout && (!bcTarget || dstFormat != DXB_FMT_BC3_UNORM)) return DXB_E_INVALIDARG;
    return DXB_S_OK;
}

uint32_t bc3_layout(const dxb200_texconv_steps* ts) { return ts ? ts->bc3Layout : 0u; }

// The layout as TransformImage channel steps: DXT5nm is XMVectorPermute<4,1,5,0>(p, g_XMIdentityR0) = (1, y, 0, x), RXGB is
// XMVectorSwizzle<3,1,2,0> = (a, g, b, r) (Texconv/texconv.cpp:3566-3595)
dxb200_channel_steps bc3_layout_steps(uint32_t layout)
{
    dxb200_channel_steps s = { { 3, 1, 2, 0 }, 0, 0, 0, 0, 0, 0 };
    if (layout == 1) { s.swizzle[0] = 0; s.zeroMask = 0x4; s.oneMask = 0x1; }
    return s;
}

int32_t plan_channel_steps(const dxb200_image* src, size_t n, const dxb200_channel_steps* steps, const dxb200_image* dst, dxb_convert_params* P);

// GenerateMipMaps (when cp->generate), then the optional coverage and premultiply steps of `steps` and the BC3 layout, on cp->chain,
// with the HRESULT of the first of those calls that would fail
int32_t plan_chain_steps(size_t items, size_t levels, uint32_t filter, const dxb200_chain_steps* steps, ChainPlan* cp, uint32_t layout = 0)
{
    const dxb200_image* chain = cp->chain.data();
    int32_t hr = DXB_S_OK;
    if (cp->generate && (hr = plan_mips(chain, items, levels, filter, &cp->mode)) != DXB_S_OK) return hr;
    cp->ref = steps ? steps->alphaReference : 0.0f;
    cp->coverage = cp->ref > 0.0f;                                                      // texconv -keepcoverage (:3304)
    if (cp->coverage && (hr = plan_alpha_coverage(chain, items * levels, chain)) != DXB_S_OK) return hr;
    cp->premultiply = steps && steps->premultiply;
    if (cp->premultiply && (hr = plan_pmalpha(chain, items * levels, steps->pmalphaFlags, chain, &cp->pm)) != DXB_S_OK) return hr;
    cp->layout = layout != 0;
    const dxb200_channel_steps ls = bc3_layout_steps(layout);
    if (cp->layout && (hr = plan_channel_steps(chain, items * levels, &ls, chain, &cp->lp)) != DXB_S_OK) return hr;
    return DXB_S_OK;
}

// Every check of the four steps (and the BC3 layout before Compress) before anything is uploaded, each with the HRESULT the
// reference's calls would return at the first step that fails; steps == nullptr (or no step enabled) = GenerateMipMaps + Compress.
int32_t plan_mipmaps_compress(const dxb200_image* base, size_t items, size_t levels, uint32_t filter, const dxb200_chain_steps* steps,
                              uint32_t dstFormat, uint32_t flags, float threshold, const dxb200_image* dst, ChainPlan* cp, uint32_t layout = 0)
{
    if (!base || !dst || !items || !levels) return DXB_E_INVALIDARG;
    std::vector<dxb200_image>& chain = cp->chain;
    chain.resize(items * levels);
    for (size_t i = 0; i < items; ++i)
    {
        size_t w = base[i].width, h = base[i].height;
        if (!base[i].pixels) return DXB_E_POINTER;
        if (levels > count_mips(w, h)) return DXB_E_INVALIDARG;
        for (size_t l = 0; l < levels; ++l)
        {
            dxb200_image& c = chain[i * levels + l];
            c.width = w; c.height = h; c.format = base[i].format;
            const int32_t hp = compute_pitch(c.format, w, h, &c.rowPitch, &c.slicePitch);
            if (hp != DXB_S_OK) return hp;
            c.pixels = const_cast<uint8_t*>(base[i].pixels);
            if (h > 1) h >>= 1;
            if (w > 1) w >>= 1;
        }
        chain[i * levels].rowPitch = base[i].rowPitch; chain[i * levels].slicePitch = base[i].slicePitch;
    }
    const int32_t hr = plan_chain_steps(items, levels, filter, steps, cp, layout);
    if (hr != DXB_S_OK) return hr;
    cp->compressed = true;
    return plan_compress(chain.data(), items * levels, dstFormat, flags, threshold, dst, &cp->compress);
}

// ---- texconv's channel steps (TransformImage, DirectXTexMisc.cpp:606-760; the rule in dxb_channel_steps.h) ------------------------
// the step word of `s`: 0 when no step is enabled (the swizzle is enabled unless it is the identity with both masks 0)
uint32_t channel_steps_word(const dxb200_channel_steps& s)
{
    uint32_t w = 0;
    for (uint32_t c = 0; c < 4; ++c) w |= (uint32_t)(s.swizzle[c] & 3u) << (DXB_CH_SWIZZLE_SHIFT + 2u * c);
    w |= (uint32_t)(s.zeroMask & 0xFu) << DXB_CH_ZERO_SHIFT | (uint32_t)(s.oneMask & 0xFu) << DXB_CH_ONE_SHIFT;
    if (s.swizzle[0] != 0 || s.swizzle[1] != 1 || s.swizzle[2] != 2 || s.swizzle[3] != 3 || s.zeroMask || s.oneMask) w |= DXB_CH_SWIZZLE;
    if (s.colorKey) w |= DXB_CH_COLOR_KEY;
    if (s.invertY) w |= DXB_CH_INVERT_Y;
    if (s.reconstructZ) w |= DXB_CH_RECONSTRUCT_Z;
    return (w & DXB_CH_STEPS) ? w : 0u;
}

// TransformImage's checks in its order (:646-701, TransformImage_ :220-227), then this library's: the steps stand in for the
// reference's pixelFunc, so none enabled is its null function (E_INVALIDARG, checked where TransformImage_ checks it, on image 0).
// P = the k_convert launch that runs them (srcFormat == dstFormat selects the steps).
int32_t plan_channel_steps(const dxb200_image* src, size_t n, const dxb200_channel_steps* steps, const dxb200_image* dst, dxb_convert_params* P)
{
    if (!src || !dst || !steps || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = src[0].format;
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;            // compressed, typeless, planar, palettized, other (:649)
    if (src[0].width > 0xFFFFFFFFull || src[0].height > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    const uint32_t word = channel_steps_word(*steps);
    const bool valid = word && steps->swizzle[0] < 4 && steps->swizzle[1] < 4 && steps->swizzle[2] < 4 && steps->swizzle[3] < 4
                    && !(steps->zeroMask & 0xF0u) && !(steps->oneMask & 0xF0u);
    for (size_t i = 0; i < n; ++i)
    {
        if (src[i].format != fmt || src[i].width > 0xFFFFFFFFull || src[i].height > 0xFFFFFFFFull) return DXB_E_FAIL;     // :683-693
        if (dst[i].format != fmt || dst[i].width != src[i].width || dst[i].height != src[i].height) return DXB_E_FAIL;  // :697, :226
        if (i == 0 && !valid) return DXB_E_INVALIDARG;                                                                 // :220
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;                                                     // :223
    }
    memset(P, 0, sizeof(*P));
    P->srcFormat = P->dstFormat = fmt; P->inF = P->outF = dxb_convert_flags(fmt);
    P->steps = word | ((dxb_convert_flags(fmt) & DXB_CONVF_UNORM) ? DXB_CH_UNORM : 0u);         // isunorm (:3252)
    dxb_color_key_vector(steps->colorKeyValue, P->key);
    return DXB_S_OK;
}

// The format texconv decompresses a BC base to when channel steps or a BC3 layout follow (:2393-2447): BC4 and BC5 hold one and two
// channels, so a step that reads or writes another channel, or a layout (dxt5nm || dxt5rxgb), needs R8G8B8A8 (UNORM or SNORM as the
// BC format); otherwise DefaultDecompress.
uint32_t channel_decompress_format(uint32_t bcFormat, const dxb200_channel_steps* s, uint32_t layout = 0)
{
    const uint32_t def = dxb_default_decompress(bcFormat);
    const bool bc4 = bcFormat == DXB_FMT_BC4_UNORM || bcFormat == DXB_FMT_BC4_SNORM, bc5 = bcFormat == DXB_FMT_BC5_UNORM || bcFormat == DXB_FMT_BC5_SNORM;
    const bool ch = s && channel_steps_word(*s);
    if ((!ch && !layout) || (!bc4 && !bc5)) return def;
    bool wide = layout != 0;
    if (ch) wide |= s->reconstructZ || (bc4 && s->invertY);
    for (uint32_t c = bc4 ? 1u : 2u; c < 4 && ch; ++c) wide |= s->swizzle[c] != c || ((s->zeroMask | s->oneMask) >> c & 1u);
    if (!wide) return def;
    return (bcFormat == DXB_FMT_BC4_SNORM || bcFormat == DXB_FMT_BC5_SNORM) ? DXB_FMT_R8G8B8A8_SNORM : DXB_FMT_R8G8B8A8_UNORM;
}

// ---- IsAlphaAllOpaque (DirectXTexImage.cpp:800-852; IsAlphaAllOpaqueBC, DirectXTexCompress.cpp:539-621) ---------------------
// The reference's answer comes without a device when scan == false: a format without alpha is opaque, nothing is read.  Otherwise
// every texel of every image has to be scanned: BC1 / BC2 / BC3 / BC7 blocks on k_decompress (blocks), any other implemented
// format with alpha on k_convert.  Images of one call share one format; a null pixel pointer is E_POINTER whatever the format.
struct AlphaOpaquePlan { bool scan, blocks; uint32_t format; };

int32_t plan_alpha_opaque(const dxb200_image* images, size_t n, const int32_t* opaque, AlphaOpaquePlan* ap)
{
    ap->scan = ap->blocks = false; ap->format = 0;
    if (!images || !opaque || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = images[0].format;
    for (size_t i = 0; i < n; ++i)
    {
        if (images[i].format != fmt) return DXB_E_INVALIDARG;
        if (!images[i].pixels) return DXB_E_POINTER;
    }
    if (!dxb_has_alpha(fmt)) return DXB_S_OK;                                            // :805-806, no pixel is read
    const bool blocks = is_compressed(fmt);
    if (blocks ? !dxb_alpha_scan_blocks(fmt) : !is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        const dxb200_image& im = images[i];
        if (!im.width || !im.height || im.width > 0xFFFFFFFFull || im.height > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
        if (!bc_pitch_ok(im)) return DXB_E_INVALIDARG;                                  // the rules of Decompress
    }
    ap->scan = true; ap->blocks = blocks; ap->format = fmt;
    return DXB_S_OK;
}

// the parameters of the scan's launch over `units` work units of `njobs` jobs (dxb_alpha_opaque.h)
dxb_compress_params alpha_opaque_block_params(const AlphaOpaquePlan& ap, uint32_t units, uint32_t njobs)
{
    dxb_compress_params P; memset(&P, 0, sizeof(P));
    P.srcFormat = ap.format; P.dstFormat = DXB_SCAN_ALPHA_OPAQUE; P.inF = dxb_convert_flags(ap.format);
    P.totalUnits = units; P.njobs = njobs;
    return P;
}
dxb_convert_params alpha_opaque_pixel_params(const AlphaOpaquePlan& ap, uint32_t units, uint32_t njobs)
{
    dxb_convert_params P; memset(&P, 0, sizeof(P));
    P.srcFormat = ap.format; P.dstFormat = DXB_SCAN_ALPHA_OPAQUE; P.inF = dxb_convert_flags(ap.format);
    P.totalUnits = units; P.njobs = njobs;
    return P;
}

// ---- what one chunk of a one-call pipeline stages and runs (run_chains) ------------------------------------------------------------
// How one image of a staged item travels: its host pixels go up before the launch, its device result comes back after the
// launch, or its bytes are only reserved in device memory (the levels of a chain that is compressed where it is built).
enum class Copy : uint8_t { Up, Down, None };

// The images a chunk can stage per item, one plane each: the caller's base, the decompressed image, level 0 in front of a Convert,
// the chain, the caller's dst and the alpha scan's result word
enum class PlaneRole : uint8_t { Base, Decompressed, Level0, Chain, Dst, Words };
constexpr size_t PLANE_ROLES = 6;

struct ChunkPlane { PlaneRole role; size_t per; Copy first, rest; };      // per = images per item; image 0 of an item travels as first

// One kind per launch site of run_chains: Channels = the channel steps (with a Convert: the swizzle), Post = those after the Convert
enum class StepKind : uint8_t { Decompress, Demultiply, Resize, BaseCopy, Channels, Convert, Post, Mips, Coverage, Premultiply, Layout,
                                Compress, Scan };

// The images of a plane a step covers: Front = the items' level 0 (every level when the items keep their levels), All = every
// image, PerLevel = level l of every item, one launch per level
enum class StepCover : uint8_t { Front, All, PerLevel };

struct ChunkStep { StepKind kind; PlaneRole src, dst; StepCover cover; };

struct ChunkPlan
{
    std::vector<ChunkPlane> planes;             // in the order the chunk's buffer holds them
    std::vector<ChunkStep> steps;               // in texconv's order
    size_t per;                                 // images per item a Front step covers: 1, or every level when the items keep theirs
    uint32_t filter;                            // GenerateMipMaps' filter
    std::vector<size_t> weight;                 // the bytes of each item's level 0 in the chain: the share of the items per device
};

// ---- Decompress -> Resize -> [channel steps] -> [Convert] -> [channel steps] -> mips ... [Compress] in one call ----------------
// The per-item device images: base[i] (the caller's, BC or not, at its pitch), decompressed[i] (the base's size in the decompress
// format at compute_pitch; in the buffer only when a resize follows, else it is level0[i]), level0[i] (what the front steps leave,
// W x H at compute_pitch; the base when no front step runs), the chain and, for a compressed output, the blocks.  Images the device
// makes carry base[i].pixels only for validation.  Which of them a chunk stages and which steps read and write them: chunk.
struct FromPlan
{
    bool decompress, demultiply, resize, channels, convert, post;
    dxb_compress_params dp;                     // the Decompress
    dxb_convert_params dm;                      // -alpha: PremultiplyAlpha(REVERSE) of what the Decompress leaves, in place
    std::vector<dxb200_image> decompressed;
    uint32_t resizeFilter, resizeMode;          // the Resize
    std::vector<dxb200_image> level0;
    dxb_convert_params cp;                      // the channel steps (with a Convert: the swizzle and masks)
    dxb_convert_params cv;                      // the Convert
    dxb_convert_params pp;                      // colour key, invert Y and reconstruct Z after the Convert
    ChainPlan chain;
    ChunkPlan chunk;                            // plan_chunk's, once every check has passed
};

// The planners' last step: IsAlphaAllOpaque of dst (when alphaAllOpaque != nullptr), then the planes and steps of a chunk.  A
// front step (Decompress or Resize) leaves level 0 in the chain (L: the chain's plane, or dst's for an uncompressed output), or in
// level 0 in front of a Convert; without one, the base goes up where a step reads it, else the chain's level 0 does (up).
int32_t plan_chunk(const dxb200_image* dst, size_t items, size_t levels, uint32_t filter, const int32_t* alphaAllOpaque, FromPlan* fp,
                   AlphaOpaquePlan* ap)
{
    if (alphaAllOpaque)
        if (const int32_t hr = plan_alpha_opaque(dst, items * levels, alphaAllOpaque, ap)) return hr;
    const ChainPlan& cp = fp->chain;
    ChunkPlan& ck = fp->chunk;
    using R = PlaneRole;
    using S = StepKind;
    const bool front = fp->decompress || fp->resize, mid = fp->decompress && fp->resize, pre = front && fp->convert;
    const bool up = !front && cp.compressed;
    const R L = cp.compressed ? R::Chain : R::Dst;
    const R W = pre ? R::Level0 : fp->convert && !front ? R::Base : L;        // what the front steps write, the channel steps run on
    const R D = mid ? R::Decompressed : W;                                      // what the Decompress writes
    const R DM = fp->decompress ? D : up ? L : R::Base;                         // what the demultiply runs on
    const Copy chainUp = up ? Copy::Up : Copy::None;
    ck.per = cp.generate ? 1 : levels;
    ck.filter = filter;
    ck.planes.clear();
    if (!up) ck.planes.push_back({ R::Base, ck.per, Copy::Up, Copy::Up });
    if (mid) ck.planes.push_back({ R::Decompressed, ck.per, Copy::None, Copy::None });
    if (pre) ck.planes.push_back({ R::Level0, ck.per, Copy::None, Copy::None });
    if (cp.compressed) ck.planes.push_back({ R::Chain, levels, chainUp, cp.generate ? Copy::None : chainUp });
    ck.planes.push_back({ R::Dst, levels, Copy::Down, Copy::Down });
    if (ap->scan) ck.planes.push_back({ R::Words, 1, Copy::Down, Copy::Down });
    ck.steps.clear();
    const auto step = [&](bool on, S kind, R src, R dst, StepCover cover) { if (on) ck.steps.push_back({ kind, src, dst, cover }); };
    const StepCover F = StepCover::Front, A = StepCover::All;
    step(fp->decompress, S::Decompress, R::Base, D, F);
    step(fp->demultiply, S::Demultiply, DM, DM, F);
    step(fp->resize, S::Resize, mid ? R::Decompressed : R::Base, W, F);
    step(!up && !front && !fp->convert, S::BaseCopy, R::Base, L, F);
    step(fp->channels, S::Channels, W, W, F);
    step(fp->convert, S::Convert, W, L, F);
    step(fp->post, S::Post, L, L, F);
    step(cp.generate, S::Mips, L, L, A);
    step(cp.coverage, S::Coverage, L, L, A);
    step(cp.premultiply, S::Premultiply, L, L, cp.generate ? StepCover::PerLevel : F);
    step(cp.layout, S::Layout, L, L, A);
    step(cp.compressed, S::Compress, R::Chain, R::Dst, A);
    step(ap->scan, S::Scan, R::Dst, R::Words, A);
    ck.weight.resize(items);
    for (size_t i = 0; i < items; ++i) ck.weight[i] = cp.chain[i * levels].slicePitch;
    return DXB_S_OK;
}

// image i of `n` of format fmt, w x h, at compute_pitch, with the pixels of base[i]
std::vector<dxb200_image> plan_images(const dxb200_image* base, size_t n, uint32_t fmt, size_t w, size_t h)
{
    std::vector<dxb200_image> out(n);
    for (size_t i = 0; i < n; ++i)
    {
        dxb200_image& im = out[i];
        im.width = w ? w : base[i].width; im.height = h ? h : base[i].height; im.format = fmt; im.rowPitch = im.slicePitch = 0;
        (void)compute_pitch(fmt, im.width, im.height, &im.rowPitch, &im.slicePitch);      // a format no pitch exists for is refused below
        im.pixels = base[i].pixels;
    }
    return out;
}

// Decompress (a BC base, when source != nullptr), -alpha's demultiply (when ts->demultiply) and Resize (when the source's size
// differs) of the base, with the HRESULT of the first that would fail; fp->level0 = the images they leave.  With no decompress format,
// a BC4 / BC5 base decompresses to channel_decompress_format of the channel steps and the BC3 layout.
int32_t plan_front(const dxb200_image* base, size_t items, const dxb200_chain_source* source, const dxb200_channel_steps* channels, FromPlan* fp,
                   const dxb200_texconv_steps* ts = nullptr)
{
    fp->decompress = fp->demultiply = fp->resize = fp->channels = fp->convert = fp->post = false;
    fp->resizeFilter = fp->resizeMode = 0;
    fp->decompressed.clear();
    fp->level0.clear();
    if (source && (!source->width) != (!source->height)) return DXB_E_INVALIDARG;
    const size_t w = source && source->width ? source->width : base[0].width, h = source && source->height ? source->height : base[0].height;
    fp->decompress = source && is_compressed(base[0].format);
    fp->resize = (w != base[0].width || h != base[0].height);
    fp->level0.assign(base, base + items);
    int32_t hr = DXB_S_OK;
    if (fp->decompress)
    {
        const uint32_t fmt = source->decompressFormat ? source->decompressFormat : channel_decompress_format(base[0].format, channels, bc3_layout(ts));
        fp->decompressed = plan_images(base, items, fmt, 0, 0);
        if ((hr = plan_decompress(base, items, fmt, fp->decompressed.data(), &fp->dp)) != DXB_S_OK) return hr;
        fp->level0 = fp->decompressed;
    }
    // texconv's -alpha (:2483-2531); REVERSE is implied
    fp->demultiply = ts && ts->demultiply;
    if (fp->demultiply && (hr = plan_pmalpha(fp->level0.data(), items, 0x2u | ts->demultiplyFlags, fp->level0.data(), &fp->dm)) != DXB_S_OK)
        return hr;
    if (fp->resize)
    {
        const std::vector<dxb200_image> resized = plan_images(base, items, fp->level0[0].format, w, h);
        if ((hr = plan_resize(fp->level0.data(), items, source->resizeFilter, resized.data(), &fp->resizeMode)) != DXB_S_OK) return hr;
        fp->resizeFilter = source->resizeFilter;
        fp->level0 = resized;
    }
    return DXB_S_OK;
}

// Every check of Decompress, -alpha's demultiply, Resize, the channel steps and the steps of plan_mipmaps_compress before anything is
// uploaded, each with the HRESULT of the first of the separate calls that would fail; check_texconv_steps comes before all of them,
// IsAlphaAllOpaque of dst (when alphaAllOpaque != nullptr) after them.  source == nullptr, or a source that changes nothing,
// channels == nullptr, or no channel step enabled, and ts == nullptr, or all zeros = plan_mipmaps_compress.
int32_t plan_mipmaps_compress_channels(const dxb200_image* base, size_t items, const dxb200_chain_source* source, const dxb200_channel_steps* channels,
                                       size_t levels, uint32_t filter, const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags,
                                       float threshold, const dxb200_image* dst, FromPlan* fp, const dxb200_texconv_steps* ts = nullptr,
                                       const int32_t* alphaAllOpaque = nullptr, AlphaOpaquePlan* ap = nullptr)
{
    AlphaOpaquePlan none;
    if (!ap) ap = &none;
    ap->scan = ap->blocks = false; ap->format = 0;
    fp->decompress = fp->demultiply = fp->resize = fp->channels = fp->convert = fp->post = false;
    fp->resizeFilter = fp->resizeMode = 0;
    fp->decompressed.clear();
    int32_t hr = check_texconv_steps(ts, dstFormat, true);
    if (hr != DXB_S_OK) return hr;
    const bool ch = channels && channel_steps_word(*channels);
    const dxb200_image* level0 = base;
    if ((!source && !ch && !(ts && ts->demultiply)) || !base || !items)
        fp->level0.clear();
    else
    {
        if ((hr = plan_front(base, items, source, channels, fp, ts)) != DXB_S_OK) return hr;
        if (ch && (hr = plan_channel_steps(fp->level0.data(), items, channels, fp->level0.data(), &fp->cp)) != DXB_S_OK) return hr;
        fp->channels = ch;
        level0 = fp->level0.data();
    }
    if ((hr = plan_mipmaps_compress(level0, items, levels, filter, steps, dstFormat, flags, threshold, dst, &fp->chain, bc3_layout(ts))) != DXB_S_OK)
        return hr;
    return plan_chunk(dst, items, levels, filter, alphaAllOpaque, fp, ap);
}

int32_t plan_mipmaps_compress_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source, size_t levels, uint32_t filter,
                                   const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags, float threshold, const dxb200_image* dst,
                                   FromPlan* fp)
{
    return plan_mipmaps_compress_channels(base, items, source, nullptr, levels, filter, steps, dstFormat, flags, threshold, dst, fp);
}

// ---- the channel steps around a Convert ------------------------------------------------------------------------------------------
// texconv runs the swizzle and masks of `channels` before its Convert (:2645-2694) and the colour key, invert Y and reconstruct Z
// after it (:3134-3300); nothing enabled in either when channels == nullptr
void split_channel_steps(const dxb200_channel_steps* channels, dxb200_channel_steps* swizzle, dxb200_channel_steps* later)
{
    *swizzle = { { 0, 1, 2, 3 }, 0, 0, 0, 0, 0, 0 };
    *later = *swizzle;
    if (!channels) return;
    memcpy(swizzle->swizzle, channels->swizzle, 4); swizzle->zeroMask = channels->zeroMask; swizzle->oneMask = channels->oneMask;
    later->colorKey = channels->colorKey; later->colorKeyValue = channels->colorKeyValue;
    later->invertY = channels->invertY; later->reconstructZ = channels->reconstructZ;
}

// Without a Convert, out[i] takes the working image work[i] as it is: the same format and size (E_INVALIDARG, as a BC row pitch the
// kernels cannot read), and pixels (E_POINTER)
int32_t plan_unconverted(const dxb200_image* work, size_t n, const dxb200_image* out)
{
    for (size_t i = 0; i < n; ++i)
    {
        if (out[i].format != work[0].format || out[i].width != work[i].width || out[i].height != work[i].height || !bc_pitch_ok(out[i]))
            return DXB_E_INVALIDARG;
        if (!out[i].pixels) return DXB_E_POINTER;
    }
    return DXB_S_OK;
}

// The images levels_from only copies into dst (no step reads them, or only the channel steps, which check neither size nor
// bounds): one format this library implements (E_NOT_SUPPORTED otherwise, as every other call answers, since its pitch is
// unknown), non-NULL pixels (E_POINTER), a size of 1 to 2^32 - 1 in both directions and a BC row pitch of whole blocks
// (E_INVALIDARG)
int32_t plan_copy(const dxb200_image* src, size_t n)
{
    const uint32_t fmt = src[0].format;
    if (!is_compressed(fmt) && !is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        if (src[i].format != fmt) return DXB_E_INVALIDARG;
        if (!src[i].pixels) return DXB_E_POINTER;
        if (!src[i].width || !src[i].height || src[i].width > 0xFFFFFFFFull || src[i].height > 0xFFFFFFFFull || !bc_pitch_ok(src[i]))
            return DXB_E_INVALIDARG;
    }
    return DXB_S_OK;
}

// Without a Convert between them, the swizzle (fp->cp, when fp->channels) and the later steps (fp->pp) run as one launch: the step
// word's flags say which steps run, each in texconv's order on the previous one's stored result
void merge_channel_launches(FromPlan* fp)
{
    const uint32_t sw = fp->channels ? fp->cp.steps & (0xFFFFu | DXB_CH_SWIZZLE) : 0u;
    fp->cp = fp->pp;
    fp->cp.steps = (fp->pp.steps & ~0xFFFFu) | sw;
    fp->channels = true; fp->post = false;
}

// ---- Decompress -> Resize -> swizzle -> Convert -> later channel steps -> mips -> coverage -> premultiply in one call --------------
// (mipmaps_convert_from) texconv's path to an uncompressed target (Texconv/texconv.cpp:2316-3560).  Every check of the nine
// separate calls before anything is uploaded, each with the HRESULT of the first that would fail: plan_front; the swizzle and
// masks of `channels` on level 0's format; Convert to dstFormat into level 0 of dst, only when level 0's format differs (texconv
// tests info.format != tformat; a BC dstFormat always goes through Convert's checks, E_INVALIDARG); colour key, invert Y and
// reconstruct Z on dst's level 0; GenerateMipMaps, coverage and premultiply on dst (plan_chain_steps); IsAlphaAllOpaque of dst
// when alphaAllOpaque != nullptr.  Without a Convert, dst's level 0 must have level 0's format and size (E_INVALIDARG), the later
// steps are checked from level 0 into dst's level 0, GenerateMipMaps on a chain whose level 0 is level 0 (every base's pixels and
// format, when no front step runs), and the two groups of channel steps run as one launch, as dxb200_mipmaps_compress_from_channels
// runs them.  levels < 2 is GenerateMipMaps' E_INVALIDARG, after the Convert's checks.
int32_t plan_mipmaps_convert_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source, const dxb200_channel_steps* channels,
                                  uint32_t dstFormat, uint32_t convertFilter, float threshold, size_t levels, uint32_t filter,
                                  const dxb200_chain_steps* steps, const dxb200_image* dst, const int32_t* alphaAllOpaque, FromPlan* fp,
                                  AlphaOpaquePlan* ap, const dxb200_texconv_steps* ts = nullptr)
{
    ap->scan = ap->blocks = false; ap->format = 0;
    int32_t hr = check_texconv_steps(ts, dstFormat, false);
    if (hr != DXB_S_OK) return hr;
    if (!base || !items) return DXB_E_INVALIDARG;
    if ((hr = plan_front(base, items, source, channels, fp, ts)) != DXB_S_OK) return hr;
    dxb200_channel_steps swizzle, later;
    split_channel_steps(channels, &swizzle, &later);
    fp->channels = channel_steps_word(swizzle) != 0;
    if (fp->channels && (hr = plan_channel_steps(fp->level0.data(), items, &swizzle, fp->level0.data(), &fp->cp)) != DXB_S_OK) return hr;
    if (!dst) return DXB_E_INVALIDARG;
    std::vector<dxb200_image>& chain = fp->chain.chain;
    chain.assign(dst, dst + items * levels);
    std::vector<dxb200_image> out0(items);
    for (size_t i = 0; i < items; ++i) out0[i] = dst[i * levels];         // levels == 0: dst[0], refused by GenerateMipMaps below
    fp->convert = fp->level0[0].format != dstFormat || is_compressed(dstFormat);
    if (fp->convert)
    {
        if ((hr = plan_convert(fp->level0.data(), items, dstFormat, convertFilter, out0.data(), &fp->cv)) != DXB_S_OK) return hr;
        fp->cv.threshold = threshold;
    }
    else if ((hr = plan_unconverted(fp->level0.data(), items, out0.data())) != DXB_S_OK)
        return hr;
    // without a Convert the later steps read level 0 as the front steps leave it (the base when none runs) and write dst's level 0
    fp->post = channel_steps_word(later) != 0;
    if (fp->post && (hr = plan_channel_steps(fp->convert ? out0.data() : fp->level0.data(), items, &later, out0.data(), &fp->pp)) != DXB_S_OK)
        return hr;
    if (!fp->convert && fp->post) merge_channel_launches(fp);
    // without a Convert, GenerateMipMaps meets a chain whose level 0 is that image: its pixels and format are checked there
    for (size_t i = 0; i < items && levels && !fp->convert; ++i) chain[i * levels] = fp->level0[i];
    if ((hr = plan_chain_steps(items, levels, filter, steps, &fp->chain)) != DXB_S_OK) return hr;
    for (size_t i = 0; i < items && levels; ++i) chain[i * levels] = dst[i * levels];
    fp->chain.compressed = false;
    return plan_chunk(dst, items, levels, filter, alphaAllOpaque, fp, ap);
}

// ---- texconv on items that keep their own levels (levels_from): Decompress -> [Resize] -> swizzle -> Convert -> later channel steps
// -> premultiply -> Compress -> IsAlphaAllOpaque, each over the items * levels images as one array ---------------------------------
// texconv keeps the input's chain when -m is not given (Texconv/texconv.cpp:2270) and makes none for -m 1, so neither the strip
// (:3325) nor GenerateMipMaps (:3419) runs.  The call's own rules come first: levels == 0, a Resize with levels > 1 (texconv's Resize
// drops the chain) and alphaReference > 0 (-keepcoverage regenerates the chain, :3325) are E_INVALIDARG.  Then every check of the
// separate calls in their order, each on the format and size the images have at that point: plan_front on all the images (a BC base
// is decompressed whatever the source); the swizzle and masks in place; Convert into dst for an uncompressed dstFormat other than the
// working format (texconv's test, :3098), else dst must be the working images (plan_unconverted); the later channel steps;
// premultiply (plan_chain_steps with generate off); Compress into dst for a BC dstFormat; IsAlphaAllOpaque of dst.  A BC base whose
// dstFormat is its own format, with no channel step, no premultiply and no Resize, passes through (texconv :3621): its Decompress is
// checked, as texconv makes it before it decides, but does not run; dst takes the base's bytes.  When the base is copied into dst
// (no front step, no Convert, no Compress), plan_copy checks it last.
int32_t plan_levels_from(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                         const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, uint32_t compressFlags,
                         float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst, const int32_t* alphaAllOpaque,
                         FromPlan* fp, AlphaOpaquePlan* ap, const dxb200_texconv_steps* ts = nullptr)
{
    ap->scan = ap->blocks = false; ap->format = 0;
    int32_t hr = check_texconv_steps(ts, dstFormat, true);
    if (hr != DXB_S_OK) return hr;
    if (!base || !items || !levels) return DXB_E_INVALIDARG;
    const size_t n = items * levels;
    const dxb200_chain_source keep = { 0, 0, 0, 0 };
    const dxb200_chain_source* src = source ? source : &keep;
    if (levels > 1 && ((src->width && src->width != base[0].width) || (src->height && src->height != base[0].height))) return DXB_E_INVALIDARG;
    if (steps && steps->alphaReference > 0.0f) return DXB_E_INVALIDARG;
    if ((hr = plan_front(base, n, src, channels, fp, ts)) != DXB_S_OK) return hr;
    ChainPlan& cp = fp->chain;
    cp.generate = false; cp.mode = 0;
    dxb200_channel_steps swizzle, later;
    split_channel_steps(channels, &swizzle, &later);
    const bool pass = is_compressed(base[0].format) && dstFormat == base[0].format && !channel_steps_word(swizzle) && !channel_steps_word(later)
                      && !(steps && steps->premultiply) && !fp->resize && !fp->demultiply && !bc3_layout(ts);
    if (pass)
    {
        fp->decompress = false;
        fp->decompressed.clear();
        fp->level0.assign(base, base + n);
    }
    fp->channels = channel_steps_word(swizzle) != 0;
    if (fp->channels && (hr = plan_channel_steps(fp->level0.data(), n, &swizzle, fp->level0.data(), &fp->cp)) != DXB_S_OK) return hr;
    // a compressed output is compressed from the working images, so the later steps and premultiply run in place on them
    cp.compressed = is_compressed(dstFormat) && !pass;
    if (!cp.compressed && !dst) return DXB_E_INVALIDARG;
    const dxb200_image* out = cp.compressed ? fp->level0.data() : dst;
    fp->convert = !is_compressed(dstFormat) && fp->level0[0].format != dstFormat;
    if (fp->convert)
    {
        if ((hr = plan_convert(fp->level0.data(), n, dstFormat, convertFilter, dst, &fp->cv)) != DXB_S_OK) return hr;
        fp->cv.threshold = threshold;
    }
    else if (!cp.compressed && (hr = plan_unconverted(fp->level0.data(), n, out)) != DXB_S_OK)
        return hr;
    fp->post = channel_steps_word(later) != 0;
    if (fp->post && (hr = plan_channel_steps(fp->convert ? out : fp->level0.data(), n, &later, out, &fp->pp)) != DXB_S_OK) return hr;
    if (!fp->convert && fp->post) merge_channel_launches(fp);
    cp.chain.assign(out, out + n);
    if ((hr = plan_chain_steps(items, levels, 0, steps, &cp, bc3_layout(ts))) != DXB_S_OK) return hr;
    if (cp.compressed && (hr = plan_compress(out, n, dstFormat, compressFlags, threshold, dst, &cp.compress)) != DXB_S_OK) return hr;
    const bool copy = !fp->decompress && !fp->resize && !fp->convert && !cp.compressed;
    if (copy && (hr = plan_copy(base, n)) != DXB_S_OK) return hr;
    return plan_chunk(dst, items, levels, 0, alphaAllOpaque, fp, ap);
}

} // namespace
