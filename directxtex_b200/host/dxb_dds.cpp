// dxb_dds.cpp — the DDS container either side of the hot path (SURVEY 8(f) rank 3): header encode / decode and
// image (de)serialisation for the formats this library implements.  Host-only code, no CUDA.
//
// Replaces (reference, all in DirectXTex/DirectXTexDDS.cpp): EncodeDDSHeader :711-1043, DecodeDDSHeader :319-683 +
// GetDXGIFormat :184-317 (the legacy subset listed below), SaveToDDSMemory :2403-2620, LoadFromDDSMemory :2008-2100 +
// CopyImage :1505-1780 (no-conversion path only).  File layout: DDS.h:28-300.
//
// Scope: TEXTURE2D resources (single images, arrays, cubemaps, mip chains).  Legacy (pre-DX10) pixel formats are
// written exactly where the reference writes them and read back when they map 1:1 onto a DXGI format; legacy formats
// that need expansion (palettes, 24 bpp, 3:3:2, ...), 1D / 3D resources, DDS_FLAGS_FORCE_DX9_LEGACY and the other
// conversion flags return HRESULT_E_NOT_SUPPORTED.
#include <cstdint>
#include <cstring>
#include "../../include/dxtex_b200.h"
#include "../csrc/dxb_formats.h"

namespace {

constexpr uint32_t fourcc(char a, char b, char c, char d)
{
    return (uint32_t)(uint8_t)a | ((uint32_t)(uint8_t)b << 8) | ((uint32_t)(uint8_t)c << 16) | ((uint32_t)(uint8_t)d << 24);
}

#pragma pack(push, 1)
struct PixelFormat { uint32_t size, flags, fourCC, bitCount, rMask, gMask, bMask, aMask; };           // DDS.h:33-43
struct Header                                                                                        // DDS.h:231-248
{
    uint32_t size, flags, height, width, pitchOrLinearSize, depth, mipMapCount, reserved1[11];
    PixelFormat ddspf;
    uint32_t caps, caps2, caps3, caps4, reserved2;
};
struct HeaderDX10 { uint32_t dxgiFormat, resourceDimension, miscFlag, arraySize, miscFlags2; };       // DDS.h:250-257
#pragma pack(pop)
static_assert(sizeof(PixelFormat) == 32 && sizeof(Header) == 124 && sizeof(HeaderDX10) == 20, "DDS header layout");

constexpr uint32_t kMagic = 0x20534444u;                              // "DDS "
constexpr size_t kMinHeader = 4 + sizeof(Header), kDX10Header = kMinHeader + sizeof(HeaderDX10);
// ddpf.flags
constexpr uint32_t PF_FOURCC = 0x4, PF_RGB = 0x40, PF_RGBA = 0x41, PF_LUM = 0x20000, PF_LUMA = 0x20001, PF_ALPHA = 0x2, PF_BUMPDUDV = 0x80000;
// header.flags / caps / caps2
constexpr uint32_t HF_TEXTURE = 0x1007, HF_MIPMAP = 0x20000, HF_VOLUME = 0x800000, HF_PITCH = 0x8, HF_LINEARSIZE = 0x80000;
constexpr uint32_t CAPS_TEXTURE = 0x1000, CAPS_MIPMAP = 0x400008, CAPS_CUBEMAP = 0x8;
constexpr uint32_t CAPS2_CUBEMAP = 0x200, CAPS2_ALLFACES = 0xFE00;
// DDS_FLAGS (DirectXTex.h:232-279) that this implementation understands
constexpr uint32_t DF_FORCE_DX10 = 0x10000, DF_FORCE_DX10_MISC2 = 0x20000, DF_ALLOW_LARGE = 0x1000000, DF_IGNORE_MIPS = 0x100;
constexpr uint32_t DF_FORCE_DX9 = 0x40000, DF_FORCE_RXGB = 0x80000;
// load-side conversion flags (LEGACY_DWORD, NO_LEGACY_EXPANSION, NO_R10B10G10A2_FIXUP, FORCE_RGB, NO_16BPP, EXPAND_LUMINANCE,
// BAD_DXTN_TAILS, PERMISSIVE) and FORCE_24BPP_RGB are outside this implementation
constexpr uint32_t DF_UNSUPPORTED = 0x1 | 0x2 | 0x4 | 0x8 | 0x10 | 0x20 | 0x40 | 0x80 | 0x100000;
constexpr uint32_t MISC_TEXTURECUBE = 0x4;

// one row per legacy encoding the reference emits for a format this library implements (EncodeDDSHeader :746-790);
// pm = only for premultiplied alpha metadata (DXT2 / DXT4); decodeOnly = accepted on load, never written
struct Legacy { uint32_t format; PixelFormat pf; bool pm, decodeOnly; };
constexpr PixelFormat FCC(uint32_t cc) { return { 32, PF_FOURCC, cc, 0, 0, 0, 0, 0 }; }
const Legacy kLegacy[] = {
    { DXB_FMT_R8G8B8A8_UNORM,     { 32, PF_RGBA, 0, 32, 0x000000ff, 0x0000ff00, 0x00ff0000, 0xff000000 }, false, false },
    { DXB_FMT_B8G8R8A8_UNORM,     { 32, PF_RGBA, 0, 32, 0x00ff0000, 0x0000ff00, 0x000000ff, 0xff000000 }, false, false },
    { DXB_FMT_B8G8R8X8_UNORM,     { 32, PF_RGB,  0, 32, 0x00ff0000, 0x0000ff00, 0x000000ff, 0 }, false, false },
    { DXB_FMT_R16G16_UNORM,       { 32, PF_RGB,  0, 32, 0x0000ffff, 0xffff0000, 0, 0 }, false, false },
    { DXB_FMT_B5G6R5_UNORM,       { 32, PF_RGB,  0, 16, 0xf800, 0x07e0, 0x001f, 0 }, false, false },                  // DDSPF_R5G6B5 (DDS.h:125)
    { DXB_FMT_B5G5R5A1_UNORM,     { 32, PF_RGBA, 0, 16, 0x7c00, 0x03e0, 0x001f, 0x8000 }, false, false },             // DDSPF_A1R5G5B5
    { DXB_FMT_B4G4R4A4_UNORM,     { 32, PF_RGBA, 0, 16, 0x0f00, 0x00f0, 0x000f, 0xf000 }, false, false },             // DDSPF_A4R4G4B4
    { DXB_FMT_R8G8_UNORM,         { 32, PF_LUMA, 0, 16, 0x00ff, 0, 0, 0xff00 }, false, false },
    { DXB_FMT_R16_UNORM,          { 32, PF_LUM,  0, 16, 0xffff, 0, 0, 0 }, false, false },
    { DXB_FMT_R8_UNORM,           { 32, PF_LUM,  0, 8, 0xff, 0, 0, 0 }, false, false },
    { DXB_FMT_A8_UNORM,           { 32, PF_ALPHA, 0, 8, 0, 0, 0, 0xff }, false, false },
    { DXB_FMT_R8G8_SNORM,         { 32, PF_BUMPDUDV, 0, 16, 0x00ff, 0xff00, 0, 0 }, false, false },
    { DXB_FMT_R8G8B8A8_SNORM,     { 32, PF_BUMPDUDV, 0, 32, 0x000000ff, 0x0000ff00, 0x00ff0000, 0xff000000 }, false, false },
    { DXB_FMT_R16G16_SNORM,       { 32, PF_BUMPDUDV, 0, 32, 0x0000ffff, 0xffff0000, 0, 0 }, false, false },
    { DXB_FMT_BC1_UNORM,          FCC(fourcc('D', 'X', 'T', '1')), false, false },
    { DXB_FMT_BC2_UNORM,          FCC(fourcc('D', 'X', 'T', '2')), true, false },
    { DXB_FMT_BC2_UNORM,          FCC(fourcc('D', 'X', 'T', '3')), false, false },
    { DXB_FMT_BC3_UNORM,          FCC(fourcc('D', 'X', 'T', '4')), true, false },
    { DXB_FMT_BC3_UNORM,          FCC(fourcc('D', 'X', 'T', '5')), false, false },
    { DXB_FMT_BC4_UNORM,          FCC(fourcc('B', 'C', '4', 'U')), false, false },
    { DXB_FMT_BC4_SNORM,          FCC(fourcc('B', 'C', '4', 'S')), false, false },
    { DXB_FMT_BC5_UNORM,          FCC(fourcc('B', 'C', '5', 'U')), false, false },
    { DXB_FMT_BC5_SNORM,          FCC(fourcc('B', 'C', '5', 'S')), false, false },
    { DXB_FMT_BC4_UNORM,          FCC(fourcc('A', 'T', 'I', '1')), false, true },
    { DXB_FMT_BC5_UNORM,          FCC(fourcc('A', 'T', 'I', '2')), false, true },
    // legacy D3DX files use the D3DFMT enum value as FourCC
    { DXB_FMT_R32G32B32A32_FLOAT, FCC(116), false, false }, { DXB_FMT_R16G16B16A16_FLOAT, FCC(113), false, false },
    { DXB_FMT_R16G16B16A16_UNORM, FCC(36), false, false },  { DXB_FMT_R16G16B16A16_SNORM, FCC(110), false, false },
    { DXB_FMT_R32G32_FLOAT,       FCC(115), false, false }, { DXB_FMT_R16G16_FLOAT, FCC(112), false, false },
    { DXB_FMT_R32_FLOAT,          FCC(114), false, false }, { DXB_FMT_R16_FLOAT, FCC(111), false, false },
};

bool format_ok(uint32_t f) { return dxb_bytes_per_pixel(f) != 0 || dxb_bc_block_bytes(f) != 0; }
bool is_pm(const dxb200_metadata& m) { return (m.miscFlags2 & 0x7u) == 2u; }

int32_t pitch(uint32_t fmt, size_t w, size_t h, size_t* row, size_t* slice) { return dxb200_compute_pitch(fmt, w, h, row, slice); }

} // namespace

extern "C" {

int32_t dxb200_dds_encode_header(const dxb200_metadata* md, uint32_t flags, void* dst, size_t maxsize, size_t* required)
{
    if (!md || !required) return DXB_E_INVALIDARG;
    if (!format_ok(md->format)) return DXB_E_NOT_SUPPORTED;
    if (flags & DF_UNSUPPORTED) return DXB_E_NOT_SUPPORTED;
    if (md->dimension != 3 /* TEX_DIMENSION_TEXTURE2D */ || md->depth != 1) return DXB_E_NOT_SUPPORTED;
    const bool cube = (md->miscFlags & MISC_TEXTURECUBE) != 0;
    // arrays other than a single cubemap need the DX10 extension (:728-738)
    if (md->arraySize > 1 && !(md->arraySize == 6 && cube))
    {
        if (flags & DF_FORCE_DX9) return (int32_t)0x80070052;
        flags |= DF_FORCE_DX10;
    }
    if (flags & DF_FORCE_DX10_MISC2) flags |= DF_FORCE_DX10;
    if ((flags & DF_FORCE_DX9) && (flags & DF_FORCE_DX10)) return (int32_t)0x80070052;      // HRESULT_E_CANNOT_MAKE (:733-734)
    const Legacy* leg = nullptr;
    PixelFormat legpf{};
    if (!(flags & DF_FORCE_DX10))
    {
        // DDS_FLAGS_FORCE_DX9_LEGACY writes the sRGB formats with their UNORM twins' legacy encodings and BC4U / BC5U as
        // ATI1 / ATI2 (:855-911); without a legacy encoding it fails with HRESULT_E_CANNOT_MAKE (:918-919)
        const uint32_t f = (flags & DF_FORCE_DX9) ? dxb_make_linear(md->format) : md->format;
        for (const Legacy& e : kLegacy)
            if (e.format == f && !e.decodeOnly && (!e.pm || is_pm(*md))) { leg = &e; break; }
        if (leg)
        {
            legpf = leg->pf;
            if ((flags & DF_FORCE_DX9) && md->format == DXB_FMT_BC4_UNORM) legpf.fourCC = fourcc('A', 'T', 'I', '1');
            if ((flags & DF_FORCE_DX9) && md->format == DXB_FMT_BC5_UNORM) legpf.fourCC = fourcc('A', 'T', 'I', '2');
            if ((flags & DF_FORCE_RXGB) && f == DXB_FMT_BC3_UNORM) legpf.fourCC = fourcc('R', 'X', 'G', 'B');      // :781-784
        }
        else if (flags & DF_FORCE_DX9)
        {
            if (md->format == DXB_FMT_R10G10B10A2_UNORM) return DXB_E_NOT_SUPPORTED;        // the D3DX-compatible mask variant is not implemented
            return (int32_t)0x80070052;
        }
    }
    *required = leg ? kMinHeader : kDX10Header;
    if (!dst) return DXB_S_OK;
    if (maxsize < *required) return (int32_t)0x8007007A;                   // E_NOT_SUFFICIENT_BUFFER
    if (md->mipLevels > 0xFFFFu || md->width > 0xFFFFFFFFull || md->height > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    uint8_t* p = static_cast<uint8_t*>(dst);
    memcpy(p, &kMagic, 4);
    Header h; memset(&h, 0, sizeof(h));
    h.size = sizeof(Header); h.flags = HF_TEXTURE; h.caps = CAPS_TEXTURE;
    if (md->mipLevels > 0)
    {
        h.flags |= HF_MIPMAP; h.mipMapCount = (uint32_t)md->mipLevels;
        if (h.mipMapCount > 1) h.caps |= CAPS_MIPMAP;
    }
    h.height = (uint32_t)md->height; h.width = (uint32_t)md->width; h.depth = 1;
    if (cube) { h.caps |= CAPS_CUBEMAP; h.caps2 |= CAPS2_ALLFACES; }
    size_t row = 0, slice = 0;
    int32_t hr = pitch(md->format, md->width, md->height, &row, &slice);
    if (hr != DXB_S_OK) return hr;
    if (row > 0xFFFFFFFFull || slice > 0xFFFFFFFFull) return DXB_E_FAIL;
    if (dxb_bc_block_bytes(md->format)) { h.flags |= HF_LINEARSIZE; h.pitchOrLinearSize = (uint32_t)slice; }
    else { h.flags |= HF_PITCH; h.pitchOrLinearSize = (uint32_t)row; }
    if (leg) h.ddspf = legpf;
    else
    {
        h.ddspf = FCC(fourcc('D', 'X', '1', '0'));
        if (md->arraySize > 0xFFFFu) return DXB_E_INVALIDARG;
        HeaderDX10 x; memset(&x, 0, sizeof(x));
        x.dxgiFormat = md->format; x.resourceDimension = md->dimension;
        x.miscFlag = md->miscFlags & ~MISC_TEXTURECUBE;
        if (cube)
        {
            x.miscFlag |= MISC_TEXTURECUBE;
            if (md->arraySize % 6) return DXB_E_INVALIDARG;
            x.arraySize = (uint32_t)(md->arraySize / 6);
        }
        else x.arraySize = (uint32_t)md->arraySize;
        if (flags & DF_FORCE_DX10_MISC2) x.miscFlags2 = md->miscFlags2;
        memcpy(p + kMinHeader, &x, sizeof(x));
    }
    memcpy(p + 4, &h, sizeof(h));
    return DXB_S_OK;
}

int32_t dxb200_dds_save_memory(const dxb200_image* images, size_t nimages, const dxb200_metadata* md, uint32_t flags,
                               void* dst, size_t maxsize, size_t* required)
{
    if (!images || !nimages || !md || !required) return DXB_E_INVALIDARG;
    size_t hdr = 0;
    int32_t hr = dxb200_dds_encode_header(md, flags, nullptr, 0, &hdr);
    if (hr != DXB_S_OK) return hr;
    // exactly the images of the texture, item-major / mip-minor (TexMetadata::ComputeIndex order, :2477-2560); images beyond
    // arraySize * mipLevels are not part of the file
    const size_t count = md->arraySize * md->mipLevels;
    if (!count || nimages < count) return DXB_E_FAIL;
    size_t total = hdr;
    for (size_t item = 0, i = 0; item < md->arraySize; ++item)
    {
        size_t w = md->width, hgt = md->height;
        for (size_t level = 0; level < md->mipLevels; ++level, ++i)
        {
            if (!images[i].pixels) return DXB_E_POINTER;
            if (images[i].format != md->format) return DXB_E_FAIL;
            if (images[i].width != w || images[i].height != hgt) return DXB_E_FAIL;
            size_t row, slice;
            hr = pitch(md->format, w, hgt, &row, &slice);
            if (hr != DXB_S_OK) return hr;
            total += slice;
            if (w > 1) w >>= 1;
            if (hgt > 1) hgt >>= 1;
        }
    }
    *required = total;
    if (!dst) return DXB_S_OK;
    if (maxsize < total) return (int32_t)0x8007007A;
    hr = dxb200_dds_encode_header(md, flags, dst, maxsize, &hdr);
    if (hr != DXB_S_OK) return hr;
    uint8_t* p = static_cast<uint8_t*>(dst) + hdr;
    for (size_t i = 0; i < count; ++i)
    {
        size_t row, slice;
        hr = pitch(md->format, images[i].width, images[i].height, &row, &slice);
        if (hr != DXB_S_OK) return hr;
        if (images[i].rowPitch == row) memcpy(p, images[i].pixels, slice);
        else
        {
            const size_t lines = row ? slice / row : 0, n = images[i].rowPitch < row ? images[i].rowPitch : row;
            for (size_t y = 0; y < lines; ++y) { memset(p + y * row, 0, row); memcpy(p + y * row, images[i].pixels + y * images[i].rowPitch, n); }
        }
        p += slice;
    }
    return DXB_S_OK;
}

int32_t dxb200_dds_get_metadata(const void* src, size_t size, uint32_t flags, dxb200_metadata* md, size_t* dataOffset)
{
    if (!src || !md) return DXB_E_POINTER;
    memset(md, 0, sizeof(*md));
    if (flags & DF_UNSUPPORTED) return DXB_E_NOT_SUPPORTED;
    if (size < kMinHeader) return (int32_t)0x8007000D;                    // HRESULT_E_INVALID_DATA
    const uint8_t* p = static_cast<const uint8_t*>(src);
    uint32_t magic; memcpy(&magic, p, 4);
    if (magic != kMagic) return DXB_E_FAIL;
    Header h; memcpy(&h, p + 4, sizeof(h));
    // DecodeDDSHeader (:352-377): a zero ddspf.size is written by some tools and accepted by the reference
    if (h.size != sizeof(Header) || (h.ddspf.size != 0 && h.ddspf.size != sizeof(PixelFormat))) return DXB_E_NOT_SUPPORTED;
    md->mipLevels = h.mipMapCount ? h.mipMapCount : 1;
    size_t offset = kMinHeader;
    if ((h.ddspf.flags & PF_FOURCC) && h.ddspf.fourCC == fourcc('D', 'X', '1', '0'))
    {
        if (size < kDX10Header) return DXB_E_FAIL;
        HeaderDX10 x; memcpy(&x, p + kMinHeader, sizeof(x));
        offset = kDX10Header;
        md->arraySize = x.arraySize ? x.arraySize : 1;
        md->format = x.dxgiFormat;
        if (!format_ok(md->format)) return DXB_E_NOT_SUPPORTED;
        md->miscFlags = x.miscFlag & ~MISC_TEXTURECUBE;
        if (x.resourceDimension != 3) return (x.resourceDimension == 2 || x.resourceDimension == 4) ? DXB_E_NOT_SUPPORTED : (int32_t)0x8007000D;
        if (x.miscFlag & MISC_TEXTURECUBE) { md->miscFlags |= MISC_TEXTURECUBE; md->arraySize *= 6; }
        md->width = h.width; md->height = h.height; md->depth = 1; md->dimension = 3;
        md->miscFlags2 = x.miscFlags2;
    }
    else
    {
        md->arraySize = 1;
        if (h.flags & HF_VOLUME) return DXB_E_NOT_SUPPORTED;
        if (h.caps2 & CAPS2_CUBEMAP)
        {
            if ((h.caps2 & CAPS2_ALLFACES) != CAPS2_ALLFACES) return DXB_E_NOT_SUPPORTED;
            md->arraySize = 6; md->miscFlags |= MISC_TEXTURECUBE;
        }
        md->width = h.width; md->height = h.height; md->depth = 1; md->dimension = 3;
        // GetDXGIFormat (:149-230): FourCC entries compare the code; the others compare the flag class and only the masks that
        // class defines (RGB(A): all four; luminance: R, plus A with DDPF_ALPHAPIXELS; alpha-only: A; bump: R, G).  The two
        // flag bits nvidia texture tools add (DDPF_SRGB 0x40000000, DDPF_NORMAL 0x80000000) do not take part.
        const uint32_t pfFlags = h.ddspf.flags & ~0xC0000000u;
        const Legacy* hit = nullptr;
        for (const Legacy& e : kLegacy)
        {
            if ((pfFlags & PF_FOURCC) && (e.pf.flags & PF_FOURCC)) { if (h.ddspf.fourCC == e.pf.fourCC) { hit = &e; break; } continue; }
            if ((pfFlags & PF_FOURCC) || (e.pf.flags & PF_FOURCC)) continue;
            if (pfFlags != e.pf.flags || h.ddspf.bitCount != e.pf.bitCount) continue;
            bool same;
            if (pfFlags & 0x40u) same = h.ddspf.rMask == e.pf.rMask && h.ddspf.gMask == e.pf.gMask && h.ddspf.bMask == e.pf.bMask && ((pfFlags & 0x1u) == 0 || h.ddspf.aMask == e.pf.aMask);   // DDPF_RGB
            else if (pfFlags & 0x20000u) same = h.ddspf.rMask == e.pf.rMask && ((pfFlags & 0x1u) == 0 || h.ddspf.aMask == e.pf.aMask);          // DDPF_LUMINANCE
            else if (pfFlags & 0x2u) same = h.ddspf.aMask == e.pf.aMask;                                                                          // DDPF_ALPHA
            else same = h.ddspf.rMask == e.pf.rMask && h.ddspf.gMask == e.pf.gMask && h.ddspf.bMask == e.pf.bMask && h.ddspf.aMask == e.pf.aMask;
            if (same) { hit = &e; break; }
        }
        if (!hit) return DXB_E_NOT_SUPPORTED;
        md->format = hit->format;
        if (hit->pm) md->miscFlags2 = (md->miscFlags2 & ~0x7u) | 2u;        // DXT2 / DXT4 imply premultiplied alpha (:640-647)
    }
    if (!(flags & DF_ALLOW_LARGE))
        if (md->width > 16384u || md->height > 16384u || md->mipLevels > 15u || md->arraySize > 2048u) return DXB_E_NOT_SUPPORTED;
    if ((flags & DF_IGNORE_MIPS) && md->arraySize == 1) md->mipLevels = 1;
    if (dataOffset) *dataOffset = offset;
    return DXB_S_OK;
}

int32_t dxb200_dds_load_memory(const void* src, size_t size, uint32_t flags, const dxb200_image* images, size_t nimages)
{
    dxb200_metadata md; size_t offset = 0;
    int32_t hr = dxb200_dds_get_metadata(src, size, flags, &md, &offset);
    if (hr != DXB_S_OK) return hr;
    if (!images || nimages < md.arraySize * md.mipLevels) return DXB_E_INVALIDARG;
    // the file stores every item's full chain even when DDS_FLAGS_IGNORE_MIPS trimmed the metadata
    Header h; memcpy(&h, static_cast<const uint8_t*>(src) + 4, sizeof(h));
    const size_t fileMips = h.mipMapCount ? h.mipMapCount : 1;
    const uint8_t* p = static_cast<const uint8_t*>(src) + offset;
    const uint8_t* end = static_cast<const uint8_t*>(src) + size;
    size_t index = 0;
    for (size_t item = 0; item < md.arraySize; ++item)
    {
        size_t w = md.width, hgt = md.height;
        for (size_t level = 0; level < fileMips; ++level)
        {
            // DDS_FLAGS_IGNORE_MIPS exists for files with broken or truncated mip tails: with a single item nothing after the
            // requested levels is read or bounds-checked (:2046-2064); arrays still have to skip every item's tail
            if (md.arraySize == 1 && level >= md.mipLevels) break;
            size_t row, slice;
            hr = pitch(md.format, w, hgt, &row, &slice);
            if (hr != DXB_S_OK) return hr;
            if (p + slice > end) return (int32_t)0x80070026;                // HRESULT_E_HANDLE_EOF
            if (level < md.mipLevels)
            {
                const dxb200_image& im = images[index++];
                if (!im.pixels) return DXB_E_POINTER;
                if (im.format != md.format || im.width != w || im.height != hgt) return DXB_E_INVALIDARG;
                if (im.rowPitch == row) memcpy(im.pixels, p, slice);
                else
                {
                    const size_t lines = row ? slice / row : 0, n = im.rowPitch < row ? im.rowPitch : row;
                    for (size_t y = 0; y < lines; ++y) memcpy(im.pixels + y * im.rowPitch, p + y * row, n);
                }
            }
            p += slice;
            if (w > 1) w >>= 1;
            if (hgt > 1) hgt >>= 1;
        }
    }
    return DXB_S_OK;
}

} // extern "C"
