// dxb_formats.h — DXGI_FORMAT values (public D3D ABI), per-format conversion flags and sizes
// for the subset of formats this backend implements.  Plain C/C++, host and device.
// Restates: the conversion-flag table DirectXTexConvert.cpp:2960-3047 (CONVF_* at
// DirectXTexP.h:355-377) and BitsPerPixel DirectXTexUtil.cpp:594.
#pragma once
#include <stdint.h>

enum
{
    DXB_FMT_UNKNOWN = 0,
    DXB_FMT_R32G32B32A32_FLOAT = 2,
    DXB_FMT_R32G32B32_FLOAT = 6,
    DXB_FMT_R16G16B16A16_FLOAT = 10,
    DXB_FMT_R16G16B16A16_UNORM = 11,
    DXB_FMT_R16G16B16A16_SNORM = 13,
    DXB_FMT_R32G32_FLOAT = 16,
    DXB_FMT_R10G10B10A2_UNORM = 24,
    DXB_FMT_R11G11B10_FLOAT = 26,
    DXB_FMT_R8G8B8A8_UNORM = 28,
    DXB_FMT_R8G8B8A8_UNORM_SRGB = 29,
    DXB_FMT_R8G8B8A8_SNORM = 31,
    DXB_FMT_R16G16_FLOAT = 34,
    DXB_FMT_R16G16_UNORM = 35,
    DXB_FMT_R16G16_SNORM = 37,
    DXB_FMT_R32_FLOAT = 41,
    DXB_FMT_R8G8_UNORM = 49,
    DXB_FMT_R8G8_SNORM = 51,
    DXB_FMT_R16_FLOAT = 54,
    DXB_FMT_R16_UNORM = 56,
    DXB_FMT_R16_SNORM = 58,
    DXB_FMT_R8_UNORM = 61,
    DXB_FMT_R8_SNORM = 63,
    DXB_FMT_A8_UNORM = 65,
    DXB_FMT_R9G9B9E5_SHAREDEXP = 67,
    DXB_FMT_BC1_UNORM = 71,
    DXB_FMT_BC1_UNORM_SRGB = 72,
    DXB_FMT_BC2_UNORM = 74,
    DXB_FMT_BC2_UNORM_SRGB = 75,
    DXB_FMT_BC3_UNORM = 77,
    DXB_FMT_BC3_UNORM_SRGB = 78,
    DXB_FMT_BC4_UNORM = 80,
    DXB_FMT_BC4_SNORM = 81,
    DXB_FMT_BC5_UNORM = 83,
    DXB_FMT_BC5_SNORM = 84,
    DXB_FMT_B5G6R5_UNORM = 85,
    DXB_FMT_B5G5R5A1_UNORM = 86,
    DXB_FMT_B8G8R8A8_UNORM = 87,
    DXB_FMT_B8G8R8X8_UNORM = 88,
    DXB_FMT_B8G8R8A8_UNORM_SRGB = 91,
    DXB_FMT_B8G8R8X8_UNORM_SRGB = 93,
    DXB_FMT_BC6H_UF16 = 95,
    DXB_FMT_BC6H_SF16 = 96,
    DXB_FMT_BC7_UNORM = 98,
    DXB_FMT_BC7_UNORM_SRGB = 99,
    DXB_FMT_B4G4R4A4_UNORM = 115,
};

// CONVERT_FLAGS (DirectXTexP.h:355-377)
enum
{
    DXB_CONVF_FLOAT = 0x1, DXB_CONVF_UNORM = 0x2, DXB_CONVF_UINT = 0x4, DXB_CONVF_SNORM = 0x8, DXB_CONVF_SINT = 0x10,
    DXB_CONVF_DEPTH = 0x20, DXB_CONVF_STENCIL = 0x40, DXB_CONVF_SHAREDEXP = 0x80, DXB_CONVF_BGR = 0x100, DXB_CONVF_XR = 0x200,
    DXB_CONVF_PACKED = 0x400, DXB_CONVF_BC = 0x800, DXB_CONVF_YUV = 0x1000, DXB_CONVF_POS_ONLY = 0x2000,
    DXB_CONVF_R = 0x10000, DXB_CONVF_G = 0x20000, DXB_CONVF_B = 0x40000, DXB_CONVF_A = 0x80000,
    DXB_CONVF_RGB_MASK = 0x70000, DXB_CONVF_RGBA_MASK = 0xF0000,
};

// TEX_FILTER_FLAGS bits used on the hot path (DirectXTex.h:741-797)
enum
{
    DXB_FILTER_WRAP_U = 0x1, DXB_FILTER_WRAP_V = 0x2, DXB_FILTER_MIRROR_U = 0x10, DXB_FILTER_MIRROR_V = 0x20,
    DXB_FILTER_SEPARATE_ALPHA = 0x100, DXB_FILTER_FLOAT_X2BIAS = 0x200,
    DXB_FILTER_RGB_COPY_RED = 0x1000, DXB_FILTER_RGB_COPY_GREEN = 0x2000, DXB_FILTER_RGB_COPY_BLUE = 0x4000, DXB_FILTER_RGB_COPY_ALPHA = 0x8000,
    DXB_FILTER_DITHER = 0x10000, DXB_FILTER_DITHER_DIFFUSION = 0x20000, DXB_FILTER_DITHER_MASK = 0xF0000,
    DXB_FILTER_POINT = 0x100000, DXB_FILTER_LINEAR = 0x200000, DXB_FILTER_CUBIC = 0x300000, DXB_FILTER_BOX = 0x400000,
    DXB_FILTER_TRIANGLE = 0x500000, DXB_FILTER_MODE_MASK = 0xF00000,
    DXB_FILTER_SRGB_IN = 0x1000000, DXB_FILTER_SRGB_OUT = 0x2000000, DXB_FILTER_SRGB_MASK = 0xF000000,
};

// TEX_COMPRESS_FLAGS / BC_FLAGS (DirectXTex.h:887-917, BC.h:30-48)
enum
{
    DXB_BC_FLAGS_DITHER_RGB = 0x10000, DXB_BC_FLAGS_DITHER_A = 0x20000, DXB_BC_FLAGS_UNIFORM = 0x40000,
    DXB_BC_FLAGS_USE_3SUBSETS = 0x80000, DXB_BC_FLAGS_FORCE_BC7_MODE6 = 0x100000,
    DXB_COMPRESS_SRGB_IN = 0x1000000, DXB_COMPRESS_SRGB_OUT = 0x2000000, DXB_COMPRESS_PARALLEL = 0x10000000,
};

// HRESULT values (Win32 ABI; SURVEY.md 8(b))
#define DXB_S_OK            ((int32_t)0)
#define DXB_E_NOTIMPL       ((int32_t)0x80004001)
#define DXB_E_POINTER       ((int32_t)0x80004003)
#define DXB_E_ABORT         ((int32_t)0x80004004)
#define DXB_E_FAIL          ((int32_t)0x80004005)
#define DXB_E_UNEXPECTED    ((int32_t)0x8000FFFF)
#define DXB_E_OUTOFMEMORY   ((int32_t)0x8007000E)
#define DXB_E_INVALIDARG    ((int32_t)0x80070057)
#define DXB_E_NOT_SUPPORTED ((int32_t)0x80070032)

#if defined(__CUDACC__)
#define DXB_FMT_FN __host__ __device__ constexpr
#elif defined(__cplusplus)
#define DXB_FMT_FN static constexpr
#else
#define DXB_FMT_FN static inline
#endif

// Conversion flags for the implemented formats; 0 = format not implemented by this backend.
DXB_FMT_FN uint32_t dxb_convert_flags(uint32_t fmt)
{
    const uint32_t R = DXB_CONVF_R, G = DXB_CONVF_G, B = DXB_CONVF_B, A = DXB_CONVF_A;
    switch (fmt)
    {
    case DXB_FMT_R32G32B32A32_FLOAT:  return DXB_CONVF_FLOAT | R | G | B | A;
    case DXB_FMT_R32G32B32_FLOAT:     return DXB_CONVF_FLOAT | R | G | B;
    case DXB_FMT_R16G16B16A16_FLOAT:  return DXB_CONVF_FLOAT | R | G | B | A;
    case DXB_FMT_R16G16B16A16_UNORM:  return DXB_CONVF_UNORM | R | G | B | A;
    case DXB_FMT_R16G16B16A16_SNORM:  return DXB_CONVF_SNORM | R | G | B | A;
    case DXB_FMT_R32G32_FLOAT:        return DXB_CONVF_FLOAT | R | G;
    case DXB_FMT_R10G10B10A2_UNORM:   return DXB_CONVF_UNORM | R | G | B | A;
    case DXB_FMT_R11G11B10_FLOAT:     return DXB_CONVF_FLOAT | DXB_CONVF_POS_ONLY | R | G | B;
    case DXB_FMT_R9G9B9E5_SHAREDEXP:  return DXB_CONVF_FLOAT | DXB_CONVF_SHAREDEXP | DXB_CONVF_POS_ONLY | R | G | B;
    case DXB_FMT_B5G6R5_UNORM:        return DXB_CONVF_UNORM | R | G | B;                     // no CONVF_BGR: the swizzle is in Load / Store (:3024-3025)
    case DXB_FMT_B5G5R5A1_UNORM:      return DXB_CONVF_UNORM | R | G | B | A;
    case DXB_FMT_B4G4R4A4_UNORM:      return DXB_CONVF_UNORM | DXB_CONVF_BGR | R | G | B | A;
    case DXB_FMT_R8G8B8A8_UNORM:
    case DXB_FMT_R8G8B8A8_UNORM_SRGB: return DXB_CONVF_UNORM | R | G | B | A;
    case DXB_FMT_R8G8B8A8_SNORM:      return DXB_CONVF_SNORM | R | G | B | A;
    case DXB_FMT_R16G16_FLOAT:        return DXB_CONVF_FLOAT | R | G;
    case DXB_FMT_R16G16_UNORM:        return DXB_CONVF_UNORM | R | G;
    case DXB_FMT_R16G16_SNORM:        return DXB_CONVF_SNORM | R | G;
    case DXB_FMT_R32_FLOAT:           return DXB_CONVF_FLOAT | R;
    case DXB_FMT_R8G8_UNORM:          return DXB_CONVF_UNORM | R | G;
    case DXB_FMT_R8G8_SNORM:          return DXB_CONVF_SNORM | R | G;
    case DXB_FMT_R16_FLOAT:           return DXB_CONVF_FLOAT | R;
    case DXB_FMT_R16_UNORM:           return DXB_CONVF_UNORM | R;
    case DXB_FMT_R16_SNORM:           return DXB_CONVF_SNORM | R;
    case DXB_FMT_R8_UNORM:            return DXB_CONVF_UNORM | R;
    case DXB_FMT_R8_SNORM:            return DXB_CONVF_SNORM | R;
    case DXB_FMT_A8_UNORM:            return DXB_CONVF_UNORM | A;
    case DXB_FMT_BC1_UNORM: case DXB_FMT_BC1_UNORM_SRGB:
    case DXB_FMT_BC2_UNORM: case DXB_FMT_BC2_UNORM_SRGB:
    case DXB_FMT_BC3_UNORM: case DXB_FMT_BC3_UNORM_SRGB:
    case DXB_FMT_BC7_UNORM: case DXB_FMT_BC7_UNORM_SRGB:
                                      return DXB_CONVF_UNORM | DXB_CONVF_BC | R | G | B | A;
    case DXB_FMT_BC4_UNORM:           return DXB_CONVF_UNORM | DXB_CONVF_BC | R;
    case DXB_FMT_BC4_SNORM:           return DXB_CONVF_SNORM | DXB_CONVF_BC | R;
    case DXB_FMT_BC5_UNORM:           return DXB_CONVF_UNORM | DXB_CONVF_BC | R | G;
    case DXB_FMT_BC5_SNORM:           return DXB_CONVF_SNORM | DXB_CONVF_BC | R | G;
    case DXB_FMT_B8G8R8A8_UNORM: case DXB_FMT_B8G8R8A8_UNORM_SRGB:
                                      return DXB_CONVF_UNORM | DXB_CONVF_BGR | R | G | B | A;
    case DXB_FMT_B8G8R8X8_UNORM: case DXB_FMT_B8G8R8X8_UNORM_SRGB:
                                      return DXB_CONVF_UNORM | DXB_CONVF_BGR | R | G | B;
    case DXB_FMT_BC6H_UF16: case DXB_FMT_BC6H_SF16:
                                      return DXB_CONVF_FLOAT | DXB_CONVF_BC | R | G | B | A;
    default: return 0;
    }
}

// bytes per pixel of an implemented uncompressed format (0 otherwise)
DXB_FMT_FN uint32_t dxb_bytes_per_pixel(uint32_t fmt)
{
    switch (fmt)
    {
    case DXB_FMT_R32G32B32A32_FLOAT: return 16;
    case DXB_FMT_R32G32B32_FLOAT: return 12;
    case DXB_FMT_R16G16B16A16_FLOAT: case DXB_FMT_R16G16B16A16_UNORM: case DXB_FMT_R16G16B16A16_SNORM: case DXB_FMT_R32G32_FLOAT: return 8;
    case DXB_FMT_R10G10B10A2_UNORM: case DXB_FMT_R8G8B8A8_UNORM: case DXB_FMT_R8G8B8A8_UNORM_SRGB: case DXB_FMT_R8G8B8A8_SNORM:
    case DXB_FMT_R16G16_FLOAT: case DXB_FMT_R16G16_UNORM: case DXB_FMT_R16G16_SNORM: case DXB_FMT_R32_FLOAT:
    case DXB_FMT_B8G8R8A8_UNORM: case DXB_FMT_B8G8R8X8_UNORM: case DXB_FMT_B8G8R8A8_UNORM_SRGB: case DXB_FMT_B8G8R8X8_UNORM_SRGB:
    case DXB_FMT_R11G11B10_FLOAT: case DXB_FMT_R9G9B9E5_SHAREDEXP: return 4;
    case DXB_FMT_R8G8_UNORM: case DXB_FMT_R8G8_SNORM: case DXB_FMT_R16_FLOAT: case DXB_FMT_R16_UNORM: case DXB_FMT_R16_SNORM:
    case DXB_FMT_B5G6R5_UNORM: case DXB_FMT_B5G5R5A1_UNORM: case DXB_FMT_B4G4R4A4_UNORM: return 2;
    case DXB_FMT_R8_UNORM: case DXB_FMT_R8_SNORM: case DXB_FMT_A8_UNORM: return 1;
    default: return 0;
    }
}

// bytes per 4x4 block of a BC format (0 otherwise) — DetermineEncoderSettings, DirectXTexCompress.cpp:46-68
DXB_FMT_FN uint32_t dxb_bc_block_bytes(uint32_t fmt)
{
    switch (fmt)
    {
    case DXB_FMT_BC1_UNORM: case DXB_FMT_BC1_UNORM_SRGB: case DXB_FMT_BC4_UNORM: case DXB_FMT_BC4_SNORM: return 8;
    case DXB_FMT_BC2_UNORM: case DXB_FMT_BC2_UNORM_SRGB: case DXB_FMT_BC3_UNORM: case DXB_FMT_BC3_UNORM_SRGB:
    case DXB_FMT_BC5_UNORM: case DXB_FMT_BC5_SNORM: case DXB_FMT_BC6H_UF16: case DXB_FMT_BC6H_SF16:
    case DXB_FMT_BC7_UNORM: case DXB_FMT_BC7_UNORM_SRGB: return 16;
    default: return 0;
    }
}

// The UNORM twin of an sRGB format, every other format itself (MakeLinear, DirectXTexUtil.cpp:1446).  Kernels and launchers
// select code on the twin: a format and its twin have the same load, store, dither store, BC block codec and conversion flags,
// so an sRGB step can only come from the resolved flags (TEX_FILTER_SRGB_IN / _OUT) or an SRGB template argument.
DXB_FMT_FN uint32_t dxb_make_linear(uint32_t fmt)
{
    switch (fmt)
    {
    case DXB_FMT_R8G8B8A8_UNORM_SRGB: return DXB_FMT_R8G8B8A8_UNORM;
    case DXB_FMT_B8G8R8A8_UNORM_SRGB: return DXB_FMT_B8G8R8A8_UNORM;
    case DXB_FMT_B8G8R8X8_UNORM_SRGB: return DXB_FMT_B8G8R8X8_UNORM;
    case DXB_FMT_BC1_UNORM_SRGB:      return DXB_FMT_BC1_UNORM;
    case DXB_FMT_BC2_UNORM_SRGB:      return DXB_FMT_BC2_UNORM;
    case DXB_FMT_BC3_UNORM_SRGB:      return DXB_FMT_BC3_UNORM;
    case DXB_FMT_BC7_UNORM_SRGB:      return DXB_FMT_BC7_UNORM;
    default: return fmt;
    }
}

DXB_FMT_FN int dxb_is_srgb_format(uint32_t fmt)
{
    switch (fmt)
    {
    case DXB_FMT_R8G8B8A8_UNORM_SRGB: case DXB_FMT_BC1_UNORM_SRGB: case DXB_FMT_BC2_UNORM_SRGB: case DXB_FMT_BC3_UNORM_SRGB:
    case DXB_FMT_B8G8R8A8_UNORM_SRGB: case DXB_FMT_B8G8R8X8_UNORM_SRGB: case DXB_FMT_BC7_UNORM_SRGB: return 1;
    default: return 0;
    }
}

// Resolve the sRGB bits exactly as ConvertScanline does (DirectXTexConvert.cpp:3121-3167).
// conversion flags CompressBC passes for a BC1-5 target when the caller gives no sRGB flags and source/target agree
// on sRGB-ness (DetermineEncoderSettings, DirectXTexCompress.cpp:46-68)
DXB_FMT_FN uint32_t dxb_bc15_default_cflags(uint32_t dstFmt)
{
    return (dstFmt == DXB_FMT_BC4_UNORM || dstFmt == DXB_FMT_BC4_SNORM) ? (uint32_t)DXB_FILTER_RGB_COPY_RED
         : (dstFmt == DXB_FMT_BC5_UNORM || dstFmt == DXB_FMT_BC5_SNORM) ? (uint32_t)(DXB_FILTER_RGB_COPY_RED | DXB_FILTER_RGB_COPY_GREEN) : 0u;
}
DXB_FMT_FN uint32_t dxb_resolve_srgb_convert(uint32_t flags, uint32_t inFmt, uint32_t outFmt)
{
    if (dxb_is_srgb_format(inFmt)) flags |= DXB_FILTER_SRGB_IN;
    else if (inFmt == DXB_FMT_A8_UNORM) flags &= ~(uint32_t)DXB_FILTER_SRGB_IN;
    if (dxb_is_srgb_format(outFmt)) flags |= DXB_FILTER_SRGB_OUT;
    else if (outFmt == DXB_FMT_A8_UNORM) flags &= ~(uint32_t)DXB_FILTER_SRGB_OUT;
    if ((flags & (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT)) == (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT))
        flags &= ~(uint32_t)(DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT);
    return flags;
}

// Resolve the sRGB bits as LoadScanlineLinear / StoreScanlineLinear do (DirectXTexConvert.cpp:2817-2855, 2889-2927).
DXB_FMT_FN uint32_t dxb_resolve_srgb_linear(uint32_t flags, uint32_t fmt)
{
    switch (fmt)
    {
    case DXB_FMT_R8G8B8A8_UNORM_SRGB: case DXB_FMT_B8G8R8A8_UNORM_SRGB: case DXB_FMT_B8G8R8X8_UNORM_SRGB:
        return flags | DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT;
    case DXB_FMT_R32G32B32A32_FLOAT: case DXB_FMT_R32G32B32_FLOAT: case DXB_FMT_R16G16B16A16_FLOAT: case DXB_FMT_R16G16B16A16_UNORM:
    case DXB_FMT_R32G32_FLOAT: case DXB_FMT_R10G10B10A2_UNORM: case DXB_FMT_R8G8B8A8_UNORM: case DXB_FMT_R16G16_FLOAT:
    case DXB_FMT_R16G16_UNORM: case DXB_FMT_R32_FLOAT: case DXB_FMT_R8G8_UNORM: case DXB_FMT_R16_FLOAT: case DXB_FMT_R16_UNORM:
    case DXB_FMT_R8_UNORM: case DXB_FMT_B8G8R8A8_UNORM: case DXB_FMT_B8G8R8X8_UNORM:
    case DXB_FMT_R11G11B10_FLOAT: case DXB_FMT_R9G9B9E5_SHAREDEXP: case DXB_FMT_B5G6R5_UNORM: case DXB_FMT_B5G5R5A1_UNORM:
    case DXB_FMT_B4G4R4A4_UNORM:
        return flags;
    default:
        return flags & ~(uint32_t)(DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT);
    }
}
