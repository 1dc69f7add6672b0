"""DXGI_FORMAT values, flag constants and size helpers (host-side mirror of dxb_formats.h)."""

DXGI_FORMAT = {
    "UNKNOWN": 0, "R32G32B32A32_FLOAT": 2, "R32G32B32_FLOAT": 6, "R16G16B16A16_FLOAT": 10, "R16G16B16A16_UNORM": 11,
    "R16G16B16A16_SNORM": 13, "R32G32_FLOAT": 16, "R10G10B10A2_UNORM": 24, "R11G11B10_FLOAT": 26, "R8G8B8A8_UNORM": 28, "R8G8B8A8_UNORM_SRGB": 29,
    "R8G8B8A8_SNORM": 31, "R16G16_FLOAT": 34, "R16G16_UNORM": 35, "R16G16_SNORM": 37, "R32_FLOAT": 41, "R8G8_UNORM": 49,
    "R8G8_SNORM": 51, "R16_FLOAT": 54, "R16_UNORM": 56, "R16_SNORM": 58, "R8_UNORM": 61, "R8_SNORM": 63, "A8_UNORM": 65, "R9G9B9E5_SHAREDEXP": 67,
    "BC1_UNORM": 71, "BC1_UNORM_SRGB": 72, "BC2_UNORM": 74, "BC2_UNORM_SRGB": 75, "BC3_UNORM": 77, "BC3_UNORM_SRGB": 78,
    "BC4_UNORM": 80, "BC4_SNORM": 81, "BC5_UNORM": 83, "BC5_SNORM": 84, "B5G6R5_UNORM": 85, "B5G5R5A1_UNORM": 86, "B8G8R8A8_UNORM": 87, "B8G8R8X8_UNORM": 88,
    "B8G8R8A8_UNORM_SRGB": 91, "B8G8R8X8_UNORM_SRGB": 93, "BC6H_UF16": 95, "BC6H_SF16": 96, "BC7_UNORM": 98, "BC7_UNORM_SRGB": 99, "B4G4R4A4_UNORM": 115,
}
globals().update({"DXGI_FORMAT_" + k: v for k, v in DXGI_FORMAT.items()})

BYTES_PER_PIXEL = {26: 4, 67: 4, 85: 2, 86: 2, 115: 2, 2: 16, 6: 12, 10: 8, 11: 8, 13: 8, 16: 8, 24: 4, 28: 4, 29: 4, 31: 4, 34: 4, 35: 4, 37: 4, 41: 4,
                   49: 2, 51: 2, 54: 2, 56: 2, 58: 2, 61: 1, 63: 1, 65: 1, 87: 4, 88: 4, 91: 4, 93: 4}
BLOCK_BYTES = {71: 8, 72: 8, 74: 16, 75: 16, 77: 16, 78: 16, 80: 8, 81: 8, 83: 16, 84: 16, 95: 16, 96: 16, 98: 16, 99: 16}

# TEX_COMPRESS_FLAGS (DirectXTex.h:887-917)
TEX_COMPRESS_DEFAULT = 0
TEX_COMPRESS_RGB_DITHER = 0x10000
TEX_COMPRESS_A_DITHER = 0x20000
TEX_COMPRESS_DITHER = 0x30000
TEX_COMPRESS_UNIFORM = 0x40000
TEX_COMPRESS_BC7_USE_3SUBSETS = 0x80000
TEX_COMPRESS_BC7_QUICK = 0x100000
TEX_COMPRESS_SRGB_IN = 0x1000000
TEX_COMPRESS_SRGB_OUT = 0x2000000
TEX_COMPRESS_SRGB = 0x3000000
TEX_COMPRESS_PARALLEL = 0x10000000
TEX_THRESHOLD_DEFAULT = 0.5

# TEX_FILTER_FLAGS (DirectXTex.h:741-797)
TEX_FILTER_DEFAULT = 0
TEX_FILTER_WRAP_U = 0x1
TEX_FILTER_WRAP_V = 0x2
TEX_FILTER_WRAP = 0x7
TEX_FILTER_MIRROR_U = 0x10
TEX_FILTER_MIRROR_V = 0x20
TEX_FILTER_MIRROR = 0x70
TEX_FILTER_FLOAT_X2BIAS = 0x200
TEX_FILTER_RGB_COPY_RED = 0x1000
TEX_FILTER_RGB_COPY_GREEN = 0x2000
TEX_FILTER_RGB_COPY_BLUE = 0x4000
TEX_FILTER_RGB_COPY_ALPHA = 0x8000
TEX_FILTER_DITHER = 0x10000
TEX_FILTER_DITHER_DIFFUSION = 0x20000
TEX_FILTER_POINT = 0x100000
TEX_FILTER_LINEAR = 0x200000
TEX_FILTER_CUBIC = 0x300000
TEX_FILTER_BOX = 0x400000
TEX_FILTER_FANT = 0x400000
TEX_FILTER_TRIANGLE = 0x500000
TEX_FILTER_SRGB_IN = 0x1000000
TEX_FILTER_SRGB_OUT = 0x2000000
TEX_FILTER_SRGB = 0x3000000

# HRESULTs
S_OK = 0
E_NOTIMPL = 0x80004001
E_POINTER = 0x80004003
E_ABORT = 0x80004004
E_FAIL = 0x80004005
E_OUTOFMEMORY = 0x8007000E
E_INVALIDARG = 0x80070057
HRESULT_E_NOT_SUPPORTED = 0x80070032


def hr_u32(hr):
    return hr & 0xFFFFFFFF


def compute_pitch(fmt, w, h):
    """(rowPitch, slicePitch) per ComputePitch (DirectXTexUtil.cpp:961-1183), CP_FLAGS_NONE."""
    if fmt in BLOCK_BYTES:
        row = max(1, (w + 3) // 4) * BLOCK_BYTES[fmt]
        return row, row * max(1, (h + 3) // 4)
    row = w * BYTES_PER_PIXEL[fmt]
    return row, row * h


def count_mips(w, h):
    n = 1
    while w > 1 or h > 1:
        w = max(1, w >> 1)
        h = max(1, h >> 1)
        n += 1
    return n


def mip_chain_layout(fmt, w, h, levels=0):
    """[(offset, width, height, rowPitch, slicePitch)] of one item's chain as ScratchImage lays it out
    (DirectXTexImage.cpp:34-268): levels back to back, each slicePitch bytes."""
    if levels == 0:
        levels = count_mips(w, h)
    out, off = [], 0
    for _ in range(levels):
        row, sl = compute_pitch(fmt, w, h)
        out.append((off, w, h, row, sl))
        off += sl
        w = max(1, w >> 1)
        h = max(1, h >> 1)
    return out, off
