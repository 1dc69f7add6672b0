"""ctypes binding of include/dxtex_b200.h.  No codec logic here; no fallback path."""
import ctypes as C
import os
import numpy as np

from . import formats as F

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DXTEX_B200_LIB") or os.path.join(_HERE, "_lib", "libdxtex_b200.so")     # env override: kernel-variant experiments

SYMBOLS = [
    "dxb200_version", "dxb200_init", "dxb200_init_devices", "dxb200_initialized_devices", "dxb200_shutdown", "dxb200_device_count", "dxb200_launch_count", "dxb200_tma_launch_count", "dxb200_kernel_launch_count", "dxb200_set_option", "dxb200_get_option", "dxb200_last_error",
    "dxb200_host_alloc", "dxb200_host_free", "dxb200_compute_pitch", "dxb200_calculate_mip_levels",
    "dxb200_compress", "dxb200_compress_ex", "dxb200_compress_device", "dxb200_convert_ex", "dxb200_mipmaps_compress", "dxb200_mipmaps_compress_ex", "dxb200_mipmaps_compress_from", "dxb200_mipmaps_compress_from_ex", "dxb200_decompress", "dxb200_decompress_device",
    "dxb200_convert", "dxb200_convert_device", "dxb200_generate_mipmaps", "dxb200_generate_mipmaps_device",
    "dxb200_resize", "dxb200_resize_device", "dxb200_premultiply_alpha", "dxb200_premultiply_alpha_device",
    "dxb200_scale_mipmaps_alpha_for_coverage", "dxb200_scale_mipmaps_alpha_for_coverage_device",
    "dxb200_is_alpha_all_opaque", "dxb200_is_alpha_all_opaque_device",
    "dxb200_apply_channel_steps", "dxb200_apply_channel_steps_device", "dxb200_mipmaps_compress_from_channels",
    "dxb200_mipmaps_convert_from", "dxb200_levels_from",
    "dxb200_mipmaps_compress_from_channels_ex", "dxb200_mipmaps_convert_from_ex", "dxb200_levels_from_ex", "dxb200_texconv_batch",
    "dxb200_texconv_batch_device",
    "dxb200_dds_encode_header", "dxb200_dds_save_memory", "dxb200_dds_get_metadata", "dxb200_dds_load_memory",
]


class Image(C.Structure):
    """dxb200_image == DirectX::Image (DirectXTex.h:437-445)."""
    _fields_ = [("width", C.c_size_t), ("height", C.c_size_t), ("format", C.c_uint32),
                ("rowPitch", C.c_size_t), ("slicePitch", C.c_size_t), ("pixels", C.c_void_p)]


class Metadata(C.Structure):
    """dxb200_metadata == DirectX::TexMetadata (DirectXTex.h:187-216)."""
    _fields_ = [("width", C.c_size_t), ("height", C.c_size_t), ("depth", C.c_size_t), ("arraySize", C.c_size_t), ("mipLevels", C.c_size_t),
                ("miscFlags", C.c_uint32), ("miscFlags2", C.c_uint32), ("format", C.c_uint32), ("dimension", C.c_uint32)]


class ChainSteps(C.Structure):
    """dxb200_chain_steps: the steps dxb200_mipmaps_compress_ex runs between the mips and the compression."""
    _fields_ = [("alphaReference", C.c_float), ("premultiply", C.c_uint32), ("pmalphaFlags", C.c_uint32)]


class ChainSource(C.Structure):
    """dxb200_chain_source: the Decompress and Resize dxb200_mipmaps_compress_from runs in front of the mips."""
    _fields_ = [("decompressFormat", C.c_uint32), ("width", C.c_size_t), ("height", C.c_size_t), ("resizeFilter", C.c_uint32)]


class ChannelSteps(C.Structure):
    """dxb200_channel_steps: texconv's swizzle, colour key, invert-Y and reconstruct-Z steps."""
    _fields_ = [("swizzle", C.c_uint8 * 4), ("zeroMask", C.c_uint8), ("oneMask", C.c_uint8), ("colorKey", C.c_uint8),
                ("invertY", C.c_uint8), ("reconstructZ", C.c_uint8), ("colorKeyValue", C.c_uint32)]


class TexconvSteps(C.Structure):
    """dxb200_texconv_steps: texconv's -alpha (demultiply) and -f BC3n / RXGB (bc3Layout 1 / 2) steps."""
    _fields_ = [("demultiply", C.c_uint32), ("demultiplyFlags", C.c_uint32), ("bc3Layout", C.c_uint32)]


class TexconvJob(C.Structure):
    """dxb200_texconv_job: one texture of dxb200_texconv_batch, the arguments of the call named by kind (0 =
    dxb200_mipmaps_compress_from_channels_ex, 1 = dxb200_mipmaps_convert_from_ex, 2 = dxb200_levels_from_ex)."""
    _fields_ = [("kind", C.c_uint32), ("base", C.POINTER(Image)), ("items", C.c_size_t), ("levels", C.c_size_t),
                ("source", C.POINTER(ChainSource)), ("channels", C.POINTER(ChannelSteps)), ("filter", C.c_uint32),
                ("steps", C.POINTER(ChainSteps)), ("ts", C.POINTER(TexconvSteps)), ("dstFormat", C.c_uint32), ("convertFilter", C.c_uint32),
                ("compressFlags", C.c_uint32), ("threshold", C.c_float), ("dst", C.POINTER(Image)), ("alphaAllOpaque", C.POINTER(C.c_int32))]


STATUS_FN = C.CFUNCTYPE(C.c_int, C.c_size_t, C.c_size_t, C.c_void_p)      # dxb200_status_fn


class DxTexError(RuntimeError):
    def __init__(self, hr, what):
        self.hr = F.hr_u32(hr)
        super().__init__("%s failed: HRESULT 0x%08X (%s)" % (what, self.hr, last_error()))


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError("libdxtex_b200.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'`. "
                          "There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    missing = [n for n in SYMBOLS if not hasattr(lib, n)]
    if missing:
        raise ImportError("%s is stale (missing %s); rebuild with `python -c 'import __graft_entry__ as g; g.build()'`" % (LIB_PATH, ", ".join(missing)))
    IP = C.POINTER(Image)
    lib.dxb200_version.restype = C.c_char_p
    lib.dxb200_last_error.restype = C.c_char_p
    lib.dxb200_launch_count.restype = C.c_uint64
    lib.dxb200_tma_launch_count.restype = C.c_uint64
    lib.dxb200_kernel_launch_count.restype = C.c_uint64
    lib.dxb200_kernel_launch_count.argtypes = [C.c_char_p]
    lib.dxb200_set_option.argtypes = [C.c_uint32, C.c_int32]
    lib.dxb200_get_option.argtypes = [C.c_uint32]
    lib.dxb200_host_alloc.restype = C.c_void_p
    lib.dxb200_host_alloc.argtypes = [C.c_size_t]
    lib.dxb200_host_free.argtypes = [C.c_void_p]
    lib.dxb200_init.argtypes = [C.c_int]
    lib.dxb200_init_devices.argtypes = [C.c_int, C.POINTER(C.c_int)]
    lib.dxb200_initialized_devices.argtypes = [C.POINTER(C.c_int), C.c_int]
    lib.dxb200_compress_ex.argtypes = [IP, C.c_size_t, C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP, STATUS_FN, C.c_void_p]
    lib.dxb200_convert_ex.argtypes = [IP, C.c_size_t, C.c_uint32, C.c_uint32, C.c_float, IP, STATUS_FN, C.c_void_p]
    lib.dxb200_mipmaps_compress.argtypes = [IP, C.c_size_t, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP]
    lib.dxb200_mipmaps_compress_ex.argtypes = [IP, C.c_size_t, C.c_size_t, C.c_uint32, C.POINTER(ChainSteps), C.c_uint32, C.c_uint32, C.c_float,
                                               C.c_float, IP]
    lib.dxb200_mipmaps_compress_from.argtypes = [IP, C.c_size_t, C.POINTER(ChainSource), C.c_size_t, C.c_uint32, C.POINTER(ChainSteps), C.c_uint32,
                                                 C.c_uint32, C.c_float, C.c_float, IP]
    lib.dxb200_mipmaps_compress_from_ex.argtypes = lib.dxb200_mipmaps_compress_from.argtypes + [C.POINTER(C.c_int32)]
    lib.dxb200_mipmaps_compress_from_channels.argtypes = [IP, C.c_size_t, C.POINTER(ChainSource), C.POINTER(ChannelSteps), C.c_size_t, C.c_uint32,
                                                          C.POINTER(ChainSteps), C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP,
                                                          C.POINTER(C.c_int32)]
    lib.dxb200_mipmaps_convert_from.argtypes = [IP, C.c_size_t, C.POINTER(ChainSource), C.POINTER(ChannelSteps), C.c_uint32, C.c_uint32,
                                                C.c_float, C.c_size_t, C.c_uint32, C.POINTER(ChainSteps), IP, C.POINTER(C.c_int32)]
    lib.dxb200_levels_from.argtypes = [IP, C.c_size_t, C.c_size_t, C.POINTER(ChainSource), C.POINTER(ChannelSteps), C.c_uint32, C.c_uint32,
                                       C.c_uint32, C.c_float, C.POINTER(ChainSteps), IP, C.POINTER(C.c_int32)]
    TP = C.POINTER(TexconvSteps)
    lib.dxb200_mipmaps_compress_from_channels_ex.argtypes = lib.dxb200_mipmaps_compress_from_channels.argtypes + [TP]
    lib.dxb200_mipmaps_convert_from_ex.argtypes = lib.dxb200_mipmaps_convert_from.argtypes + [TP]
    lib.dxb200_levels_from_ex.argtypes = lib.dxb200_levels_from.argtypes + [TP]
    lib.dxb200_texconv_batch.argtypes = [C.POINTER(TexconvJob), C.c_size_t, C.POINTER(C.c_int32)]
    lib.dxb200_texconv_batch.restype = C.c_int32
    lib.dxb200_texconv_batch_device.argtypes = [C.POINTER(TexconvJob), C.c_size_t, C.POINTER(C.c_int32), C.c_void_p]
    lib.dxb200_texconv_batch_device.restype = C.c_int32
    lib.dxb200_apply_channel_steps.argtypes = [IP, C.c_size_t, C.POINTER(ChannelSteps), IP]
    lib.dxb200_apply_channel_steps_device.argtypes = [IP, C.c_size_t, C.POINTER(ChannelSteps), IP, C.c_void_p]
    lib.dxb200_is_alpha_all_opaque.argtypes = [IP, C.c_size_t, C.POINTER(C.c_int32)]
    lib.dxb200_is_alpha_all_opaque_device.argtypes = [IP, C.c_size_t, C.POINTER(C.c_int32), C.c_void_p]
    lib.dxb200_compute_pitch.argtypes = [C.c_uint32, C.c_size_t, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.dxb200_calculate_mip_levels.argtypes = [C.c_size_t, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.dxb200_compress.argtypes = [IP, C.c_size_t, C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP]
    lib.dxb200_compress_device.argtypes = [IP, C.c_size_t, C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP, C.c_void_p]
    lib.dxb200_decompress.argtypes = [IP, C.c_size_t, C.c_uint32, IP]
    lib.dxb200_decompress_device.argtypes = [IP, C.c_size_t, C.c_uint32, IP, C.c_void_p]
    lib.dxb200_convert.argtypes = [IP, C.c_size_t, C.c_uint32, C.c_uint32, C.c_float, IP]
    lib.dxb200_convert_device.argtypes = [IP, C.c_size_t, C.c_uint32, C.c_uint32, C.c_float, IP, C.c_void_p]
    lib.dxb200_generate_mipmaps.argtypes = [IP, C.c_size_t, C.c_size_t, C.c_uint32]
    lib.dxb200_generate_mipmaps_device.argtypes = [IP, C.c_size_t, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.dxb200_resize.argtypes = [IP, C.c_size_t, C.c_uint32, IP]
    lib.dxb200_resize_device.argtypes = [IP, C.c_size_t, C.c_uint32, IP, C.c_void_p]
    lib.dxb200_premultiply_alpha.argtypes = [IP, C.c_size_t, C.c_uint32, IP]
    lib.dxb200_premultiply_alpha_device.argtypes = [IP, C.c_size_t, C.c_uint32, IP, C.c_void_p]
    lib.dxb200_scale_mipmaps_alpha_for_coverage.argtypes = [IP, C.c_size_t, C.c_float, IP]
    lib.dxb200_scale_mipmaps_alpha_for_coverage_device.argtypes = [IP, C.c_size_t, C.c_float, IP, C.c_void_p]
    lib.dxb200_scale_mipmaps_alpha_for_coverage.restype = C.c_int32
    lib.dxb200_scale_mipmaps_alpha_for_coverage_device.restype = C.c_int32
    MP, SP = C.POINTER(Metadata), C.POINTER(C.c_size_t)
    lib.dxb200_dds_encode_header.argtypes = [MP, C.c_uint32, C.c_void_p, C.c_size_t, SP]
    lib.dxb200_dds_save_memory.argtypes = [IP, C.c_size_t, MP, C.c_uint32, C.c_void_p, C.c_size_t, SP]
    lib.dxb200_dds_get_metadata.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, MP, SP]
    lib.dxb200_dds_load_memory.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, IP, C.c_size_t]
    for name in ("dxb200_dds_encode_header", "dxb200_dds_save_memory", "dxb200_dds_get_metadata", "dxb200_dds_load_memory"):
        getattr(lib, name).restype = C.c_int32
    for name in ("dxb200_init", "dxb200_init_devices", "dxb200_initialized_devices", "dxb200_compress_ex", "dxb200_convert_ex", "dxb200_mipmaps_compress", "dxb200_mipmaps_compress_ex", "dxb200_mipmaps_compress_from", "dxb200_mipmaps_compress_from_ex", "dxb200_is_alpha_all_opaque", "dxb200_is_alpha_all_opaque_device", "dxb200_apply_channel_steps", "dxb200_apply_channel_steps_device", "dxb200_mipmaps_compress_from_channels", "dxb200_mipmaps_convert_from", "dxb200_levels_from", "dxb200_mipmaps_compress_from_channels_ex", "dxb200_mipmaps_convert_from_ex", "dxb200_levels_from_ex", "dxb200_device_count", "dxb200_compute_pitch", "dxb200_calculate_mip_levels", "dxb200_compress",
                 "dxb200_compress_device", "dxb200_decompress", "dxb200_decompress_device", "dxb200_convert",
                 "dxb200_convert_device", "dxb200_generate_mipmaps", "dxb200_generate_mipmaps_device", "dxb200_resize", "dxb200_resize_device", "dxb200_premultiply_alpha", "dxb200_premultiply_alpha_device"):
        getattr(lib, name).restype = C.c_int32
    return lib


lib = _load()


def last_error():
    return (lib.dxb200_last_error() or b"").decode()


def launch_count():
    return int(lib.dxb200_launch_count())


OPT_BC7_FEED = 1
OPT_MIP_KERNELS = 2


def tma_launch_count():
    return int(lib.dxb200_tma_launch_count())


def kernel_launch_count(kernel):
    """launches of the __global__ function `kernel`, named without template arguments (e.g. "k_mip_tile"), so far in this process"""
    return int(lib.dxb200_kernel_launch_count(kernel.encode()))


def make_image(ptr, w, h, fmt, row_pitch=0):
    row, sl = F.compute_pitch(fmt, w, h)
    if row_pitch and row_pitch != row:
        sl = row_pitch * (max(1, (h + 3) // 4) if fmt in F.BLOCK_BYTES else h)
        row = row_pitch
    return Image(w, h, fmt, row, sl, ptr)


def images(seq):
    arr = (Image * len(seq))(*seq)
    return arr


def _np_ptr(a):
    return a.ctypes.data


# ------------------------------------------------------------------------------------------------
# host-pointer calls (numpy in / numpy out) — what a DirectX::Compress caller sees
def compress(src, w, h, src_fmt, dst_fmt, flags=0, threshold=0.5, alpha_weight=1.0):
    """src: C-contiguous numpy array holding the image rows; returns uint8 array of blocks."""
    src = np.ascontiguousarray(src)
    _, sl = F.compute_pitch(dst_fmt, w, h) if dst_fmt in F.BLOCK_BYTES else (0, 0)
    out = np.zeros(max(sl, 1), np.uint8)
    s = images([make_image(_np_ptr(src), w, h, src_fmt)])
    d = images([Image(w, h, dst_fmt, *(F.compute_pitch(dst_fmt, w, h) if dst_fmt in F.BLOCK_BYTES else (0, 0)), _np_ptr(out))])
    hr = lib.dxb200_compress(s, 1, dst_fmt, flags, threshold, alpha_weight, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_compress")
    return out[:sl]


def init_devices(devices):
    arr = (C.c_int * len(devices))(*devices)
    hr = lib.dxb200_init_devices(len(devices), arr)
    if hr != 0:
        raise DxTexError(hr, "dxb200_init_devices")


def compress_with_status(src, w, h, src_fmt, dst_fmt, callback, flags=0):
    """dxb200_compress_ex of one image; callback(done, total) -> bool (False aborts).  Returns (hr, blocks)."""
    src = np.ascontiguousarray(src)
    row, sl = F.compute_pitch(dst_fmt, w, h)
    out = np.zeros(sl, np.uint8)
    s = images([make_image(_np_ptr(src), w, h, src_fmt)])
    d = images([Image(w, h, dst_fmt, row, sl, _np_ptr(out))])
    cb = STATUS_FN(lambda done, total, user: 1 if callback(done, total) else 0)
    hr = lib.dxb200_compress_ex(s, 1, dst_fmt, flags, 0.5, 1.0, d, cb, None)
    return F.hr_u32(hr), out


def chain_steps(alpha_reference=0.0, premultiply=False, pmalpha_flags=0):
    """the dxb200_chain_steps of texconv's -keepcoverage (alpha_reference > 0) and -pmalpha (premultiply, with pmalpha_flags)"""
    return ChainSteps(alpha_reference, 1 if premultiply else 0, pmalpha_flags)


def mipmaps_compress(srcs, w, h, src_fmt, dst_fmt, filter=0, levels=0, flags=0, steps=None):
    """dxb200_mipmaps_compress_ex of an array of equally sized host images, with the ChainSteps `steps` (None: mips and compression
    only); returns one packed BC chain (bytes) per image."""
    srcs = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in srcs]
    levels = levels or F.count_mips(w, h)
    olayout, total = texture_layout(dst_fmt, w, h, 1, levels)
    row, sl = F.compute_pitch(src_fmt, w, h)
    outs = [np.zeros(total, np.uint8) for _ in srcs]
    s = images([Image(w, h, src_fmt, row, sl, _np_ptr(a)) for a in srcs])
    d = images([Image(lw, lh, dst_fmt, r, sp, _np_ptr(o) + off) for o in outs for (off, lw, lh, r, sp) in olayout])
    hr = lib.dxb200_mipmaps_compress_ex(s, len(srcs), levels, filter, C.byref(steps) if steps is not None else None, dst_fmt, flags, 0.5, 1.0, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_mipmaps_compress_ex")
    return outs


def chain_source(decompress_format=0, width=0, height=0, resize_filter=0):
    """the dxb200_chain_source of texconv's Decompress (a BC base, to decompress_format; 0 = DefaultDecompress) and Resize (to
    width x height with resize_filter; both 0 = the base's size)"""
    return ChainSource(decompress_format, width, height, resize_filter)


def _from_args(bases, w, h, base_fmt, dst_fmt, source, filter, levels, flags, steps, row_pitch):
    """(the arguments of dxb200_mipmaps_compress_from, the output arrays)"""
    bases = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in bases]
    cw, ch = (source.width, source.height) if source is not None and source.width else (w, h)
    levels = levels or F.count_mips(cw, ch)
    olayout, total = texture_layout(dst_fmt, cw, ch, 1, levels)
    outs = [np.zeros(total, np.uint8) for _ in bases]
    s = images([make_image(_np_ptr(a), w, h, base_fmt, row_pitch) for a in bases])
    d = images([Image(lw, lh, dst_fmt, r, sp, _np_ptr(o) + off) for o in outs for (off, lw, lh, r, sp) in olayout])
    return (s, len(bases), C.byref(source) if source is not None else None, levels, filter, C.byref(steps) if steps is not None else None,
            dst_fmt, flags, 0.5, 1.0, d), outs


def mipmaps_compress_from(bases, w, h, base_fmt, dst_fmt, source=None, filter=0, levels=0, flags=0, steps=None, row_pitch=0):
    """dxb200_mipmaps_compress_from of an array of equally sized w x h host images of base_fmt (BC or not; rows row_pitch bytes
    apart, 0 = tight) with the ChainSource `source` and the ChainSteps `steps` (None: none); returns one packed BC chain (bytes)
    per image, of the chain's level 0 size (source's width x height, or w x h)"""
    args, outs = _from_args(bases, w, h, base_fmt, dst_fmt, source, filter, levels, flags, steps, row_pitch)
    hr = lib.dxb200_mipmaps_compress_from(*args)
    if hr != 0:
        raise DxTexError(hr, "dxb200_mipmaps_compress_from")
    return outs


def mipmaps_compress_from_ex(bases, w, h, base_fmt, dst_fmt, source=None, filter=0, levels=0, flags=0, steps=None, row_pitch=0):
    """mipmaps_compress_from through dxb200_mipmaps_compress_from_ex: (the chains, IsAlphaAllOpaque of the output as a bool)"""
    args, outs = _from_args(bases, w, h, base_fmt, dst_fmt, source, filter, levels, flags, steps, row_pitch)
    opaque = C.c_int32(-1)
    hr = lib.dxb200_mipmaps_compress_from_ex(*args, C.byref(opaque))
    if hr != 0:
        raise DxTexError(hr, "dxb200_mipmaps_compress_from_ex")
    return outs, opaque.value == 1


def channel_steps(swizzle=(0, 1, 2, 3), zero_mask=0, one_mask=0, color_key=None, invert_y=False, reconstruct_z=False):
    """the dxb200_channel_steps of texconv's -swizzle (output channel c takes source channel swizzle[c]; bit c of zero_mask /
    one_mask forces channel c to 0 / 1), -c (color_key = 0xRRGGBB, None = off), -inverty and -reconstructz"""
    return ChannelSteps((C.c_uint8 * 4)(*swizzle), zero_mask, one_mask, 0 if color_key is None else 1, 1 if invert_y else 0,
                        1 if reconstruct_z else 0, 0 if color_key is None else color_key)


def texconv_steps(demultiply=False, demultiply_flags=0, bc3_layout=0):
    """the dxb200_texconv_steps of texconv's -alpha (demultiply, with demultiply_flags; REVERSE is implied) and -f BC3n / DXT5nm
    (bc3_layout = 1) or RXGB (bc3_layout = 2)"""
    return TexconvSteps(1 if demultiply else 0, demultiply_flags, bc3_layout)


def mipmaps_compress_from_channels(bases, w, h, base_fmt, dst_fmt, source=None, channels=None, filter=0, levels=0, flags=0, steps=None,
                                   row_pitch=0, texconv=None):
    """mipmaps_compress_from_ex through dxb200_mipmaps_compress_from_channels_ex with the ChannelSteps `channels` and the TexconvSteps
    `texconv` (None: none): (the chains, IsAlphaAllOpaque of the output as a bool)"""
    args, outs = _from_args(bases, w, h, base_fmt, dst_fmt, source, filter, levels, flags, steps, row_pitch)
    opaque = C.c_int32(-1)
    hr = lib.dxb200_mipmaps_compress_from_channels_ex(*args[:3], C.byref(channels) if channels is not None else None, *args[3:], C.byref(opaque),
                                                      C.byref(texconv) if texconv is not None else None)
    if hr != 0:
        raise DxTexError(hr, "dxb200_mipmaps_compress_from_channels_ex")
    return outs, opaque.value == 1


def _ref(x):
    return C.pointer(x) if x is not None else None


def _convert_args(bases, w, h, base_fmt, dst_fmt, source=None, channels=None, convert_filter=0, threshold=0.5, filter=0, levels=0,
                  steps=None, texconv=None):
    """(the dxb200_texconv_job of mipmaps_convert_from's call, without alphaAllOpaque; the output arrays; what the job points to)"""
    bases = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in bases]
    cw, ch = (source.width, source.height) if source is not None and source.width else (w, h)
    levels = levels or F.count_mips(cw, ch)
    olayout, total = texture_layout(dst_fmt, cw, ch, 1, levels)
    outs = [np.zeros(total, np.uint8) for _ in bases]
    s = images([make_image(_np_ptr(a), w, h, base_fmt) for a in bases])
    d = images([Image(lw, lh, dst_fmt, r, sp, _np_ptr(o) + off) for o in outs for (off, lw, lh, r, sp) in olayout])
    job = TexconvJob(1, s, len(bases), levels, _ref(source), _ref(channels), filter, _ref(steps), _ref(texconv), dst_fmt, convert_filter, 0,
                     threshold, d, None)
    return job, outs, (bases, s, d, source, channels, steps, texconv)


def mipmaps_convert_from(bases, w, h, base_fmt, dst_fmt, source=None, channels=None, convert_filter=0, threshold=0.5, filter=0, levels=0,
                         steps=None, texconv=None):
    """dxb200_mipmaps_convert_from_ex of an array of equally sized w x h host images of base_fmt (BC or not) into dst_fmt chains,
    with the ChainSource `source`, the ChannelSteps `channels`, the ChainSteps `steps` and the TexconvSteps `texconv` (None: none):
    (one chain per image, laid out as texture_layout(dst_fmt, W, H, 1, levels), IsAlphaAllOpaque of the output as a bool)"""
    j, outs, _keep = _convert_args(bases, w, h, base_fmt, dst_fmt, source, channels, convert_filter, threshold, filter, levels, steps, texconv)
    opaque = C.c_int32(-1)
    hr = lib.dxb200_mipmaps_convert_from_ex(j.base, j.items, j.source, j.channels, j.dstFormat, j.convertFilter, j.threshold, j.levels,
                                            j.filter, j.steps, j.dst, C.byref(opaque), j.ts)
    if hr != 0:
        raise DxTexError(hr, "dxb200_mipmaps_convert_from_ex")
    return outs, opaque.value == 1


def _levels_args(bases, sizes, base_fmt, dst_fmt, source=None, channels=None, convert_filter=0, compress_flags=0, threshold=0.5, steps=None,
                 texconv=None):
    """(the dxb200_texconv_job of levels_from's call, without alphaAllOpaque; the output arrays; what the job points to)"""
    levels = len(sizes)
    osizes = [(source.width, source.height)] if levels == 1 and source is not None and source.width else list(sizes)
    bases = [[np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in item] for item in bases]
    outs = [[np.zeros(F.compute_pitch(dst_fmt, w, h)[1], np.uint8) for (w, h) in osizes] for _ in bases]
    s = images([make_image(_np_ptr(a), w, h, base_fmt) for item in bases for a, (w, h) in zip(item, sizes)])
    d = images([make_image(_np_ptr(o), w, h, dst_fmt) for item in outs for o, (w, h) in zip(item, osizes)])
    job = TexconvJob(2, s, len(bases), levels, _ref(source), _ref(channels), 0, _ref(steps), _ref(texconv), dst_fmt, convert_filter,
                     compress_flags, threshold, d, None)
    return job, outs, (bases, s, d, source, channels, steps, texconv)


def levels_from(bases, sizes, base_fmt, dst_fmt, source=None, channels=None, convert_filter=0, compress_flags=0, threshold=0.5,
                steps=None, texconv=None):
    """dxb200_levels_from_ex of items that keep their own levels: bases[i][l] = level l of item i (host, tight, of base_fmt, BC or
    not), (w, h) = sizes[l] for every item; the ChainSource `source`, the ChannelSteps `channels`, the ChainSteps `steps` and the
    TexconvSteps `texconv` (None: none).  Returns (outs[i][l] = that level in dst_fmt, tight; IsAlphaAllOpaque of the output as a bool)."""
    j, outs, _keep = _levels_args(bases, sizes, base_fmt, dst_fmt, source, channels, convert_filter, compress_flags, threshold, steps, texconv)
    opaque = C.c_int32(-1)
    hr = lib.dxb200_levels_from_ex(j.base, j.items, j.levels, j.source, j.channels, j.dstFormat, j.convertFilter, j.compressFlags,
                                   j.threshold, j.steps, j.dst, C.byref(opaque), j.ts)
    if hr != 0:
        raise DxTexError(hr, "dxb200_levels_from_ex")
    return outs, opaque.value == 1


def _compress_args(bases, w, h, base_fmt, dst_fmt, source=None, channels=None, filter=0, levels=0, flags=0, steps=None, row_pitch=0,
                   texconv=None):
    """(the dxb200_texconv_job of mipmaps_compress_from_channels' call, without alphaAllOpaque; the output arrays; what it points to)"""
    args, outs = _from_args(bases, w, h, base_fmt, dst_fmt, source, filter, levels, flags, steps, row_pitch)
    s, n, _, levels, filter, _, dst_fmt, flags, threshold, _, d = args
    job = TexconvJob(0, s, n, levels, _ref(source), _ref(channels), filter, _ref(steps), _ref(texconv), dst_fmt, 0, flags, threshold, d, None)
    return job, outs, (s, d, source, channels, steps, texconv)


TEXCONV_KINDS = {"compress": _compress_args, "convert": _convert_args, "levels": _levels_args}


def texconv_batch(jobs):
    """dxb200_texconv_batch of a list of (kind, kwargs): kind "compress" takes mipmaps_compress_from_channels' arguments, "convert"
    mipmaps_convert_from's and "levels" levels_from's.  Returns (the batch's HRESULT, [(HRESULT, outputs as the helper returns them,
    IsAlphaAllOpaque as a bool) per job])."""
    built = [TEXCONV_KINDS[kind](**kw) for kind, kw in jobs]
    opaque = [C.c_int32(-1) for _ in built]
    for (j, _, _), o in zip(built, opaque):
        j.alphaAllOpaque = C.pointer(o)
    table = (TexconvJob * len(built))(*[j for j, _, _ in built])
    results = (C.c_int32 * len(built))()
    hr = lib.dxb200_texconv_batch(table, len(built), results)
    return F.hr_u32(hr), [(F.hr_u32(results[i]), built[i][1], opaque[i].value == 1) for i in range(len(built))]


def texconv_batch_device(jobs, stream=None):
    """dxb200_texconv_batch_device of a list of TexconvJob records whose base and dst pixels are device memory of one device (for
    example torch CUDA tensors' data_ptr()), on `stream`: a torch.cuda.Stream, a raw cudaStream_t handle, or None for the legacy
    default stream.  Returns (the batch's HRESULT, [HRESULT per job]).  Without a job asking for the alpha answer the work is only
    enqueued: synchronise the stream before reading dst."""
    handle = getattr(stream, "cuda_stream", stream)
    table = (TexconvJob * len(jobs))(*jobs)
    results = (C.c_int32 * len(jobs))()
    hr = lib.dxb200_texconv_batch_device(table, len(jobs), results, handle)
    return F.hr_u32(hr), [F.hr_u32(r) for r in results]


def apply_channel_steps(arrays, w, h, fmt, channels, row_pitch=0):
    """dxb200_apply_channel_steps of equally sized w x h host images of fmt (rows row_pitch bytes apart, 0 = tight) with the
    ChannelSteps `channels`: one output array per image, of the input's layout"""
    arrays = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in arrays]
    outs = [np.zeros_like(a) for a in arrays]
    s = images([make_image(_np_ptr(a), w, h, fmt, row_pitch) for a in arrays])
    d = images([make_image(_np_ptr(o), w, h, fmt, row_pitch) for o in outs])
    hr = lib.dxb200_apply_channel_steps(s, len(arrays), C.byref(channels), d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_apply_channel_steps")
    return outs


def is_alpha_all_opaque(arrays, w, h, fmt, row_pitch=0):
    """dxb200_is_alpha_all_opaque of equally sized w x h host images of fmt (rows row_pitch bytes apart, 0 = tight): a bool"""
    arrays = [np.ascontiguousarray(a) for a in arrays]
    s = images([make_image(_np_ptr(a), w, h, fmt, row_pitch) for a in arrays])
    opaque = C.c_int32(-1)
    hr = lib.dxb200_is_alpha_all_opaque(s, len(arrays), C.byref(opaque))
    if hr != 0:
        raise DxTexError(hr, "dxb200_is_alpha_all_opaque")
    return opaque.value == 1


def compress_array(srcs, w, h, src_fmt, dst_fmt, flags=0, threshold=0.5):
    srcs = [np.ascontiguousarray(s) for s in srcs]
    row, sl = F.compute_pitch(dst_fmt, w, h)
    outs = [np.zeros(sl, np.uint8) for _ in srcs]
    s = images([make_image(_np_ptr(a), w, h, src_fmt) for a in srcs])
    d = images([Image(w, h, dst_fmt, row, sl, _np_ptr(o)) for o in outs])
    hr = lib.dxb200_compress(s, len(srcs), dst_fmt, flags, threshold, 1.0, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_compress")
    return outs


def _tight_images(bufs, sizes, fmt):
    return images([Image(w, h, fmt, *F.compute_pitch(fmt, w, h), _np_ptr(b)) for b, (w, h) in zip(bufs, sizes)])


def _outputs(sizes, fmt):
    return [np.zeros(F.compute_pitch(fmt, w, h)[1], np.uint8) for (w, h) in sizes]


def compress_images(srcs, sizes, src_fmt, dst_fmt, flags=0, threshold=0.5):
    """dxb200_compress of host images of DIFFERENT sizes ((w, h) per image) in one call; one block array per image."""
    srcs, outs = [np.ascontiguousarray(a) for a in srcs], _outputs(sizes, dst_fmt)
    hr = lib.dxb200_compress(_tight_images(srcs, sizes, src_fmt), len(srcs), dst_fmt, flags, threshold, 1.0, _tight_images(outs, sizes, dst_fmt))
    if hr != 0:
        raise DxTexError(hr, "dxb200_compress")
    return outs


def convert_images(srcs, sizes, src_fmt, dst_fmt, filter=0, threshold=0.5):
    """dxb200_convert of host images of different sizes in one call; one result per image."""
    srcs, outs = [np.ascontiguousarray(a) for a in srcs], _outputs(sizes, dst_fmt)
    hr = lib.dxb200_convert(_tight_images(srcs, sizes, src_fmt), len(srcs), dst_fmt, filter, threshold, _tight_images(outs, sizes, dst_fmt))
    if hr != 0:
        raise DxTexError(hr, "dxb200_convert")
    return outs


def decompress_images(blocks, sizes, bc_fmt, dst_fmt):
    """dxb200_decompress of block streams of different image sizes in one call; one result per image."""
    blocks, outs = [np.ascontiguousarray(a) for a in blocks], _outputs(sizes, dst_fmt)
    hr = lib.dxb200_decompress(_tight_images(blocks, sizes, bc_fmt), len(blocks), dst_fmt, _tight_images(outs, sizes, dst_fmt))
    if hr != 0:
        raise DxTexError(hr, "dxb200_decompress")
    return outs


def premultiply_alpha_images(srcs, sizes, fmt, flags=0):
    """dxb200_premultiply_alpha of host images of different sizes in one call; one result per image."""
    srcs, outs = [np.ascontiguousarray(a) for a in srcs], _outputs(sizes, fmt)
    hr = lib.dxb200_premultiply_alpha(_tight_images(srcs, sizes, fmt), len(srcs), flags, _tight_images(outs, sizes, fmt))
    if hr != 0:
        raise DxTexError(hr, "dxb200_premultiply_alpha")
    return outs


def generate_mipmaps_images(srcs, w, h, fmt, filter=0, levels=0):
    """dxb200_generate_mipmaps of several equally sized host images in one call; one chain (ScratchImage layout) per image."""
    layout, total = F.mip_chain_layout(fmt, w, h, levels)
    chains = [np.zeros(total, np.uint8) for _ in srcs]
    for chain, src in zip(chains, srcs):
        chain[:layout[0][4]] = np.ascontiguousarray(src).view(np.uint8).reshape(-1)[:layout[0][4]]
    imgs = images([Image(lw, lh, fmt, row, sl, _np_ptr(c) + off) for c in chains for (off, lw, lh, row, sl) in layout])
    hr = lib.dxb200_generate_mipmaps(imgs, len(chains), len(layout), filter)
    if hr != 0:
        raise DxTexError(hr, "dxb200_generate_mipmaps")
    return chains


def resize_images(srcs, w, h, fmt, width, height, filter=0):
    """dxb200_resize of several equally sized host images in one call; one tightly packed width x height result per image."""
    srcs, outs = [np.ascontiguousarray(a) for a in srcs], _outputs([(width, height)] * len(srcs), fmt)
    hr = lib.dxb200_resize(_tight_images(srcs, [(w, h)] * len(srcs), fmt), len(srcs), filter, _tight_images(outs, [(width, height)] * len(srcs), fmt))
    if hr != 0:
        raise DxTexError(hr, "dxb200_resize")
    return outs


def convert(src, w, h, src_fmt, dst_fmt, filter=0, threshold=0.5):
    src = np.ascontiguousarray(src)
    if dst_fmt not in F.BYTES_PER_PIXEL:
        out = np.zeros(16, np.uint8)
        d = images([Image(w, h, dst_fmt, 0, 0, _np_ptr(out))])
    else:
        row, sl = F.compute_pitch(dst_fmt, w, h)
        out = np.zeros(sl, np.uint8)
        d = images([Image(w, h, dst_fmt, row, sl, _np_ptr(out))])
    s = images([make_image(_np_ptr(src), w, h, src_fmt) if src_fmt in F.BYTES_PER_PIXEL or src_fmt in F.BLOCK_BYTES
                else Image(w, h, src_fmt, 0, 0, _np_ptr(src))])
    hr = lib.dxb200_convert(s, 1, dst_fmt, filter, threshold, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_convert")
    return out


def generate_mipmaps(src, w, h, fmt, filter=0, levels=0):
    """Returns (chain bytes laid out as a ScratchImage would, layout list)."""
    src = np.ascontiguousarray(src).view(np.uint8).reshape(-1)
    layout, total = F.mip_chain_layout(fmt, w, h, levels)
    chain = np.zeros(total, np.uint8)
    chain[:layout[0][4]] = src[:layout[0][4]]
    imgs = images([Image(lw, lh, fmt, row, sl, _np_ptr(chain) + off) for (off, lw, lh, row, sl) in layout])
    hr = lib.dxb200_generate_mipmaps(imgs, 1, len(layout), filter)
    if hr != 0:
        raise DxTexError(hr, "dxb200_generate_mipmaps")
    return chain, layout


def resize(src, w, h, fmt, width, height, filter=0):
    """DirectX::Resize of one image; returns the width x height result as tightly packed bytes."""
    src = np.ascontiguousarray(src).view(np.uint8).reshape(-1)
    srow, ssl = F.compute_pitch(fmt, w, h)
    drow, dsl = F.compute_pitch(fmt, width, height)
    out = np.zeros(dsl, np.uint8)
    s = images([Image(w, h, fmt, srow, ssl, _np_ptr(src))])
    d = images([Image(width, height, fmt, drow, dsl, _np_ptr(out))])
    hr = lib.dxb200_resize(s, 1, filter, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_resize")
    return out


def premultiply_alpha(src, w, h, fmt, flags=0):
    """DirectX::PremultiplyAlpha of one image (flags = TEX_PMALPHA_FLAGS); returns the result bytes."""
    src = np.ascontiguousarray(src).view(np.uint8).reshape(-1)
    row, sl = F.compute_pitch(fmt, w, h)
    out = np.zeros(sl, np.uint8)
    s = images([Image(w, h, fmt, row, sl, _np_ptr(src))])
    d = images([Image(w, h, fmt, row, sl, _np_ptr(out))])
    hr = lib.dxb200_premultiply_alpha(s, 1, flags, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_premultiply_alpha")
    return out


def texture_layout(fmt, w, h, array_size=1, mip_levels=1):
    """(list of (offset, w, h, rowPitch, slicePitch) item-major / mip-minor, total bytes) as ScratchImage::Initialize lays it out."""
    out, off = [], 0
    for _ in range(array_size):
        lw, lh = w, h
        for _ in range(mip_levels):
            row, sl = F.compute_pitch(fmt, lw, lh)
            out.append((off, lw, lh, row, sl))
            off += sl
            lw, lh = max(1, lw >> 1), max(1, lh >> 1)
    return out, off


def dds_save(pixels, fmt, w, h, array_size=1, mip_levels=1, misc_flags=0, misc_flags2=0, flags=0):
    """SaveToDDSMemory of a 2D texture whose images are packed in `pixels` in ScratchImage order; returns the file bytes."""
    pixels = np.ascontiguousarray(pixels).view(np.uint8).reshape(-1)
    layout, total = texture_layout(fmt, w, h, array_size, mip_levels)
    assert pixels.size == total
    imgs = images([Image(lw, lh, fmt, row, sl, _np_ptr(pixels) + off) for (off, lw, lh, row, sl) in layout])
    md = Metadata(w, h, 1, array_size, mip_levels, misc_flags, misc_flags2, fmt, 3)
    need = C.c_size_t()
    hr = lib.dxb200_dds_save_memory(imgs, len(layout), C.byref(md), flags, None, 0, C.byref(need))
    if hr != 0:
        raise DxTexError(hr, "dxb200_dds_save_memory")
    out = np.zeros(need.value, np.uint8)
    hr = lib.dxb200_dds_save_memory(imgs, len(layout), C.byref(md), flags, _np_ptr(out), out.size, C.byref(need))
    if hr != 0:
        raise DxTexError(hr, "dxb200_dds_save_memory")
    return out


def dds_load(data, flags=0):
    """LoadFromDDSMemory; returns (Metadata, pixels packed in ScratchImage order)."""
    data = np.ascontiguousarray(data).view(np.uint8).reshape(-1)
    md = Metadata()
    off = C.c_size_t()
    hr = lib.dxb200_dds_get_metadata(_np_ptr(data), data.size, flags, C.byref(md), C.byref(off))
    if hr != 0:
        raise DxTexError(hr, "dxb200_dds_get_metadata")
    layout, total = texture_layout(md.format, md.width, md.height, md.arraySize, md.mipLevels)
    pixels = np.zeros(total, np.uint8)
    imgs = images([Image(lw, lh, md.format, row, sl, _np_ptr(pixels) + o) for (o, lw, lh, row, sl) in layout])
    hr = lib.dxb200_dds_load_memory(_np_ptr(data), data.size, flags, imgs, len(layout))
    if hr != 0:
        raise DxTexError(hr, "dxb200_dds_load_memory")
    return md, pixels


def scale_mipmaps_alpha_for_coverage(chain, w, h, fmt, alpha_ref):
    """DirectX::ScaleMipMapsAlphaForCoverage on one mip chain (bytes in ScratchImage layout); returns the new chain."""
    chain = np.ascontiguousarray(chain).view(np.uint8).reshape(-1)
    layout, total = F.mip_chain_layout(fmt, w, h, 0)
    out = np.zeros(total, np.uint8)
    s = images([Image(lw, lh, fmt, row, sl, _np_ptr(chain) + off) for (off, lw, lh, row, sl) in layout])
    d = images([Image(lw, lh, fmt, row, sl, _np_ptr(out) + off) for (off, lw, lh, row, sl) in layout])
    hr = lib.dxb200_scale_mipmaps_alpha_for_coverage(s, len(layout), alpha_ref, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_scale_mipmaps_alpha_for_coverage")
    return out


def decompress(blocks, w, h, bc_fmt, dst_fmt):
    blocks = np.ascontiguousarray(blocks)
    row, sl = F.compute_pitch(dst_fmt, w, h) if dst_fmt in F.BYTES_PER_PIXEL else (0, 0)
    out = np.zeros(max(sl, 1), np.uint8)
    s = images([make_image(_np_ptr(blocks), w, h, bc_fmt) if bc_fmt in F.BLOCK_BYTES else Image(w, h, bc_fmt, 0, 0, _np_ptr(blocks))])
    d = images([Image(w, h, dst_fmt, row, sl, _np_ptr(out))])
    hr = lib.dxb200_decompress(s, 1, dst_fmt, d)
    if hr != 0:
        raise DxTexError(hr, "dxb200_decompress")
    return out[:sl]
