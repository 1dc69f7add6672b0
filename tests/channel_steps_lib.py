"""TEST INFRASTRUCTURE for texconv's channel steps (swizzle, colour key, invert Y, reconstruct Z): the reference's answer
(tests/cpp/channel_steps_probe.cpp linked with the reference build: one TransformImage per enabled step), the host emulator's
(tests/emul/channel_steps.cpp) and the corpus every suite runs: every implemented uncompressed format, with every 8-bit code, every
16-bit code or half, the fp32 edge list, NaNs in the float formats, normals with x*x + y*y > 1 and colour-key distances of 50, 51
and 52 codes around the key."""
import ctypes as C
import os
import subprocess

import numpy as np

from directxtex_b200 import capi, formats as F
from tests import special_values as SV
from tests.bc7_ranking_build import host_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
IP = C.POINTER(capi.Image)
SP = C.POINTER(capi.ChannelSteps)

FORMATS = tuple(sorted(F.BYTES_PER_PIXEL))           # every implemented uncompressed format
KEY = 0x4080C0                                       # the corpus's colour key: 64, 128, 192 (every channel can move 52 codes both ways)
W, H = 256, 256                                      # 65536 pixels: every code of a 16-bit channel

# texconv option sets: each step alone (the swizzle twice: a permutation, and a copy with both masks) and all four together
CONFIGS = {
    "swizzle": dict(swizzle=(3, 2, 0, 1)),
    "swizzle_masks": dict(swizzle=(1, 0, 0, 3), zero_mask=0b0100, one_mask=0b1000),
    "color_key": dict(color_key=KEY),
    "invert_y": dict(invert_y=True),
    "reconstruct_z": dict(reconstruct_z=True),
    "all": dict(swizzle=(1, 0, 2, 3), one_mask=0b1000, color_key=KEY, invert_y=True, reconstruct_z=True),
}


def steps(**kw):
    return capi.channel_steps(**kw)


class Probe:
    """probe_channel_steps of tests/cpp/channel_steps_probe.cpp, linked with the reference build"""

    def __init__(self, out_dir):
        lib_dir = os.path.join(ROOT, "oracle", "_ref")
        out = os.path.join(str(out_dir), "channel_steps_probe_ref.so")
        subprocess.run([CXX, "-std=c++17", "-w", "-msse2", "-mfpmath=sse", "-ffp-contract=off", "-O1", "-fPIC", "-shared",
                        "-I", os.path.join(ROOT, "directxtex_b200", "host"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(ROOT, "oracle", "compat"), os.path.join(ROOT, "tests", "cpp", "channel_steps_probe.cpp"), "-o", out,
                        os.path.join(lib_dir, "libdxtex_ref.so"), "-Wl,-rpath," + lib_dir], check=True)
        self.L = C.CDLL(out)
        self.L.probe_channel_steps.argtypes = [IP, C.c_size_t, C.POINTER(C.c_uint8), C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_int,
                                               C.c_int, C.c_void_p, C.c_size_t]
        self.L.probe_channel_steps.restype = C.c_int32

    def call(self, imgs, n, s, out=None):
        """(HRESULT as u32) of the reference's steps `s` (a ChannelSteps) on the n images imgs; the result goes to out (uint8 array)"""
        hr = self.L.probe_channel_steps(imgs, n, s.swizzle, s.zeroMask, s.oneMask, s.colorKey, s.colorKeyValue, s.invertY, s.reconstructZ,
                                        out.ctypes.data if out is not None else None, out.nbytes if out is not None else 0)
        return F.hr_u32(hr)

    def apply(self, fmt, w, h, arrays, s):
        """the reference's output of a w x h array of tight images of fmt"""
        arrays = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in arrays]
        imgs = capi.images([capi.make_image(a.ctypes.data, w, h, fmt) for a in arrays])
        out = np.zeros(sum(a.nbytes for a in arrays), np.uint8)
        hr = self.call(imgs, len(arrays), s, out)
        assert hr == 0, (fmt, hex(hr))
        return np.split(out, len(arrays))

    def is_unorm(self, fmt):
        return self.L.probe_is_unorm(fmt) == 1


def load_emul(out_dir):
    L = host_lib("channel_steps.cpp", out_dir, os.path.join(ROOT, "tests", "emul"))
    L.emul_apply_channel_steps.argtypes = [IP, C.c_size_t, SP, IP]
    L.emul_apply_channel_steps.restype = C.c_int32
    L.emul_plan_mipmaps_compress_from_channels.argtypes = [IP, C.c_size_t, C.POINTER(capi.ChainSource), SP, C.c_size_t, C.c_uint32,
                                                           C.POINTER(capi.ChainSteps), C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP,
                                                           C.POINTER(C.c_uint64)]
    L.emul_plan_mipmaps_compress_from_channels.restype = C.c_int32
    L.emul_channel_decompress_format.argtypes = [C.c_uint32, SP]
    L.emul_channel_decompress_format.restype = C.c_uint32
    L.emul_channel_unorm.argtypes = [C.c_uint32]
    return L


def emul_apply(E, fmt, w, h, arrays, s):
    arrays = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in arrays]
    outs = [np.zeros_like(a) for a in arrays]
    src = capi.images([capi.make_image(a.ctypes.data, w, h, fmt) for a in arrays])
    dst = capi.images([capi.make_image(o.ctypes.data, w, h, fmt) for o in outs])
    hr = F.hr_u32(E.emul_apply_channel_steps(src, len(arrays), C.byref(s), dst))
    assert hr == 0, (fmt, hex(hr))
    return outs


# ---- the corpus ---------------------------------------------------------------------------------------------------------------
def _key_pixels(fmt):
    """pixels of an 8-bit-channel UNORM format whose r, g and b lie 50, 51 or 52 codes from the key's (all 27 combinations, both
    directions), with alpha 0x80"""
    kr, kg, kb = (KEY >> 16) & 0xFF, (KEY >> 8) & 0xFF, KEY & 0xFF
    d = [-52, -51, -50, 50, 51, 52, 0]
    px = np.array([[kr + a, kg + b, kb + c, 0x80] for a in d for b in d for c in d], np.uint8)
    if fmt in (87, 88, 91, 93):
        px = px[:, [2, 1, 0, 3]]
    return px.reshape(-1)


def _nan_pixels(fmt, n):
    """n pixels of a float format holding NaNs (quiet, signalling-pattern and negative) in every channel position"""
    if fmt in SV.F32_FORMATS:
        c = SV.CHANNELS[fmt]
        v = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0x3F800000], np.uint32)
        return np.resize(np.roll(np.resize(v, (n, c)), 1, 1), (n, c)).astype(np.uint32).view(np.uint8).reshape(-1)
    c = SV.CHANNELS[fmt]
    v = np.array([0x7E00, 0xFE00, 0x7C01, 0x3C00], np.uint16)
    return np.resize(v, (n, c)).view(np.uint8).reshape(-1)


def corpus(fmt, w=W, h=H, seed=0):
    """a w x h tight image of fmt: special_values.source_image (every code / half / the fp32 edges) with, in its first rows, the
    colour-key distances (8-bit UNORM RGBA / BGRA), NaNs (float formats) and x = y = 1 normals (every format: code all-ones)"""
    bpp = F.BYTES_PER_PIXEL[fmt]
    img = SV.source_image(fmt, w, h, seed).copy()
    at = 0
    extra = []
    if fmt in (28, 29, 87, 88, 91, 93):
        extra.append(_key_pixels(fmt))
    if fmt in SV.F32_FORMATS or fmt in SV.F16_FORMATS:
        extra.append(_nan_pixels(fmt, 16))
    if fmt in SV.F32_FORMATS:
        c = SV.CHANNELS[fmt]
        extra.append(np.resize(np.array([1.0, 1.0, 0.5, 1.0, 0.8, 0.8, 0.0, 1.0], np.float32), 2 * c).view(np.uint8))
    for e in extra:
        img[at:at + e.nbytes] = e
        at += e.nbytes
    assert at <= img.nbytes and img.nbytes == w * h * bpp
    return img
