"""TEST INFRASTRUCTURE for IsAlphaAllOpaque: the reference's answer (tests/cpp/alpha_opaque_probe.cpp linked with the reference
build), the mirror's (the same probe linked with libdxtex_b200.so), the host emulator's (tests/emul/alpha_opaque.cpp) and the
corpus every suite runs: alpha boundary codes of every implemented uncompressed format with alpha, and BC blocks by class."""
import ctypes as C
import os
import subprocess

import numpy as np

from directxtex_b200 import capi, formats as F
from tests.bc7_ranking_build import host_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
IP = C.POINTER(capi.Image)

# the implemented uncompressed formats with alpha (HasAlpha), and the BC formats IsAlphaAllOpaqueBC decodes
PIXEL_FORMATS = (2, 10, 11, 13, 24, 28, 29, 31, 65, 86, 87, 91, 115)
BLOCK_FORMATS = (71, 72, 74, 75, 77, 78, 98, 99)
# implemented formats without alpha: answered without a device
NO_ALPHA_FORMATS = tuple(sorted(set(F.BYTES_PER_PIXEL) - set(PIXEL_FORMATS))) + (80, 81, 83, 84, 95, 96)


class Probe:
    """probe_is_alpha_all_opaque of tests/cpp/alpha_opaque_probe.cpp, linked with the reference build or with the mirror"""

    def __init__(self, out_dir, reference):
        lib_dir = os.path.join(ROOT, "oracle", "_ref") if reference else os.path.join(ROOT, "directxtex_b200", "_lib")
        lib = os.path.join(lib_dir, "libdxtex_ref.so" if reference else "libdxtex_b200.so")
        out = os.path.join(str(out_dir), "alpha_opaque_probe_%s.so" % ("ref" if reference else "ours"))
        subprocess.run([CXX, "-std=c++17", "-w", "-msse2", "-O1", "-fPIC", "-shared", "-I", os.path.join(ROOT, "directxtex_b200", "host"),
                        "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "alpha_opaque_probe.cpp"), "-o", out, lib,
                        "-Wl,-rpath," + lib_dir], check=True)
        self.L = C.CDLL(out)
        self.L.probe_is_alpha_all_opaque.argtypes = [C.c_int, C.c_uint32, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t]

    def opaque(self, fmt, w, h, pixels, items=1, levels=1, cube=False):
        """IsAlphaAllOpaque of Initialize2D(fmt, w, h, items, levels) (InitializeCube with `items` cubes) holding `pixels`"""
        pixels = np.ascontiguousarray(pixels).view(np.uint8).reshape(-1)
        r = self.L.probe_is_alpha_all_opaque(1 if cube else 0, fmt, w, h, items, levels, pixels.ctypes.data, pixels.nbytes)
        assert r in (0, 1), (fmt, w, h, items, levels, cube, pixels.nbytes)
        return r == 1


def load_emul(out_dir):
    L = host_lib("alpha_opaque.cpp", out_dir, os.path.join(ROOT, "tests", "emul"))
    L.emul_is_alpha_all_opaque.argtypes = [IP, C.c_size_t, C.POINTER(C.c_int32)]
    L.emul_is_alpha_all_opaque.restype = C.c_int32
    return L


def container_images(fmt, w, h, pixels, items=1, levels=1, row_pitch=0):
    """the dxb200_image array of a texture in ScratchImage layout held by `pixels` (items x levels images); row_pitch != 0 lays every
    image of level 0 out at that pitch instead (the images then follow each other at pitch x rows)"""
    layout, _ = capi.texture_layout(fmt, w, h, items, levels)
    base = pixels.ctypes.data
    if row_pitch:
        rows = lambda lh: (lh + 3) // 4 if fmt in F.BLOCK_BYTES else lh
        return capi.images([capi.Image(w, h, fmt, row_pitch, row_pitch * rows(h), base + i * row_pitch * rows(h)) for i in range(items)])
    return capi.images([capi.Image(lw, lh, fmt, r, sp, base + off) for (off, lw, lh, r, sp) in layout])


def call(fn, imgs, n):
    """(HRESULT as u32, opaque) of a dxb200_is_alpha_all_opaque-shaped call"""
    opaque = C.c_int32(-1)
    hr = F.hr_u32(fn(imgs, n, C.byref(opaque)))
    return hr, opaque.value


# ---- the uncompressed corpus -------------------------------------------------------------------------------------------------
def alpha_field(fmt):
    """(bits of the alpha field, function(codes) -> one pixel per code, every other field 0) of an uncompressed format with alpha"""
    bpp = F.BYTES_PER_PIXEL[fmt]

    def put(dtype, index, count):
        def make(codes):
            px = np.zeros((len(codes), count), dtype)
            px[:, index] = np.asarray(codes).astype(np.uint64).astype(dtype)
            return px.view(np.uint8).reshape(len(codes), bpp)
        return make

    if fmt == 2:
        return 32, put(np.uint32, 3, 4)
    if fmt in (10, 11, 13):
        return 16, put(np.uint16, 3, 4)
    if fmt in (28, 29, 31, 87, 91):
        return 8, put(np.uint8, 3, 4)
    if fmt == 65:
        return 8, put(np.uint8, 0, 1)
    shift, bits = {24: (30, 2), 86: (15, 1), 115: (12, 4)}[fmt]
    word = np.uint32 if bpp == 4 else np.uint16

    def packed(codes):
        return (np.asarray(codes, np.uint64) << np.uint64(shift)).astype(word).view(np.uint8).reshape(len(codes), bpp)
    return bits, packed


def f32_codes():
    """the fp32 alpha values of the contract: 0.997 and its neighbours, +-0, denormals, +-Inf, FLT_MAX, 1 and 0.99 (as bit patterns)"""
    t = np.float32(0.997)
    vals = [t, np.nextafter(t, np.float32(2)), np.nextafter(t, np.float32(0)), np.float32(0), np.float32(-0.0), np.float32(1e-45),
            np.float32(-1e-45), np.float32(1.1754942e-38), np.float32(np.inf), np.float32(-np.inf), np.finfo(np.float32).max,
            -np.finfo(np.float32).max, np.float32(1), np.float32(0.99), np.float32(2)]
    return np.array(vals, np.float32).view(np.uint32)


def alpha_codes(fmt):
    """every code of the alpha field (fp32: f32_codes; fp16: every non-NaN half)"""
    bits, _ = alpha_field(fmt)
    if fmt == 2:
        return f32_codes()
    codes = np.arange(1 << bits, dtype=np.uint64)
    if fmt == 10:
        codes = codes[~np.isnan(codes.astype(np.uint16).view(np.float16))]
    return codes


def code_values(fmt, codes):
    """the value the alpha code stands for, for ordering only"""
    if fmt == 2:
        return np.asarray(codes, np.uint32).view(np.float32).astype(np.float64)
    if fmt == 10:
        return np.asarray(codes, np.uint16).view(np.float16).astype(np.float64)
    if fmt in (13, 31):
        bits = 16 if fmt == 13 else 8
        c = np.asarray(codes, np.int64)
        return np.where(c >= (1 << (bits - 1)), c - (1 << bits), c).astype(np.float64)
    return np.asarray(codes, np.float64)


def per_code(probe_fn, fmt, codes):
    """the answer for a 1x1 image of each code"""
    _, make = alpha_field(fmt)
    px = make(codes)
    return np.array([probe_fn(fmt, 1, 1, px[i]) for i in range(len(codes))], bool)


def boundary_codes(fmt, opaque_of_code, codes):
    """(the largest non-opaque code, the smallest opaque code) by value"""
    vals = code_values(fmt, codes)
    non, op = codes[~opaque_of_code], codes[opaque_of_code]
    return non[np.argmax(vals[~opaque_of_code])], op[np.argmin(vals[opaque_of_code])]


def placed(fmt, w, h, code, where, fill):
    """a w x h image of opaque `fill` codes with `code` at position where ('first', 'middle', 'last'); (pixels as uint8 rows)"""
    _, make = alpha_field(fmt)
    px = make([fill] * (w * h))
    i = {"first": 0, "middle": (w * h) // 2, "last": w * h - 1}[where]
    px[i] = make([code])[0]
    return px.reshape(-1)


# ---- the BC corpus -------------------------------------------------------------------------------------------------------------
def bc7_mode_blocks(rng, mode, n):
    """n random BC7 blocks of `mode` (8: the reserved mode, no mode bit set, which decodes to zeros)"""
    b = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    if mode == 8:
        b[:, 0] = 0
    else:
        b[:, 0] = (b[:, 0] & np.uint8((0xFF << (mode + 1)) & 0xFF)) | np.uint8(1 << mode)
    return b


def bc1_three_colour(index3):
    """a BC1 block in the three-colour mode (c0 <= c1) whose texels take index 3 (transparent black) where index3[y][x]"""
    bits = 0
    for t in range(16):
        if index3[t // 4][t % 4]:
            bits |= 3 << (2 * t)
    return np.frombuffer(np.array([0x1234, 0xF00F], np.uint16).tobytes() + np.uint32(bits).tobytes(), np.uint8).copy()


def bc1_partial_image(w, h, inside):
    """the blocks of a w x h BC1 image whose index-3 texels lie only in the padding of its partial blocks (inside=False), or one
    of them inside the image (inside=True)"""
    nbx, nby = (w + 3) // 4, (h + 3) // 4
    out = []
    for by in range(nby):
        for bx in range(nbx):
            pad = [[bx * 4 + x >= w or by * 4 + y >= h for x in range(4)] for y in range(4)]
            if inside and by == nby - 1 and bx == nbx - 1:
                pad[(h - 1) % 4][(w - 1) % 4] = True
            out.append(bc1_three_colour(pad))
    return np.concatenate(out)


def bc2_block(nibble, where=5):
    """a BC2 block of opaque texels (nibble 15) but texel `where`, which has alpha nibble `nibble`"""
    a = np.full(16, 15, np.uint8)
    a[where] = nibble
    alpha = (a[0::2] | (a[1::2] << 4)).astype(np.uint8)
    return np.concatenate([alpha, np.array([0xFF, 0xFF, 0, 0, 0, 0, 0, 0], np.uint8)])


def bc3_block(a0, a1, index):
    """a BC3 block whose 16 texels all take alpha index `index` of the palette (a0, a1)"""
    bits = 0
    for t in range(16):
        bits |= index << (3 * t)
    head = bytes([a0, a1]) + bits.to_bytes(6, "little")
    return np.frombuffer(head + bytes([0xFF, 0xFF, 0, 0, 0, 0, 0, 0]), np.uint8).copy()


LINEAR = {72: 71, 75: 74, 78: 77, 99: 98}        # the UNORM twin of each sRGB BC format


def random_blocks(fmt, rng, n):
    return rng.integers(0, 256, (n, F.BLOCK_BYTES[fmt]), dtype=np.uint8)


def block_corpus(fmt, rng):
    """single-block (4x4) images of a BC format: a list of block byte strings covering the format's classes"""
    blocks = list(random_blocks(fmt, rng, 64))
    base = LINEAR.get(fmt, fmt)
    if base == 71:
        blocks += [bc1_three_colour([[False] * 4] * 4), bc1_three_colour([[True] + [False] * 3] + [[False] * 4] * 3)]
    if base == 74:
        blocks += [bc2_block(n, w) for n in (13, 14, 15) for w in (0, 7, 15)]
    if base == 77:
        blocks += [bc3_block(a0, a1, k) for a0 in range(244, 256) for a1 in range(244, 256) for k in range(8)]
        blocks += [bc3_block(a0, a1, k) for (a0, a1) in ((0, 255), (252, 253), (253, 252), (250, 255)) for k in range(8)]
    if base == 98:
        for mode in range(9):
            blocks += list(bc7_mode_blocks(rng, mode, 24))
    return [np.ascontiguousarray(b, np.uint8) for b in blocks]


def reference_encoded(oracle, fmt, kinds=("alpha_uncorr", "cluster2", "gradient"), w=32, h=32, opaque=False):
    """blocks the reference's encoder makes from synth contract classes (RGBA32F; alpha forced to 1 when opaque)"""
    from directxtex_b200 import synth
    out = []
    for kind in kinds:
        img = np.ascontiguousarray(synth.content_ldr(kind, w, h, seed=3))
        if opaque:
            img[..., 3] = 1.0
        hr, blocks = oracle.compress(img, w, h, 2, fmt)
        assert hr == 0, (fmt, kind, hex(hr))
        out.append(blocks)
    return out
