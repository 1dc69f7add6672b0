"""TEST INFRASTRUCTURE: BC6H and BC7 compression from every source format, anchored on the reference's own encoder input.

CompressBC (DirectXTexCompress.cpp:125-194) loads a block of the source format, replicates a partial block, runs
ConvertScanline(temp, 16, target, source, cflags | srgb) and hands the floats to the encoder.  encoder_input() rebuilds those
floats for a whole image as an R32G32B32A32_FLOAT image X, from the reference's own Convert; compressing X to the target's
linear twin with the flags the recipe gives must then produce the same blocks as compressing the source.  The relation is
checked on the reference itself (the recipe is right), on the host emulator and on the device (the library's load, channel
rules, SNORM bias and sRGB steps are right for every source format), without any agreement between encoders.

Never imported by the product."""
import collections
import concurrent.futures
import os

import numpy as np

from directxtex_b200 import formats as F
from tests import special_values as S

IN, OUT, SRGB = F.TEX_FILTER_SRGB_IN, F.TEX_FILTER_SRGB_OUT, F.TEX_FILTER_SRGB
DITHER_UNIFORM = F.TEX_COMPRESS_DITHER | F.TEX_COMPRESS_UNIFORM
QUICK, THREE = F.TEX_COMPRESS_BC7_QUICK, F.TEX_COMPRESS_BC7_USE_3SUBSETS

SOURCES = sorted(F.BYTES_PER_PIXEL)
TARGETS = (95, 96, 98, 99)
BC6H = (95, 96)
SRGB_FLAGS = (0, IN, OUT, SRGB)
# 22 x 14: partial blocks (CompressBC's {0, 0, 0, 1} replication) and rows that are not 16-byte aligned; 32 x 16: full blocks
SIZES = ((22, 14), (32, 16))
# the linear twin of every sRGB format (MakeLinear): the same bytes and load, no sRGB step of its own
LINEAR_TWIN = {29: 28, 91: 87, 93: 88, 78: 77, 99: 98}
# targets whose output side is UNORM (BC3 has BC7's conversion flags and is bit-exact, so it checks the recipe's input side)
UNORM_OUT = (77, 78, 98, 99)
BC3_TWIN = {98: 77, 99: 78}
# the sources DITHER | UNIFORM runs on, and one BC7 source per class for QUICK and USE_3SUBSETS
DITHER_SOURCES = (28, 31, 85, 26)
BC7_CLASS_SOURCES = {"SNORM": 13, "sRGB": 91, "packed BGR": 115, "R only": 56, "POS_ONLY float": 67, "no alpha": 88}

Case = collections.namedtuple("Case", "sf T flags w h")


def _cases():
    out = [Case(sf, T, f, w, h) for sf in SOURCES for T in TARGETS for f in SRGB_FLAGS for (w, h) in SIZES]
    out += [Case(sf, T, DITHER_UNIFORM | f, 22, 14) for sf in DITHER_SOURCES for T in TARGETS for f in (0, OUT)]
    out += [Case(sf, T, f, 22, 14) for sf in BC7_CLASS_SOURCES.values() for T in (98, 99) for f in (QUICK, THREE, THREE | IN)]
    return out


CASES = _cases()


def case_id(c):
    return "%d->%d flags %#x %dx%d" % (c.sf, c.T, c.flags, c.w, c.h)


def seed(c):
    return c.sf * 1009 + c.T * 31 + c.w + (c.flags >> 16)


# ---- the anchor ------------------------------------------------------------------------------------------------------------
def encoder_input(oracle, src, w, h, sf, T, f):
    """(X, T', f_X): X = the floats CompressBC hands T's encoder for `src` (format sf, compress flags f), as an RGBA32F image;
    compressing X to T' with f_X gives the blocks of compressing `src` to T with f.

    - r, the sRGB steps ConvertScanline runs for (sf -> T, f), is special_values.resolve_srgb.
    - The input side is the reference's Convert of the source, as its linear twin, to RGBA32F with r's SRGB_IN step: the load,
      the channel rules (RGBA32F and every BC6H / BC7 target carry R, G, B and A) and sRGB -> linear.
    - SNORM into a UNORM-output target adds ConvertScanline's SNORM -> UNORM bias (DirectXTexConvert.cpp:3456-3465), v * 0.5 + 0.5
      with two roundings; a FLOAT-out conversion skips it.  For such a target FLOAT -> UNORM's saturate and r's SRGB_OUT step need
      nothing here: compressing X, a FLOAT source into the same target, runs them itself, in that order.
    - BC6H's output side is FLOAT: nothing runs between the input side and r's SRGB_OUT step, so X takes that step too, from the
      reference's Convert to R32G32B32_FLOAT (alpha untouched).  X is then exactly the encoder's input, and compressing it runs no
      sRGB step: an sRGB-out step lost on the source's path cannot be lost the same way on X's.
    - The output side compresses X to T's linear twin with f's encoder flags and, for BC7, r's SRGB_OUT (the blocks do not depend
      on the sRGB tag)."""
    r = S.resolve_srgb(f, sf, T)
    if sf == 2:
        # Convert refuses RGBA32F -> RGBA32F: take the RGB of RGBA32F -> R32G32B32_FLOAT, whose channel rules leave R, G, B
        # alone, and the source's alpha, which no sRGB step touches
        hr, rgb = oracle.convert(src, w, h, 2, 6, r & IN)
        x = np.concatenate([rgb.view(np.float32).reshape(h, w, 3), np.asarray(src).view(np.float32).reshape(h, w, 4)[..., 3:]], -1)
    else:
        hr, x = oracle.convert(src, w, h, LINEAR_TWIN.get(sf, sf), 2, r & IN)
        x = x.view(np.float32).reshape(h, w, 4)
    assert hr == 0, (sf, hex(hr))
    if T in UNORM_OUT and sf in S.SNORM_FORMATS:
        x = (x * np.float32(0.5)).astype(np.float32) + np.float32(0.5)
    if T in BC6H:
        if r & OUT:
            hr, rgb = oracle.convert(np.ascontiguousarray(x), w, h, 2, 6, OUT)
            assert hr == 0
            x = np.concatenate([rgb.view(np.float32).reshape(h, w, 3), x[..., 3:]], -1)
        return np.ascontiguousarray(x, np.float32), T, f & ~SRGB
    return np.ascontiguousarray(x, np.float32), LINEAR_TWIN.get(T, T), (f & ~SRGB) | (r & OUT)


# ---- sources ---------------------------------------------------------------------------------------------------------------
def source(sf, T, f, w, h, seed):
    """the case's source (tightly packed bytes): special_values.source_image, or, where the case runs powf, an image on which
    CUDA's and glibc's powf agree (srgb_safe_image; for an SNORM source into BC6H with an sRGB-out step, _unbiased_out_safe)"""
    d = S.powf_direction(f, sf, T)
    if not d:
        return S.source_image(sf, w, h, seed)
    if d == OUT and T in BC6H and sf in S.SNORM_FORMATS:
        return _unbiased_out_safe(sf, w, h, seed)
    return S.srgb_safe_image(sf, d, w, h, seed)


_SNORM_LAYOUT = {13: (np.int16, 4), 31: (np.int8, 4), 37: (np.int16, 2), 51: (np.int8, 2), 58: (np.int16, 1), 63: (np.int8, 1)}
_UNSAFE = {}


def _unsafe_values(vals):
    """the float32 values (as uint32 bits) among `vals` on which the device's linear -> sRGB step differs from the reference's;
    none without a CUDA device"""
    device = S._device_convert()
    if device is None:
        return np.zeros(0, np.uint32)
    from tests import oracle_lib
    m = -(-len(vals) // 256) * 256
    probe = np.zeros(m, np.uint32)
    probe[:len(vals)] = vals
    hr, want = oracle_lib.load_ref().convert(probe.view(np.float32), 256, m // 256, 41, 2, OUT)
    assert hr == 0
    got = device(probe.view(np.float32), 256, m // 256, 41, 2, OUT)
    same = got.view(np.uint32).reshape(m, 4)[:, 0] == want.view(np.uint32).reshape(m, 4)[:, 0]
    return vals[~same[:len(vals)]]


def _unbiased_out_safe(sf, w, h, seed):
    """An SNORM source for a BC6H target with an sRGB-out step: BC6H's output side is FLOAT, so the loaded values enter powf
    without the SNORM -> UNORM bias that srgb_safe_image's SRGB_OUT images are chosen for.  Every code of source_image whose
    loaded value the two powf disagree on is replaced by 0 (alpha never goes through powf)."""
    from tests import oracle_lib
    dt, c = _SNORM_LAYOUT[sf]
    codes = S.source_image(sf, w, h, seed).view(dt).reshape(w * h, c).copy()
    if sf not in _UNSAFE:
        every = np.arange(np.iinfo(dt).min, np.iinfo(dt).max + 1, dtype=np.int64).astype(dt)
        full = np.repeat(every[:, None], c, 1)
        hr, dec = oracle_lib.load_ref().convert(full, len(every), 1, sf, 2)
        assert hr == 0
        vals = dec.view(np.float32).reshape(-1, 4)[:, 0].view(np.uint32)
        _UNSAFE[sf] = every[np.isin(vals, _unsafe_values(np.unique(vals)))]
    for ch in range(min(c, 3)):
        codes[np.isin(codes[:, ch], _UNSAFE[sf]), ch] = 0
    return np.ascontiguousarray(codes).view(np.uint8).reshape(-1)


def case_source(c):
    return source(c.sf, c.T, c.flags, c.w, c.h, seed(c))


# ---- running many reference encodes ----------------------------------------------------------------------------------------
def parallel_map(fn, items):
    """fn over items on one thread per core: the reference's encoders release the GIL and each call runs its serial CompressBC,
    which keeps every core busy on images of a few dozen blocks (its OpenMP path would not)"""
    with concurrent.futures.ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as ex:
        return list(ex.map(fn, items))


# R16_SNORM and R8_SNORM load their lowest code as a value below -1 (DirectXTexConvert.cpp:1087, :1138) and SNORM -> UNORM does
# not saturate (:3456-3465), so for a BC7 target the reference's encoder is given a value below 0, which it reads beside its 8-bit
# staging (OptimizeRGB on aHDRPixels, BC6HBC7.cpp:2541).  No RGBA32F source can give it that value: FLOAT -> UNORM saturates
# (:3476-3484).  (R)'s BC7 encodes of these sources therefore raise that code to the next one, whose value is exactly -1 (0 after
# the bias on both paths); BC3, the emulator and the device keep it.
LOWEST_SNORM_CODE = {58: (np.int16, -32768), 63: (np.int8, -128)}


def reference_relation(oracle, c, src):
    """(R) for one case and its source: [(target, the reference's blocks from the source, its blocks from X)] for the case's
    target and, for a BC7 target, its BC3 twin"""
    out = []
    for T in (c.T,) + ((BC3_TWIN[c.T],) if c.T in BC3_TWIN else ()):
        s = src
        if T in (98, 99) and c.sf in LOWEST_SNORM_CODE:
            dt, low = LOWEST_SNORM_CODE[c.sf]
            codes = np.array(src).view(dt)
            codes[codes == low] = low + 1
            s = codes.view(np.uint8)
        x, Tx, fx = encoder_input(oracle, s, c.w, c.h, c.sf, T, c.flags)
        hr1, direct = oracle.compress(s, c.w, c.h, c.sf, T, c.flags, parallel=False)
        hr2, via_x = oracle.compress(x, c.w, c.h, 2, Tx, fx, parallel=False)
        assert hr1 == 0 and hr2 == 0, (case_id(c), T, hex(hr1), hex(hr2))
        out.append((T, direct, via_x))
    return out


def differing_blocks(a, b):
    return int((np.asarray(a).reshape(-1, 16) != np.asarray(b).reshape(-1, 16)).any(1).sum())
