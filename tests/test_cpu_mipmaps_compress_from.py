"""CPU suite: the argument checks of dxb200_mipmaps_compress_from (Decompress -> Resize -> GenerateMipMaps -> ... -> Compress).

Every check of every step happens before anything is uploaded, so the HRESULT table needs no device: each case is run through
the library, through the planner alone (dxb_plan.h built on the host by tests/emul/from_plan.cpp) and, where it exists, through the
separate library call that fails first.  The DefaultDecompress table of dxb_formats.h is held against the format the reference's
own Decompress(..., DXGI_FORMAT_UNKNOWN, ...) writes."""
import ctypes as C
import os

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests.bc7_ranking_build import host_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = capi.lib
NO_DEVICE = L.dxb200_device_count() == 0
IP = C.POINTER(capi.Image)


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    P = host_lib("from_plan.cpp", tmp_path_factory.mktemp("from_plan"), os.path.join(ROOT, "tests", "emul"))
    P.emul_plan_mipmaps_compress_from.argtypes = [IP, C.c_size_t, C.POINTER(capi.ChainSource), C.c_size_t, C.c_uint32,
                                                  C.POINTER(capi.ChainSteps), C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP,
                                                  C.POINTER(C.c_uint64)]
    P.emul_plan_mipmaps_compress_from.restype = C.c_int32
    return P


class Call:
    """the arguments of one dxb200_mipmaps_compress_from call: `items` bases of base_fmt, bw x bh, at row pitch `pitch` (0: tight),
    and destinations of dst_fmt laid out for a dw x dh chain of `levels` levels (dw x dh: the source's size, else the base's)"""

    def __init__(self, base_fmt, bw, bh, source=None, levels=0, filter=0, steps=None, dst_fmt=98, items=1, pitch=0,
                 dst_size=None, sizes=None, null_base=False):
        self.keep = []
        sizes = sizes or [(bw, bh)] * items
        imgs = []
        for (w, h) in sizes:
            row, sl = F.compute_pitch(base_fmt, w, h) if (base_fmt in F.BLOCK_BYTES or base_fmt in F.BYTES_PER_PIXEL) else (w * 4, w * h * 4)
            if pitch:
                sl = pitch * (sl // row)
                row = pitch
            buf = np.zeros(sl + 64, np.uint8)
            self.keep.append(buf)
            imgs.append(capi.Image(w, h, base_fmt, row, sl, None if null_base else buf.ctypes.data))
        self.base = capi.images(imgs)
        self.items = len(sizes)
        self.source = source
        cw, ch = dst_size or ((source.width, source.height) if source is not None and source.width and source.height else (bw, bh))
        self.levels = levels or F.count_mips(cw, ch)
        layout, total = capi.texture_layout(dst_fmt, cw, ch, 1, min(self.levels, F.count_mips(cw, ch)))
        layout = (layout * (self.levels // len(layout) + 1))[:self.levels]
        out = np.zeros(total + 64, np.uint8)
        self.keep.append(out)
        self.dst = capi.images([capi.Image(lw, lh, dst_fmt, r, sp, out.ctypes.data + off) for _ in range(self.items) for (off, lw, lh, r, sp) in layout])
        self.filter, self.steps, self.dst_fmt = filter, steps, dst_fmt

    def args(self):
        return (self.base, self.items, C.byref(self.source) if self.source is not None else None, self.levels, self.filter,
                C.byref(self.steps) if self.steps is not None else None, self.dst_fmt, 0, 0.5, 1.0, self.dst)

    def library(self):
        return F.hr_u32(L.dxb200_mipmaps_compress_from(*self.args()))

    def plan(self, P):
        out = (C.c_uint64 * 6)()
        hr = F.hr_u32(P.emul_plan_mipmaps_compress_from(*self.args(), out))
        return hr, tuple(int(v) for v in out)


def decompress_hr(base_fmt, w, h, dst_fmt, pitch=0):
    """HRESULT of dxb200_decompress of one w x h image into dst_fmt laid out at its compute_pitch"""
    row, sl = F.compute_pitch(base_fmt, w, h)
    if pitch:
        sl, row = pitch * (sl // row), pitch
    src, dst = np.zeros(sl, np.uint8), np.zeros(w * h * 16 + 16, np.uint8)
    drow, dsl = F.compute_pitch(dst_fmt, w, h) if dst_fmt in F.BYTES_PER_PIXEL else (0, 0)
    return F.hr_u32(L.dxb200_decompress(capi.images([capi.Image(w, h, base_fmt, row, sl, src.ctypes.data)]), 1, dst_fmt,
                                        capi.images([capi.Image(w, h, dst_fmt, drow, dsl, dst.ctypes.data)])))


def resize_hr(fmt, w, h, dw, dh, filter):
    src, dst = np.zeros(w * h * 16, np.uint8), np.zeros(dw * dh * 16, np.uint8)
    return F.hr_u32(L.dxb200_resize(capi.images([capi.Image(w, h, fmt, *F.compute_pitch(fmt, w, h), src.ctypes.data)]), 1, filter,
                                    capi.images([capi.Image(dw, dh, fmt, *F.compute_pitch(fmt, dw, dh), dst.ctypes.data)])))


def src(decompress_format=0, width=0, height=0, resize_filter=0):
    return capi.chain_source(decompress_format, width, height, resize_filter)


BOX, LINEAR, CUBIC = F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC
# (name, Call arguments, HRESULT): one case per check of every step, in the order the separate calls would meet them
TABLE = [
    ("width without height", dict(base_fmt=77, bw=64, bh=64, source=src(0, 32, 0)), F.E_INVALIDARG),
    ("height without width", dict(base_fmt=28, bw=64, bh=64, source=src(0, 0, 32)), F.E_INVALIDARG),
    ("no items", dict(base_fmt=77, bw=64, bh=64, items=0, source=src()), F.E_INVALIDARG),
    ("BC base without pixels", dict(base_fmt=77, bw=64, bh=64, source=src(), null_base=True), F.E_POINTER),
    ("resized base without pixels", dict(base_fmt=28, bw=64, bh=64, source=src(0, 32, 32), null_base=True), F.E_POINTER),
    ("decompress to a BC format", dict(base_fmt=77, bw=64, bh=64, source=src(71)), F.E_INVALIDARG),
    ("decompress to an unimplemented format", dict(base_fmt=77, bw=64, bh=64, source=src(20)), F.HRESULT_E_NOT_SUPPORTED),
    ("BC row pitch off the block size", dict(base_fmt=77, bw=64, bh=64, source=src(), pitch=16 * 16 + 8), F.E_INVALIDARG),
    ("BC1 row pitch off the block size", dict(base_fmt=71, bw=64, bh=64, source=src(), pitch=8 * 16 + 4), F.E_INVALIDARG),
    ("BOX resize at 3:1", dict(base_fmt=77, bw=96, bh=96, source=src(0, 32, 32, BOX)), F.E_FAIL),
    ("BOX resize of an uncompressed base at 1:2", dict(base_fmt=28, bw=32, bh=32, source=src(0, 64, 64, BOX)), F.E_FAIL),
    ("unknown resize filter", dict(base_fmt=28, bw=64, bh=64, source=src(0, 32, 32, 0x600000)), F.HRESULT_E_NOT_SUPPORTED),
    ("items of two sizes with a resize", dict(base_fmt=77, bw=64, bh=64, sizes=[(64, 64), (32, 32)], source=src(0, 16, 16)), F.E_INVALIDARG),
    ("items of two sizes, decompress only", dict(base_fmt=77, bw=64, bh=64, sizes=[(64, 64), (32, 32)], source=src()), F.E_INVALIDARG),
    ("levels above the resized chain's", dict(base_fmt=77, bw=64, bh=64, source=src(0, 16, 16), levels=6), F.E_INVALIDARG),
    ("levels = 1", dict(base_fmt=77, bw=64, bh=64, source=src(0, 32, 32), levels=1), F.E_INVALIDARG),
    ("BOX mips on a resized non-power-of-two chain", dict(base_fmt=77, bw=64, bh=64, source=src(0, 48, 48, LINEAR), filter=BOX), F.E_FAIL),
    ("dst sized for the base", dict(base_fmt=77, bw=64, bh=64, source=src(0, 32, 32), dst_size=(64, 64), levels=6), F.E_FAIL),
    ("premultiply of BC4's default R8", dict(base_fmt=80, bw=64, bh=64, source=src(), steps=capi.chain_steps(premultiply=True)),
     F.HRESULT_E_NOT_SUPPORTED),
    ("coverage of BC5's default R8G8", dict(base_fmt=83, bw=64, bh=64, source=src(), steps=capi.chain_steps(0.5)), F.S_OK),
    ("BC base to a BC target", dict(base_fmt=77, bw=64, bh=64, source=src(), dst_fmt=28), F.E_INVALIDARG),
]

# (name, Call arguments, (decompress, resize, level-0 format, width, height)) of calls every step accepts
VALID = [
    ("BC3, DefaultDecompress", dict(base_fmt=77, bw=64, bh=16, source=src()), (1, 0, 28, 64, 16)),
    ("BC7 sRGB, DefaultDecompress", dict(base_fmt=99, bw=37, bh=22, source=src()), (1, 0, 29, 37, 22)),
    ("BC4 SNORM to R8G8B8A8_SNORM", dict(base_fmt=81, bw=37, bh=22, source=src(31)), (1, 0, 31, 37, 22)),
    ("BC6H to RGBA16F, resized 3:1", dict(base_fmt=95, bw=96, bh=48, source=src(10, 32, 16, LINEAR)), (1, 1, 10, 32, 16)),
    ("BC1 resized 1:3 CUBIC", dict(base_fmt=71, bw=16, bh=16, source=src(0, 48, 48, CUBIC)), (1, 1, 28, 48, 48)),
    ("RGBA8 resized 2:1, filter 0", dict(base_fmt=28, bw=64, bh=32, source=src(0, 32, 16)), (0, 1, 28, 32, 16)),
    ("RGBA8, no-op source", dict(base_fmt=28, bw=64, bh=32, source=src(0, 64, 32, BOX)), (0, 0, 28, 64, 32)),
    ("RGBA8, no source", dict(base_fmt=28, bw=64, bh=32), (0, 0, 28, 64, 32)),
    ("BC3 with coverage and premultiply", dict(base_fmt=77, bw=64, bh=64, source=src(0, 32, 32), steps=capi.chain_steps(0.5, True)),
     (1, 1, 28, 32, 32)),
    ("BC3 at a row pitch wider than tight", dict(base_fmt=77, bw=64, bh=64, source=src(), pitch=16 * 16 + 32), (1, 0, 28, 64, 64)),
]


@pytest.mark.parametrize("name,kw,want", TABLE, ids=[t[0] for t in TABLE])
def test_hresult_table(planner, name, kw, want):
    """The library's HRESULT, the planner's and the expected one agree; an accepted call fails only for want of a device."""
    c = Call(**kw)
    hr_plan, _ = c.plan(planner)
    assert hr_plan == want, (name, hex(hr_plan))
    hr = c.library()
    if want == F.S_OK:
        assert hr == (F.E_FAIL if NO_DEVICE else F.S_OK), (name, hex(hr))
    else:
        assert hr == want, (name, hex(hr))


def test_first_failing_separate_call():
    """The step each error comes from returns that error as a separate call."""
    assert decompress_hr(77, 64, 64, 71) == F.E_INVALIDARG
    assert decompress_hr(77, 64, 64, 20) == F.HRESULT_E_NOT_SUPPORTED
    assert decompress_hr(77, 64, 64, 28, pitch=16 * 16 + 8) == F.E_INVALIDARG
    assert resize_hr(28, 96, 96, 32, 32, BOX) == F.E_FAIL
    assert resize_hr(28, 32, 32, 64, 64, BOX) == F.E_FAIL
    assert resize_hr(28, 64, 64, 32, 32, 0x600000) == F.HRESULT_E_NOT_SUPPORTED


def test_reference_resize_box_ratio(oracle):
    """The reference's Resize refuses BOX at 3:1 as the library does."""
    img = np.zeros(96 * 96 * 4, np.uint8)
    hr, _ = oracle.resize(img, 96, 96, 28, 32, 32, BOX)
    assert F.hr_u32(hr) == F.E_FAIL


@pytest.mark.parametrize("name,kw,want", VALID, ids=[v[0] for v in VALID])
def test_valid_calls(planner, name, kw, want):
    """Calls every step accepts: the planner stages the front steps and level 0 the separate calls would make (compute_pitch of
    its format); the library, with no device, fails with E_FAIL as every compute entry point does."""
    c = Call(**kw)
    hr, out = c.plan(planner)
    assert hr == F.S_OK, (name, hex(hr))
    assert out[:5] == want, (name, out)
    if out[0] or out[1]:
        assert out[5] == F.compute_pitch(out[2], out[3], out[4])[0]
    hr = c.library()
    assert hr == (F.E_FAIL if NO_DEVICE else F.S_OK), (name, hex(hr))


def ref_decompress(oracle, blocks, w, h, fmt, dst_fmt, nbytes):
    """the reference's Decompress of one w x h image into dst_fmt (0: DXGI_FORMAT_UNKNOWN), copied into `nbytes` bytes; (hr, bytes)"""
    out = np.zeros(nbytes, np.uint8)
    hr = oracle.L.ref_decompress(blocks.ctypes.data, w, h, fmt, dst_fmt, out.ctypes.data, nbytes)
    return F.hr_u32(hr), out


# formats whose Decompress results are the same bytes whatever the blocks: the reference writes a one-channel source's red into
# A8_UNORM's alpha as it writes it into R8_UNORM's red
BYTE_TWINS = {61: {65}}


def test_default_decompress_is_the_references(planner, oracle):
    """For every BC format, the format the planner decompresses to when asked for UNKNOWN is the one the reference's own
    Decompress(..., DXGI_FORMAT_UNKNOWN, ...) writes: that result has exactly the size of the planner's format (one byte less does
    not hold it) and its bytes, and no other implemented format of that size gives those bytes (but a byte twin)."""
    w = h = 16
    rng = np.random.default_rng(11)
    for fmt in sorted(F.BLOCK_BYTES):
        blocks = rng.integers(0, 256, (w // 4) * (h // 4) * F.BLOCK_BYTES[fmt], dtype=np.uint8)
        hr, out = Call(fmt, w, h, source=src(), dst_fmt=98 if fmt not in (95, 96) else 95).plan(planner)
        assert hr == F.S_OK, (fmt, hex(hr))
        mine = out[2]
        n = w * h * F.BYTES_PER_PIXEL[mine]
        hr, default = ref_decompress(oracle, blocks, w, h, fmt, 0, n)
        assert hr == F.S_OK, (fmt, hex(hr))
        assert ref_decompress(oracle, blocks, w, h, fmt, 0, n - 1)[0] != F.S_OK, (fmt, "the default result is larger")
        same = [f for f, bpp in sorted(F.BYTES_PER_PIXEL.items()) if bpp == F.BYTES_PER_PIXEL[mine]
                and _equal(ref_decompress(oracle, blocks, w, h, fmt, f, n), default)]
        assert mine in same and set(same) - {mine} <= BYTE_TWINS.get(mine, set()), (fmt, mine, same)


def _equal(result, want):
    hr, got = result
    return hr == F.S_OK and np.array_equal(got, want)
