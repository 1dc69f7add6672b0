"""CPU suite: dxb200_mipmaps_convert_from's argument checks and plans, without a device.  Each failing call returns the HRESULT of the
first of the separate calls it stands for that would fail (dxb200_decompress, dxb200_resize, dxb200_apply_channel_steps with the
swizzle, dxb200_convert, dxb200_apply_channel_steps with the later steps, dxb200_generate_mipmaps, coverage, premultiply,
dxb200_is_alpha_all_opaque), through the library and through its planner on the host (tests/emul/convert_from.cpp).  A valid call's
plan says which launches a chunk runs, the Convert's source format and the chain's level 0."""
import ctypes as C
import os

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests.bc7_ranking_build import host_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = capi.lib
IP = C.POINTER(capi.Image)
E_INVALIDARG, E_POINTER, E_FAIL, E_NOT_SUPPORTED = 0x80070057, 0x80004003, 0x80004005, 0x80070032
BUF = np.zeros(1 << 22, np.uint8)
NOUT = 12


@pytest.fixture(scope="module")
def em(tmp_path_factory):
    E = host_lib("convert_from.cpp", tmp_path_factory.mktemp("convert_from_emul"), os.path.join(ROOT, "tests", "emul"))
    E.emul_plan_mipmaps_convert_from.argtypes = [IP, C.c_size_t, C.POINTER(capi.ChainSource), C.POINTER(capi.ChannelSteps), C.c_uint32,
                                                 C.c_uint32, C.c_float, C.c_size_t, C.c_uint32, C.POINTER(capi.ChainSteps), IP,
                                                 C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]
    E.emul_plan_mipmaps_convert_from.restype = C.c_int32
    return E


def _img(w, h, fmt, ptr=True, row_pitch=0):
    p = BUF.ctypes.data if ptr else None
    if fmt in F.BYTES_PER_PIXEL or fmt in F.BLOCK_BYTES:
        return capi.make_image(p, w, h, fmt, row_pitch)
    return capi.Image(w, h, fmt, 0, 0, p)


def _chain(w, h, fmt, levels, items=1, bad=None, row_pitch=0):
    """dst: `items` chains of `levels` levels of fmt from w x h; bad = (level, field, value) changes one level of item 0"""
    out = []
    for _ in range(items):
        lw, lh = w, h
        for l in range(levels):
            out.append(_img(lw, lh, fmt, row_pitch=row_pitch if l == 0 else 0))
            lw, lh = max(1, lw // 2), max(1, lh // 2)
    if bad is not None:
        l, field, value = bad
        setattr(out[l], field, value)
    return out


# (name, base fmt, w, h, source kwargs (None: NULL), channels kwargs (None: NULL), dst fmt, convert filter, levels, dst change,
# chain steps, HRESULT, the separate call that fails first)
CASES = [
    ("null_base", None, 16, 16, None, None, 28, 0, 2, None, None, E_INVALIDARG, "all"),
    ("source_one_size", 28, 16, 16, dict(width=8), None, 10, 0, 2, None, None, E_INVALIDARG, "source"),
    ("decompress_to_bc", 77, 16, 16, dict(decompress_format=71), None, 10, 0, 2, None, None, E_INVALIDARG, "decompress"),
    ("decompress_unimplemented", 77, 16, 16, dict(decompress_format=3), None, 10, 0, 2, None, None, E_NOT_SUPPORTED, "decompress"),
    ("resize_box_odd", 28, 16, 16, dict(width=5, height=5, resize_filter=F.TEX_FILTER_BOX), None, 10, 0, 2, None, None, E_FAIL, "resize"),
    ("swizzle_on_bc_base_without_source", 77, 16, 16, None, dict(swizzle=(2, 1, 0, 3)), 28, 0, 2, None, None, E_NOT_SUPPORTED, "swizzle"),
    ("swizzle_element", 2, 16, 16, None, dict(swizzle=(0, 1, 2, 7), invert_y=True), 28, 0, 2, None, None, E_INVALIDARG, "swizzle"),
    ("mask_bit", 2, 16, 16, None, dict(zero_mask=0x20), 28, 0, 2, None, None, E_INVALIDARG, "swizzle"),
    ("swizzle_before_bc_target", 2, 16, 16, None, dict(swizzle=(9, 1, 2, 3)), 98, 0, 2, None, None, E_INVALIDARG, "swizzle"),
    ("bc_base_without_source", 77, 16, 16, None, None, 28, 0, 2, None, None, E_INVALIDARG, "convert"),
    ("bc_target", 2, 16, 16, None, None, 98, 0, 2, None, None, E_INVALIDARG, "convert"),
    ("bc_target_equal_to_base", 98, 16, 16, None, None, 98, 0, 2, None, None, E_INVALIDARG, "convert"),
    ("bc_target_after_decompress", 77, 16, 16, dict(), dict(invert_y=True), 77, 0, 2, None, None, E_INVALIDARG, "convert"),
    ("dithered_b5g6r5", 28, 16, 16, None, None, 85, F.TEX_FILTER_DITHER, 2, None, None, E_NOT_SUPPORTED, "convert"),
    ("diffused_b4g4r4a4", 28, 16, 16, None, None, 115, F.TEX_FILTER_DITHER_DIFFUSION, 2, None, None, E_NOT_SUPPORTED, "convert"),
    ("unknown_dither_bit", 2, 16, 16, None, None, 28, 0x40000, 2, None, None, E_NOT_SUPPORTED, "convert"),
    ("target_unimplemented", 2, 16, 16, None, None, 3, 0, 2, None, None, E_NOT_SUPPORTED, "convert"),
    ("null_dst", 2, 16, 16, None, None, 28, 0, 2, "null", None, E_INVALIDARG, "convert"),
    ("dst_level0_format", 2, 16, 16, None, None, 28, 0, 2, (0, "format", 87), None, E_INVALIDARG, "convert"),
    ("dst_level0_size", 2, 16, 16, None, None, 28, 0, 2, (0, "width", 8), None, E_FAIL, "convert"),
    ("dst_level0_pixels", 2, 16, 16, None, dict(color_key=0x102030), 28, 0, 2, (0, "pixels", None), None, E_POINTER, "convert"),
    ("dst_level0_format_without_convert", 28, 16, 16, None, None, 28, 0, 2, (0, "format", 87), None, E_INVALIDARG, "level 0"),
    ("dst_level0_size_without_convert", 28, 16, 16, None, None, 28, 0, 2, (0, "height", 8), None, E_INVALIDARG, "level 0"),
    ("color_key_on_null_level0", 28, 16, 16, None, dict(color_key=0x102030), 28, 0, 2, (0, "pixels", None), None, E_POINTER, "later steps"),
    ("dst_level1_format", 2, 16, 16, None, None, 28, 0, 2, (1, "format", 87), None, E_INVALIDARG, "mips"),
    ("dst_level1_size", 2, 16, 16, None, dict(invert_y=True), 28, 0, 2, (1, "width", 4), None, E_INVALIDARG, "mips"),
    ("dst_level1_pixels", 2, 16, 16, None, None, 28, 0, 2, (1, "pixels", None), None, E_POINTER, "mips"),
    ("levels_1", 2, 16, 16, None, None, 28, 0, 1, None, None, E_INVALIDARG, "mips"),
    ("levels_too_many", 2, 16, 16, None, None, 28, 0, 6, None, None, E_INVALIDARG, "mips"),
    ("levels_1_after_failing_convert", 28, 16, 16, None, None, 85, F.TEX_FILTER_DITHER, 1, None, None, E_NOT_SUPPORTED, "convert"),
    ("levels_0_after_failing_convert", 28, 16, 16, None, None, 85, F.TEX_FILTER_DITHER, 0, None, None, E_NOT_SUPPORTED, "convert"),
    ("levels_0", 2, 16, 16, None, None, 28, 0, 0, None, None, E_INVALIDARG, "mips"),
    ("levels_0_without_convert", 28, 16, 16, None, dict(color_key=0x102030), 28, 0, 0, None, None, E_INVALIDARG, "mips"),
    ("premultiply_target_without_alpha", 28, 16, 16, None, None, 85, 0, 2, None, capi.chain_steps(0.0, True), E_NOT_SUPPORTED, "premultiply"),
    ("premultiply_r16g16_snorm", 2, 16, 16, None, None, 37, 0, 2, None, capi.chain_steps(0.5, True), E_NOT_SUPPORTED, "premultiply"),
]


def _args(case):
    name, bf, w, h, src_kw, ch_kw, df, cf, levels, change, steps = case[:11]
    source = capi.chain_source(**src_kw) if src_kw is not None else None
    channels = capi.channel_steps(**ch_kw) if ch_kw is not None else None
    lw, lh = (source.width or w, source.height or h) if source is not None and src_kw.get("height") else (w, h)
    base = capi.images([_img(w, h, bf)]) if bf is not None else None
    dst = None if change == "null" else capi.images(_chain(lw, lh, df, max(levels, 1), bad=change))
    return (base, 1, C.byref(source) if source is not None else None, C.byref(channels) if channels is not None else None, df, cf, 0.5,
            levels, 0, C.byref(steps) if steps is not None else None, dst)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_hresults(case, em):
    want = case[11]
    args = _args(case)
    opaque = C.c_int32(-1)
    assert F.hr_u32(L.dxb200_mipmaps_convert_from(*args, C.byref(opaque))) == want, case[0]
    assert F.hr_u32(L.dxb200_mipmaps_convert_from(*args, None)) == want, case[0]
    out = (C.c_uint64 * NOUT)()
    assert F.hr_u32(em.emul_plan_mipmaps_convert_from(*args, C.byref(opaque), out)) == want, case[0]
    assert opaque.value == -1


# Two items whose second base differs: (name, base 1's format (None: base 0's), base 1's pixels, channels kwargs, dst fmt, HRESULT of the
# first separate call that fails).  Without a front step or a Convert the base is level 0 itself: the later steps read it, and
# GenerateMipMaps meets it as level 0 of the chain.
BASES = [
    ("mixed_formats", 2, True, None, 28, E_INVALIDARG, "mips"),
    ("mixed_formats_color_key", 2, True, dict(color_key=0x102030), 28, E_FAIL, "later steps"),
    ("mixed_formats_swizzle", 2, True, dict(swizzle=(2, 1, 0, 3)), 28, E_FAIL, "swizzle"),
    ("mixed_formats_convert", 2, True, None, 10, E_INVALIDARG, "convert"),
    ("null_pixels", None, False, None, 28, E_POINTER, "mips"),
    ("null_pixels_color_key", None, False, dict(color_key=0x102030), 28, E_POINTER, "later steps"),
    ("null_pixels_invert_y", None, False, dict(invert_y=True), 28, E_POINTER, "later steps"),
    ("null_pixels_convert", None, False, None, 10, E_POINTER, "convert"),
]


@pytest.mark.parametrize("case", BASES, ids=[c[0] for c in BASES])
def test_every_base_is_checked(case, em):
    name, fmt1, ptr1, ch_kw, df, want, _ = case
    base = capi.images([_img(16, 16, 28), _img(16, 16, fmt1 or 28, ptr=ptr1)])
    channels = capi.channel_steps(**ch_kw) if ch_kw is not None else None
    dst = capi.images(_chain(16, 16, df, 5, items=2))
    args = (base, 2, None, C.byref(channels) if channels is not None else None, df, 0, 0.5, 5, 0, None, dst)
    opaque = C.c_int32(-1)
    assert F.hr_u32(L.dxb200_mipmaps_convert_from(*args, C.byref(opaque))) == want, name
    out = (C.c_uint64 * NOUT)()
    assert F.hr_u32(em.emul_plan_mipmaps_convert_from(*args, None, out)) == want, name
    # the same two items with base 1 fixed plan
    base[1] = _img(16, 16, 28)
    assert em.emul_plan_mipmaps_convert_from(*((base,) + args[1:]), None, out) == 0, name


def test_mip_filter_checks_after_the_convert(em):
    """GenerateMipMaps' BOX on a size that is not a power of two (E_FAIL) and an unknown filter mode (E_NOT_SUPPORTED), after a
    Convert that would pass, and after one that fails first"""
    base = capi.images([_img(12, 12, 2)])
    for df, cf, filt, want in ((28, 0, F.TEX_FILTER_BOX, E_FAIL), (28, 0, 0x700000, E_NOT_SUPPORTED), (98, 0, F.TEX_FILTER_BOX, E_INVALIDARG)):
        dst = capi.images(_chain(12, 12, df, 2))
        args = (base, 1, None, None, df, cf, 0.5, 2, filt, None, dst, None)
        assert F.hr_u32(L.dxb200_mipmaps_convert_from(*args)) == want, (df, filt)
        assert F.hr_u32(em.emul_plan_mipmaps_convert_from(*args, None)) == want, (df, filt)


def test_alpha_opaque_null_words_are_not_an_error(em):
    """the scan runs only when alphaAllOpaque is given: a format without alpha needs no scan either way"""
    for df, scan in ((10, 1), (85, 0), (26, 0)):
        base = capi.images([_img(16, 16, 2)])
        dst = capi.images(_chain(16, 16, df, 5))
        out = (C.c_uint64 * NOUT)()
        opaque = C.c_int32(-1)
        assert em.emul_plan_mipmaps_convert_from(base, 1, None, None, df, 0, 0.5, 5, 0, None, dst, C.byref(opaque), out) == 0
        assert out[11] == scan, df
        assert em.emul_plan_mipmaps_convert_from(base, 1, None, None, df, 0, 0.5, 5, 0, None, dst, None, out) == 0
        assert out[11] == 0


SW, KEY, INV, REC, UNORM = 1 << 16, 1 << 17, 1 << 18, 1 << 19, 1 << 20
# (name, base fmt, w, h, items, source kwargs, channels kwargs, dst fmt, dst row pitch (0: tight),
#  { decompress, resize, channels, convert, post, convert source, level-0 fmt, width, height, row pitch, step flags })
PLANS = [
    ("equal_formats", 10, 16, 16, 2, None, None, 10, 0, [0, 0, 0, 0, 0, 0, 10, 16, 16, 128, 0]),
    ("rgba32f_to_half", 2, 64, 32, 3, None, None, 10, 0, [0, 0, 0, 1, 0, 2, 10, 64, 32, 512, 0]),
    ("bc5_reconstruct_z_forces_rgba8_then_r8g8", 83, 16, 16, 1, dict(), dict(reconstruct_z=True), 49, 0,
     [1, 0, 0, 1, 1, 28, 49, 16, 16, 32, 0]),
    ("bc4_swizzle_forces_rgba8_then_r8g8_snorm", 80, 16, 16, 1, dict(), dict(swizzle=(0, 0, 0, 3)), 51, 0,
     [1, 0, 1, 1, 0, 28, 51, 16, 16, 32, SW | UNORM]),
    ("bc5_snorm_invert_y_to_r16g16_snorm", 84, 16, 16, 1, dict(), dict(invert_y=True), 37, 0, [1, 0, 0, 1, 1, 51, 37, 16, 16, 64, 0]),
    ("swizzle_only", 28, 16, 16, 1, None, dict(swizzle=(2, 1, 0, 3)), 87, 0, [0, 0, 1, 1, 0, 28, 87, 16, 16, 64, SW | UNORM]),
    ("later_steps_only", 2, 16, 16, 1, None, dict(invert_y=True, reconstruct_z=True), 28, 0, [0, 0, 0, 1, 1, 2, 28, 16, 16, 64, 0]),
    ("color_key_after_convert", 28, 16, 16, 1, None, dict(swizzle=(2, 1, 0, 3), color_key=0), 115, 0, [0, 0, 1, 1, 1, 28, 115, 16, 16, 32, SW | UNORM]),
    ("no_convert_one_launch", 28, 16, 16, 1, None, dict(swizzle=(1, 0, 2, 3), invert_y=True, reconstruct_z=True), 28, 0,
     [0, 0, 1, 0, 0, 0, 28, 16, 16, 64, SW | INV | REC | UNORM]),
    ("no_convert_later_steps_only", 28, 16, 16, 1, None, dict(color_key=0x4080C0), 28, 0, [0, 0, 1, 0, 0, 0, 28, 16, 16, 64, KEY | UNORM]),
    ("bc5_swizzle_and_reconstruct_z_no_convert", 83, 16, 16, 1, dict(), dict(swizzle=(1, 0, 2, 3), reconstruct_z=True), 28, 0,
     [1, 0, 1, 0, 0, 0, 28, 16, 16, 64, SW | REC | UNORM]),
    ("resize_in_front", 28, 1000, 600, 1, dict(width=512, height=512, resize_filter=F.TEX_FILTER_LINEAR), None, 10, 0,
     [0, 1, 0, 1, 0, 28, 10, 512, 512, 4096, 0]),
    ("caller_pitch", 2, 16, 16, 2, None, None, 28, 96, [0, 0, 0, 1, 0, 2, 28, 16, 16, 96, 0]),
]


@pytest.mark.parametrize("plan", PLANS, ids=[p[0] for p in PLANS])
def test_plans(plan, em):
    name, bf, w, h, items, src_kw, ch_kw, df, pitch, want = plan
    source = capi.chain_source(**src_kw) if src_kw is not None else None
    channels = capi.channel_steps(**ch_kw) if ch_kw is not None else None
    lw, lh = (source.width, source.height) if source is not None and source.width else (w, h)
    levels = F.count_mips(lw, lh)
    base = capi.images([_img(w, h, bf) for _ in range(items)])
    dst = capi.images(_chain(lw, lh, df, levels, items, row_pitch=pitch))
    out = (C.c_uint64 * NOUT)()
    hr = em.emul_plan_mipmaps_convert_from(base, items, C.byref(source) if source is not None else None,
                                           C.byref(channels) if channels is not None else None, df, 0, 0.5, levels, 0, None, dst, None, out)
    assert F.hr_u32(hr) == 0, (name, hex(F.hr_u32(hr)))
    got = list(out[:10]) + [out[10] & (SW | KEY | INV | REC | UNORM)]
    assert got == want, (name, got)
