"""CPU suite: dxb200_levels_from's argument checks and plans, without a device.  Each failing call returns the HRESULT of the call's
own rules (levels == 0, a Resize with levels > 1, alphaReference > 0) or of the first of the separate calls it stands for that would
fail (dxb200_decompress, dxb200_resize, dxb200_apply_channel_steps with the swizzle, dxb200_convert or the unconverted dst,
dxb200_apply_channel_steps with the later steps, dxb200_premultiply_alpha, dxb200_compress, dxb200_is_alpha_all_opaque), through the
library and through its planner on the host (tests/emul/levels_from.cpp).  A valid call's plan says which launches a chunk runs,
the decompress format, the working format and whether a BC base passes through; with one level it is the plan of the generating
call with the same arguments, less its mips."""
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
NOUT = 14
SW, KEY, INV, REC, UNORM = 1 << 16, 1 << 17, 1 << 18, 1 << 19, 1 << 20
ARGS = [IP, C.c_size_t, C.c_size_t, C.POINTER(capi.ChainSource), C.POINTER(capi.ChannelSteps), C.c_uint32, C.c_uint32, C.c_uint32,
        C.c_float, C.POINTER(capi.ChainSteps), IP]


@pytest.fixture(scope="module")
def em(tmp_path_factory):
    E = host_lib("levels_from.cpp", tmp_path_factory.mktemp("levels_from_emul"), os.path.join(ROOT, "tests", "emul"))
    E.emul_plan_levels_from.argtypes = ARGS + [C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]
    E.emul_plan_levels_from.restype = C.c_int32
    E.emul_plan_generating.argtypes = ARGS + [C.POINTER(C.c_uint64)]
    E.emul_plan_generating.restype = C.c_int32
    return E


def _img(w, h, fmt, ptr=True, row_pitch=0):
    p = BUF.ctypes.data if ptr else None
    if fmt in F.BYTES_PER_PIXEL or fmt in F.BLOCK_BYTES:
        return capi.make_image(p, w, h, fmt, row_pitch)
    return capi.Image(w, h, fmt, 0, 0, p)


def _sizes(w, h, levels):
    out = []
    for _ in range(levels):
        out.append((w, h))
        w, h = max(1, w // 2), max(1, h // 2)
    return out


def _levels(fmt, sizes, items, bad=None):
    """items x len(sizes) images of fmt; bad = (index, field, value) changes image index (item-major); field "pitch" sets a row
    pitch"""
    out = [_img(w, h, fmt) for _ in range(items) for (w, h) in sizes]
    if bad is not None:
        i, field, value = bad
        if field == "pitch":
            out[i] = _img(out[i].width, out[i].height, fmt, row_pitch=value)
        else:
            setattr(out[i], field, value)
    return out


def _args(bf, sizes, items, src_kw, ch_kw, df, cf=0, flags=0, steps=None, base_bad=None, dst_bad=None, levels=None):
    source = capi.chain_source(**src_kw) if src_kw is not None else None
    channels = capi.channel_steps(**ch_kw) if ch_kw is not None else None
    osizes = [(source.width, source.height)] if len(sizes) == 1 and source is not None and source.width and source.height else sizes
    base = capi.images(_levels(bf, sizes, items, base_bad)) if bf is not None else None
    dst = None if dst_bad == "null" else capi.images(_levels(df, osizes, items, dst_bad))
    return (base, items, len(sizes) if levels is None else levels, C.byref(source) if source is not None else None,
            C.byref(channels) if channels is not None else None, df, cf, flags, 0.5, C.byref(steps) if steps is not None else None, dst)


S16 = _sizes(16, 16, 5)             # 16x16 down to 1x1: partial blocks at 2x2 and 1x1
PM = capi.chain_steps(0.0, True)
# (name, base fmt, sizes, items, source kwargs, channels kwargs, dst fmt, convert filter, steps, base change, dst change, levels
#  (None: len(sizes)), HRESULT, the call that fails first); a change is (image index, field, value), image index = item * levels + l
CASES = [
    # the call's own rules
    ("levels_0", 28, S16, 1, None, None, 28, 0, None, None, None, 0, E_INVALIDARG, "levels"),
    ("levels_0_before_coverage", 28, S16, 1, None, None, 28, 0, capi.chain_steps(0.5), None, None, 0, E_INVALIDARG, "levels"),
    ("resize_with_levels", 28, S16, 1, dict(width=8, height=8), None, 28, 0, None, None, None, None, E_INVALIDARG, "resize rule"),
    ("resize_width_only_with_levels", 77, S16, 1, dict(width=12, height=16), None, 98, 0, None, None, None, None, E_INVALIDARG, "resize rule"),
    ("resize_before_coverage", 28, S16, 1, dict(width=8, height=8), None, 28, 0, capi.chain_steps(0.5), None, None, None, E_INVALIDARG,
     "resize rule"),
    ("coverage", 28, S16, 1, None, None, 28, 0, capi.chain_steps(0.5), None, None, None, E_INVALIDARG, "coverage rule"),
    ("coverage_before_decompress", 77, S16, 1, dict(decompress_format=3), None, 98, 0, capi.chain_steps(0.5, True), None, None, None,
     E_INVALIDARG, "coverage rule"),
    ("null_base", None, S16, 1, None, None, 28, 0, None, None, None, None, E_INVALIDARG, "all"),
    ("source_one_size", 28, S16[:1], 1, dict(width=8), None, 10, 0, None, None, None, None, E_INVALIDARG, "source"),
    ("source_one_size_equal_width", 28, S16, 1, dict(width=16), None, 10, 0, None, None, None, None, E_INVALIDARG, "source"),
    # Decompress, every level of the base
    ("decompress_to_bc", 77, S16, 1, dict(decompress_format=71), None, 98, 0, None, None, None, None, E_INVALIDARG, "decompress"),
    ("decompress_unimplemented", 77, S16, 1, dict(decompress_format=3), None, 98, 0, None, None, None, None, E_NOT_SUPPORTED, "decompress"),
    ("base_level2_format_bc", 77, S16, 2, None, None, 98, 0, None, (7, "format", 71), None, None, E_INVALIDARG, "decompress"),
    ("base_level3_pixels_bc", 77, S16, 1, None, None, 28, 0, None, (3, "pixels", None), None, None, E_POINTER, "decompress"),
    ("base_level1_bc_pitch", 71, S16, 1, None, None, 28, 0, None, (1, "pitch", 20), None, None, E_INVALIDARG, "decompress"),
    ("pass_through_decompress_checked", 71, S16, 1, dict(decompress_format=3), None, 71, 0, None, None, None, None, E_NOT_SUPPORTED,
     "decompress"),
    ("pass_through_base_level2_pixels", 71, S16, 1, None, None, 71, 0, None, (2, "pixels", None), None, None, E_POINTER, "decompress"),
    # Resize (one level)
    ("resize_box_odd", 28, S16[:1], 1, dict(width=5, height=5, resize_filter=F.TEX_FILTER_BOX), None, 10, 0, None, None, None, None, E_FAIL,
     "resize"),
    ("resize_bc_base_unknown_filter", 77, S16[:1], 1, dict(width=8, height=8, resize_filter=0x700000), None, 98, 0, None, None, None, None,
     E_NOT_SUPPORTED, "resize"),
    # the swizzle and masks
    ("swizzle_element", 2, S16, 1, None, dict(swizzle=(0, 1, 2, 7), invert_y=True), 28, 0, None, None, None, None, E_INVALIDARG, "swizzle"),
    ("mask_bit", 2, S16, 1, None, dict(zero_mask=0x20), 98, 0, None, None, None, None, E_INVALIDARG, "swizzle"),
    ("swizzle_base_level2_format", 28, S16, 1, None, dict(swizzle=(2, 1, 0, 3)), 10, 0, None, (2, "format", 87), None, None, E_FAIL, "swizzle"),
    ("swizzle_base_level4_pixels", 28, S16, 2, None, dict(swizzle=(2, 1, 0, 3)), 10, 0, None, (9, "pixels", None), None, None, E_POINTER,
     "swizzle"),
    # Convert, or the unconverted dst
    ("base_level2_format_convert", 28, S16, 1, None, None, 10, 0, None, (2, "format", 87), None, None, E_INVALIDARG, "convert"),
    ("base_level1_pixels_convert", 28, S16, 1, None, None, 10, 0, None, (1, "pixels", None), None, None, E_POINTER, "convert"),
    ("dithered_b5g6r5", 28, S16, 1, None, None, 85, F.TEX_FILTER_DITHER, None, None, None, None, E_NOT_SUPPORTED, "convert"),
    ("diffused_b4g4r4a4", 28, S16, 1, None, None, 115, F.TEX_FILTER_DITHER_DIFFUSION, None, None, None, None, E_NOT_SUPPORTED, "convert"),
    ("target_unimplemented", 2, S16, 1, None, None, 3, 0, None, None, None, None, E_NOT_SUPPORTED, "convert"),
    ("null_dst_convert", 2, S16, 1, None, None, 28, 0, None, None, "null", None, E_INVALIDARG, "convert"),
    ("dst_level2_size_convert", 2, S16, 1, None, None, 28, 0, None, None, (2, "width", 8), None, E_FAIL, "convert"),
    ("dst_level3_format_convert", 2, S16, 1, None, None, 28, 0, None, None, (3, "format", 87), None, E_INVALIDARG, "convert"),
    ("dst_level1_pixels_convert", 2, S16, 1, None, None, 28, 0, None, None, (1, "pixels", None), None, E_POINTER, "convert"),
    ("dst_level2_format_unconverted", 28, S16, 1, None, dict(invert_y=True), 28, 0, None, None, (2, "format", 87), None, E_INVALIDARG,
     "unconverted"),
    ("dst_level3_size_unconverted", 77, S16, 2, None, None, 28, 0, None, None, (8, "height", 8), None, E_INVALIDARG, "unconverted"),
    ("dst_level1_pixels_unconverted", 28, S16, 1, None, None, 28, 0, None, None, (1, "pixels", None), None, E_POINTER, "unconverted"),
    ("null_dst_unconverted", 28, S16, 1, None, None, 28, 0, None, None, "null", None, E_INVALIDARG, "unconverted"),
    ("pass_through_dst_level1_bc_pitch", 71, S16, 1, None, None, 71, 0, None, None, (1, "pitch", 20), None, E_INVALIDARG, "pass-through"),
    ("pass_through_dst_level2_format", 71, S16, 1, None, None, 71, 0, None, None, (2, "format", 72), None, E_INVALIDARG, "pass-through"),
    ("pass_through_dst_level4_size", 98, S16, 1, None, None, 98, 0, None, None, (4, "width", 2), None, E_INVALIDARG, "pass-through"),
    ("pass_through_dst_level3_pixels", 98, S16, 1, None, None, 98, 0, None, None, (3, "pixels", None), None, E_POINTER, "pass-through"),
    # the later channel steps
    ("color_key_base_level2_pixels", 28, S16, 1, None, dict(color_key=0x102030), 28, 0, None, (2, "pixels", None), None, None, E_POINTER,
     "later steps"),
    ("color_key_base_level3_format", 28, S16, 1, None, dict(color_key=0x102030), 28, 0, None, (3, "format", 87), None, None, E_FAIL,
     "later steps"),
    # premultiply
    ("premultiply_target_without_alpha", 28, S16, 1, None, None, 85, 0, PM, None, None, None, E_NOT_SUPPORTED, "premultiply"),
    ("premultiply_bc4_working_r8", 80, S16, 1, None, None, 98, 0, PM, None, None, None, E_NOT_SUPPORTED, "premultiply"),
    ("premultiply_base_level2_pixels_bc_target", 28, S16, 1, None, None, 98, 0, PM, (2, "pixels", None), None, None, E_POINTER, "premultiply"),
    # Compress
    ("null_dst_compress", 28, S16, 1, None, None, 98, 0, None, None, "null", None, E_INVALIDARG, "compress"),
    ("dst_level2_format_compress", 77, S16, 1, None, None, 98, 0, None, None, (2, "format", 71), None, E_INVALIDARG, "compress"),
    ("dst_level1_size_compress", 28, S16, 1, None, None, 71, 0, None, None, (1, "width", 4), None, E_FAIL, "compress"),
    ("dst_level3_pixels_compress", 77, S16, 2, None, None, 72, 0, None, None, (8, "pixels", None), None, E_POINTER, "compress"),
    ("dst_level1_bc_pitch_compress", 2, S16, 1, None, None, 95, 0, None, None, (1, "pitch", 20), None, E_INVALIDARG, "compress"),
    ("base_level2_pixels_compress", 28, S16, 1, None, None, 98, 0, None, (2, "pixels", None), None, None, E_POINTER, "compress"),
    ("base_level3_format_compress", 28, S16, 1, None, None, 98, 0, None, (3, "format", 87), None, None, E_INVALIDARG, "compress"),
    # a base that is only copied
    ("copy_base_level2_pixels", 28, S16, 1, None, None, 28, 0, None, (2, "pixels", None), None, None, E_POINTER, "copy"),
    ("copy_base_level3_format", 28, S16, 1, None, None, 28, 0, None, (3, "format", 87), None, None, E_INVALIDARG, "copy"),
    ("copy_premultiply_base_level1_pixels", 28, S16, 1, None, None, 28, 0, PM, (1, "pixels", None), None, None, E_POINTER, "copy"),
    ("pass_through_base_level2_bc_pitch", 71, S16, 1, None, None, 71, 0, None, (2, "pitch", 20), None, None, E_INVALIDARG, "decompress"),
    ("copy_unimplemented_r8g8b8a8_uint", 30, S16, 2, None, None, 30, 0, None, None, None, None, E_NOT_SUPPORTED, "copy"),
    ("copy_unimplemented_r16_uint", 57, S16, 1, None, None, 57, 0, None, None, None, None, E_NOT_SUPPORTED, "copy"),
    ("copy_zero_width_level2", 28, S16, 1, None, None, 28, 0, None, (2, "width", 0), (2, "width", 0), None, E_INVALIDARG, "copy"),
    ("copy_zero_size_level3_invert_y", 49, S16, 2, None, dict(invert_y=True), 49, 0, None, (8, "height", 0), (8, "height", 0), None,
     E_INVALIDARG, "copy"),
    ("copy_zero_size_level1_color_key", 28, S16, 1, None, dict(color_key=0x102030), 28, 0, None, (1, "width", 0), (1, "width", 0), None,
     E_INVALIDARG, "copy"),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_hresults(case, em):
    name, bf, sizes, items, src_kw, ch_kw, df, cf, steps, base_bad, dst_bad, levels, want = case[:13]
    args = _args(bf, sizes, items, src_kw, ch_kw, df, cf, 0, steps, base_bad, dst_bad, levels)
    opaque = C.c_int32(-1)
    assert F.hr_u32(L.dxb200_levels_from(*args, C.byref(opaque))) == want, name
    assert F.hr_u32(L.dxb200_levels_from(*args, None)) == want, name
    out = (C.c_uint64 * NOUT)()
    assert F.hr_u32(em.emul_plan_levels_from(*args, C.byref(opaque), out)) == want, name
    assert opaque.value == -1


def test_every_case_fixed_plans(em):
    """each failing case plans once its one change is undone: the table tests the check it names and no other"""
    for case in CASES:
        name, bf, sizes, items, src_kw, ch_kw, df, cf, steps, base_bad, dst_bad, levels, _, first = case
        if first in ("levels", "resize rule", "coverage rule", "all", "source") or base_bad is None and dst_bad is None:
            continue
        args = _args(bf, sizes, items, src_kw, ch_kw, df, cf, 0, steps, None, None, levels)
        assert em.emul_plan_levels_from(*args, None, None) == 0, name


# (name, base fmt, sizes, items, source kwargs, channels kwargs, dst fmt, steps,
#  { decompress, resize, channels, convert, post, premultiply, compress, decompress format, working format, step flags, pass-through })
PLANS = [
    ("bc3_to_bc7_premultiply", 77, S16, 3, None, None, 98, PM, [1, 0, 0, 0, 0, 1, 1, 28, 28, 0, 0]),
    ("bc5_invert_y_to_bc5", 83, S16, 2, None, dict(invert_y=True), 83, None, [1, 0, 1, 0, 0, 0, 1, 49, 49, INV | UNORM, 0]),
    ("bc5_reconstruct_z_to_bc5_wide", 83, S16, 1, None, dict(reconstruct_z=True), 83, None, [1, 0, 1, 0, 0, 0, 1, 28, 28, REC | UNORM, 0]),
    ("bc1_passes_through", 71, S16, 2, None, None, 71, None, [0, 0, 0, 0, 0, 0, 0, 0, 71, 0, 1]),
    ("bc7_passes_through_with_source", 98, S16, 1, dict(decompress_format=2), None, 98, None, [0, 0, 0, 0, 0, 0, 0, 0, 98, 0, 1]),
    ("bc1_to_bc1_srgb_reencodes", 71, S16, 1, None, None, 72, None, [1, 0, 0, 0, 0, 0, 1, 28, 28, 0, 0]),
    ("bc3_premultiply_reencodes", 77, S16, 1, None, None, 77, PM, [1, 0, 0, 0, 0, 1, 1, 28, 28, 0, 0]),
    ("bc7_to_rgba8_no_convert", 98, S16, 1, None, None, 28, None, [1, 0, 0, 0, 0, 0, 0, 28, 28, 0, 0]),
    ("bc7_to_rgba8_srgb_converts", 98, S16, 1, None, None, 29, None, [1, 0, 0, 1, 0, 0, 0, 28, 28, 0, 0]),
    ("bc3_to_rgba32f_decompress_format", 77, S16, 1, dict(decompress_format=2), None, 10, None, [1, 0, 0, 1, 0, 0, 0, 2, 2, 0, 0]),
    ("rgba8_copied", 28, S16, 2, None, None, 28, None, [0, 0, 0, 0, 0, 0, 0, 0, 28, 0, 0]),
    ("rgba8_premultiply_in_dst", 28, S16, 1, None, None, 28, PM, [0, 0, 0, 0, 0, 1, 0, 0, 28, 0, 0]),
    ("rgba32f_to_bc6h", 2, S16, 1, None, None, 95, None, [0, 0, 0, 0, 0, 0, 1, 0, 2, 0, 0]),
    ("rgba16f_swizzle_to_bc1", 10, S16, 1, None, dict(swizzle=(2, 1, 0, 3)), 71, None, [0, 0, 1, 0, 0, 0, 1, 0, 10, SW, 0]),
    ("rgba8_swizzle_color_key_to_bc3_one_launch", 28, S16, 1, None, dict(swizzle=(2, 1, 0, 3), color_key=0), 77, None,
     [0, 0, 1, 0, 0, 0, 1, 0, 28, SW | KEY | UNORM, 0]),
    ("rgba8_swizzle_convert_color_key", 28, S16, 1, None, dict(swizzle=(2, 1, 0, 3), color_key=0), 115, None,
     [0, 0, 1, 1, 1, 0, 0, 0, 28, SW | UNORM, 0]),
    ("one_level_resize_then_convert", 28, [(1000, 600)], 2, dict(width=512, height=512, resize_filter=F.TEX_FILTER_LINEAR), None, 10, None,
     [0, 1, 0, 1, 0, 0, 0, 0, 28, 0, 0]),
    ("one_level_bc_resize_to_bc7", 77, [(64, 64)], 1, dict(width=32, height=32), None, 98, None, [1, 1, 0, 0, 0, 0, 1, 28, 28, 0, 0]),
    ("levels_that_do_not_halve", 28, [(64, 48), (40, 40), (3, 5), (1, 1)], 2, None, dict(invert_y=True), 10, None,
     [0, 0, 0, 1, 1, 0, 0, 0, 28, 0, 0]),
    ("same_size_source_keeps_levels", 77, S16, 1, dict(width=16, height=16), None, 98, None, [1, 0, 0, 0, 0, 0, 1, 28, 28, 0, 0]),
]


def _plan(em, args):
    out = (C.c_uint64 * NOUT)()
    hr = em.emul_plan_levels_from(*args, None, out)
    assert F.hr_u32(hr) == 0, hex(F.hr_u32(hr))
    return list(out)


@pytest.mark.parametrize("plan", PLANS, ids=[p[0] for p in PLANS])
def test_plans(plan, em):
    name, bf, sizes, items, src_kw, ch_kw, df, steps, want = plan
    out = _plan(em, _args(bf, sizes, items, src_kw, ch_kw, df, 0, 0, steps))
    got = out[0:7] + out[9:11] + [out[11] & (SW | KEY | INV | REC | UNORM), out[12]]
    assert got == want, (name, got)
    assert out[7] == 0 and out[8] == 0, name          # no mips, no coverage


def test_alpha_scan_planned_only_when_asked(em):
    """the scan is planned for a dst format with alpha when alphaAllOpaque is given, a passed-through BC1 chain included"""
    for bf, df, scan in ((71, 71, 1), (77, 98, 1), (83, 83, 0), (28, 85, 0), (2, 10, 1)):
        args = _args(bf, S16, 1, None, None, df)
        out = (C.c_uint64 * NOUT)()
        opaque = C.c_int32(-1)
        assert em.emul_plan_levels_from(*args, C.byref(opaque), out) == 0
        assert out[13] == scan, (bf, df)
        assert em.emul_plan_levels_from(*args, None, out) == 0
        assert out[13] == 0


# one level: (name, base fmt, w, h, source kwargs, channels kwargs, dst fmt, steps)
ONE_LEVEL = [
    ("bc3_to_bc7_premultiply", 77, 64, 64, dict(), None, 98, PM),
    ("bc5_invert_y_to_bc5", 83, 64, 64, dict(), dict(invert_y=True), 83, None),
    ("bc4_swizzle_to_bc1", 80, 32, 32, dict(), dict(swizzle=(0, 0, 0, 3)), 71, None),
    ("rgba8_resize_to_bc3", 28, 100, 60, dict(width=64, height=32, resize_filter=F.TEX_FILTER_CUBIC), dict(color_key=0x102030), 77, None),
    ("bc7_resize_to_rgba16f", 98, 64, 64, dict(width=32, height=16), dict(swizzle=(1, 0, 2, 3), invert_y=True), 10, PM),
    ("rgba32f_to_rgba8_srgb", 2, 40, 24, None, None, 29, None),
    ("rgba8_swizzle_no_convert", 28, 40, 24, None, dict(swizzle=(2, 1, 0, 3), reconstruct_z=True), 28, None),
    ("bc3_decompress_format_to_b4g4r4a4", 77, 32, 32, dict(decompress_format=2), dict(swizzle=(3, 2, 1, 0), color_key=0), 115, PM),
]


@pytest.mark.parametrize("case", ONE_LEVEL, ids=[c[0] for c in ONE_LEVEL])
def test_one_level_plan_is_the_generating_plan(case, em):
    """levels == 1: the same launches, decompress format, working format and step word as dxb200_mipmaps_compress_from_channels (BC
    target) or dxb200_mipmaps_convert_from (uncompressed target) with the same arguments and two levels, minus the mips"""
    name, bf, w, h, src_kw, ch_kw, df, steps = case
    mine = _plan(em, _args(bf, [(w, h)], 2, src_kw, ch_kw, df, 0, 0, steps))
    source = capi.chain_source(**src_kw) if src_kw is not None else None
    channels = capi.channel_steps(**ch_kw) if ch_kw is not None else None
    lw, lh = (source.width, source.height) if source is not None and source.width else (w, h)
    base = capi.images(_levels(bf, [(w, h)], 2))
    dst = capi.images(_levels(df, _sizes(lw, lh, 2), 2))
    theirs = (C.c_uint64 * NOUT)()
    hr = em.emul_plan_generating(base, 2, 2, C.byref(source) if source is not None else None, C.byref(channels) if channels is not None else None,
                                 df, 0, 0, 0.5, C.byref(steps) if steps is not None else None, dst, theirs)
    assert F.hr_u32(hr) == 0, (name, hex(F.hr_u32(hr)))
    theirs = list(theirs)
    assert theirs[7] == 1 and mine[7] == 0, name
    for out in (mine, theirs):          # the swizzle's bits of a step word count only when the swizzle is enabled
        out[11] &= ~0 if out[11] & SW else ~0xFFFF
    assert mine[:7] + mine[8:13] == theirs[:7] + theirs[8:13], (name, mine, theirs)
