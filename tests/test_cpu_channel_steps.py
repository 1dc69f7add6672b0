"""CPU suite: texconv's channel steps (swizzle, colour key, invert Y, reconstruct Z).  The HRESULTs of dxb200_apply_channel_steps
through the library, the emulator's planner and the reference's TransformImage; the HRESULTs of dxb200_mipmaps_compress_from_channels
against the first separate call that fails; reconstruct Z's UNORM rule against the reference's FormatDataType; the decompress format
texconv picks for BC4 / BC5 bases; and the emulator (the library's planner and per-pixel rule on the host) bit for bit against the
reference on every implemented uncompressed format, for each step alone and all four together."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import channel_steps_lib as CS
from tests import special_values as SV

L = capi.lib
E_INVALIDARG, E_POINTER, E_FAIL, E_NOT_SUPPORTED = 0x80070057, 0x80004003, 0x80004005, 0x80070032


@pytest.fixture(scope="module")
def ref(tmp_path_factory, oracle):
    return CS.Probe(tmp_path_factory.mktemp("channel_ref"))


@pytest.fixture(scope="module")
def em(tmp_path_factory):
    return CS.load_emul(tmp_path_factory.mktemp("channel_emul"))


# ---- dxb200_apply_channel_steps: HRESULTs --------------------------------------------------------------------------------------
BUF = np.zeros(1 << 16, np.uint8)


def _img(fmt=28, w=4, h=4, ptr=True, base=0):
    im = capi.make_image(BUF.ctypes.data + base if ptr else None, w, h, fmt) if fmt in F.BYTES_PER_PIXEL or fmt in F.BLOCK_BYTES \
        else capi.Image(w, h, fmt, 0, 0, BUF.ctypes.data if ptr else None)
    return im


def _chain(w, h, fmt):
    """the two-level destination chain of a w x h level 0"""
    return capi.images([capi.make_image(BUF.ctypes.data, w, h, fmt), capi.make_image(BUF.ctypes.data, max(1, w // 2), max(1, h // 2), fmt)])


GOOD = dict(invert_y=True)
# (name, source images, destination images (None: the sources), steps kwargs (None: NULL), n override, HRESULT, reference?)
CASES = [
    ("null_src", None, [_img()], GOOD, 1, E_INVALIDARG, True),
    ("zero_images", [_img()], [_img()], GOOD, 0, E_INVALIDARG, True),
    ("null_steps", [_img()], [_img()], None, 1, E_INVALIDARG, False),
    ("bc_format", [_img(71)], [_img(71)], GOOD, 1, E_NOT_SUPPORTED, True),
    ("bc7_format", [_img(98)], [_img(98)], GOOD, 1, E_NOT_SUPPORTED, True),
    ("typeless", [_img(27)], [_img(27)], GOOD, 1, E_NOT_SUPPORTED, True),
    ("not_implemented", [_img(3)], [_img(3)], GOOD, 1, E_NOT_SUPPORTED, False),
    ("too_wide", [_img(28, 1 << 32, 1)], [_img(28, 1 << 32, 1)], GOOD, 1, E_INVALIDARG, True),
    ("mixed_formats", [_img(28), _img(87)], [_img(28), _img(87)], GOOD, 2, E_FAIL, True),
    ("dst_size", [_img(28)], [_img(28, 4, 2)], GOOD, 1, E_FAIL, False),
    ("dst_format", [_img(28)], [_img(87)], GOOD, 1, E_FAIL, False),
    ("no_step", [_img()], [_img()], dict(), 1, E_INVALIDARG, True),
    ("no_step_before_null_pixels", [_img(ptr=False)], [_img()], dict(), 1, E_INVALIDARG, True),
    ("no_step_before_mixed_formats", [_img(28), _img(87)], [_img(28), _img(87)], dict(), 2, E_INVALIDARG, True),
    ("swizzle_element", [_img()], [_img()], dict(swizzle=(0, 1, 4, 3)), 1, E_INVALIDARG, False),
    ("zero_mask_bit", [_img()], [_img()], dict(zero_mask=0x10), 1, E_INVALIDARG, False),
    ("one_mask_bit", [_img()], [_img()], dict(one_mask=0x80), 1, E_INVALIDARG, False),
    ("null_src_pixels", [_img(ptr=False)], [_img()], GOOD, 1, E_POINTER, True),
    ("null_dst_pixels", [_img()], [_img(ptr=False)], GOOD, 1, E_POINTER, False),
    ("null_pixels_second", [_img(), _img(ptr=False)], [_img(), _img()], GOOD, 2, E_POINTER, True),
    ("fail_after_null_pixels", [_img(ptr=False), _img(87)], [_img(), _img(87)], GOOD, 2, E_POINTER, True),
]


def _args(src, dst, kw, n):
    s = capi.images(src) if src is not None else None
    d = capi.images(dst if dst is not None else src) if (dst is not None or src is not None) else None
    st = CS.steps(**kw) if kw is not None else None
    return s, n, st, d


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_apply_hresults(case, ref, em):
    name, src, dst, kw, n, want, through_ref = case
    s, n, st, d = _args(src, dst, kw, n)
    pst = C.byref(st) if st is not None else None
    assert F.hr_u32(L.dxb200_apply_channel_steps(s, n, pst, d)) == want, name
    assert F.hr_u32(L.dxb200_apply_channel_steps_device(s, n, pst, d, None)) == want, name
    assert F.hr_u32(em.emul_apply_channel_steps(s, n, pst, d)) == want, name
    if through_ref:
        assert ref.call(C.cast(s, CS.IP) if s is not None else None, n, st if st is not None else CS.steps()) == want, name


# ---- reconstruct Z's UNORM rule ------------------------------------------------------------------------------------------------
def test_unorm_rule_is_the_references_format_data_type(ref, em):
    for fmt in CS.FORMATS:
        assert em.emul_channel_unorm(fmt) == ref.is_unorm(fmt), fmt


# ---- the decompress format texconv picks ---------------------------------------------------------------------------------------
def _texconv_pick(bc, s):
    """Texconv/texconv.cpp:2393-2447 restated over ChannelSteps s (0: let Decompress pick)"""
    sw, z, o = list(s.swizzle), s.zeroMask, s.oneMask
    if bc in (80, 81):
        wide = s.invertY or s.reconstructZ or sw[1:] != [1, 2, 3] or any((z | o) >> c & 1 for c in (1, 2, 3))
    else:
        wide = s.reconstructZ or sw[2:] != [2, 3] or any((z | o) >> c & 1 for c in (2, 3))
    return (31 if bc in (81, 84) else 28) if wide else 0


STEP_SETS = [dict()] + [dict(swizzle=sw) for sw in ((1, 1, 2, 3), (0, 0, 2, 3), (0, 1, 0, 3), (0, 1, 2, 0), (3, 2, 1, 0))] \
    + [dict(zero_mask=1 << c) for c in range(4)] + [dict(one_mask=1 << c) for c in range(4)] \
    + [dict(invert_y=True), dict(reconstruct_z=True), dict(color_key=0x123456), dict(invert_y=True, color_key=1),
       dict(swizzle=(1, 0, 2, 3), invert_y=True)]


@pytest.mark.parametrize("bc", [80, 81, 83, 84])
def test_decompress_format_rule(bc, em):
    for kw in STEP_SETS:
        s = CS.steps(**kw)
        pick = _texconv_pick(bc, s)
        got = em.emul_channel_decompress_format(bc, C.byref(s))
        default = em.emul_channel_decompress_format(bc, None)
        assert got == (pick or default), (bc, kw, got)
        # through the pipeline planner: a 16 x 16 base into BC7 chains
        base = capi.images([capi.make_image(BUF.ctypes.data, 16, 16, bc)])
        dst = _chain(16, 16, 98)
        out = (C.c_uint64 * 8)()
        hr = em.emul_plan_mipmaps_compress_from_channels(base, 1, C.byref(capi.chain_source()), C.byref(s), 2, 0, None, 98, 0, 0.5, 1.0,
                                                         dst, out)
        assert hr == 0, (bc, kw, hex(F.hr_u32(hr)))
        assert out[0] == 1 and out[3] == (pick or default) and out[4] == (pick or default), (bc, kw, list(out))
        assert out[2] == (1 if kw else 0), (bc, kw)
    # an explicit decompress format wins over the rule
    s = CS.steps(reconstruct_z=True)
    base = capi.images([capi.make_image(BUF.ctypes.data, 16, 16, bc)])
    dst = _chain(16, 16, 98)
    out = (C.c_uint64 * 8)()
    assert em.emul_plan_mipmaps_compress_from_channels(base, 1, C.byref(capi.chain_source(2)), C.byref(s), 2, 0, None, 98, 0, 0.5, 1.0,
                                                       dst, out) == 0
    assert out[3] == 2


# ---- dxb200_mipmaps_compress_from_channels: the HRESULT of the first separate call that fails ---------------------------------
PIPE = [
    # (name, base fmt, w, h, source kwargs (None: NULL), channels kwargs (None: NULL), dst fmt, HRESULT of the first separate call
# that fails: dxb200_decompress, dxb200_resize, dxb200_apply_channel_steps on level 0, dxb200_mipmaps_compress_from_ex)
    ("bc_base_no_source", 83, 16, 16, None, dict(invert_y=True), 98, E_NOT_SUPPORTED),
    ("decompress_to_bc", 83, 16, 16, dict(decompress_format=71), dict(invert_y=True), 98, E_INVALIDARG),
    ("decompress_unimplemented", 83, 16, 16, dict(decompress_format=3), dict(invert_y=True), 98, E_NOT_SUPPORTED),
    ("resize_box_odd", 28, 16, 16, dict(width=5, height=5, resize_filter=0x400000), dict(invert_y=True), 98, E_FAIL),
    ("channels_bad_swizzle", 28, 16, 16, dict(), dict(swizzle=(0, 1, 2, 7)), 98, E_INVALIDARG),
    ("channels_bad_mask", 83, 16, 16, dict(), dict(zero_mask=0x20), 98, E_INVALIDARG),
    ("channels_before_compress", 28, 16, 16, None, dict(swizzle=(9, 1, 2, 3)), 28, E_INVALIDARG),
    ("compress_target_not_bc", 28, 16, 16, None, dict(invert_y=True), 28, E_INVALIDARG),
    ("compress_after_bc5_decompress", 83, 16, 16, dict(), dict(reconstruct_z=True), 61, E_INVALIDARG),
]


@pytest.mark.parametrize("case", PIPE, ids=[c[0] for c in PIPE])
def test_pipeline_hresults(case, em):
    name, bf, w, h, src_kw, ch_kw, df, want = case
    source = capi.chain_source(**src_kw) if src_kw is not None else None
    channels = CS.steps(**ch_kw) if ch_kw is not None else None
    lw, lh = (source.width or w, source.height or h) if source is not None else (w, h)
    base = capi.images([capi.make_image(BUF.ctypes.data, w, h, bf)])
    dst = _chain(lw, lh, df)
    args = (base, 1, C.byref(source) if source is not None else None, C.byref(channels) if channels is not None else None, 2, 0, None, df, 0,
            0.5, 1.0, dst)
    assert F.hr_u32(L.dxb200_mipmaps_compress_from_channels(*args, None)) == want, name
    out = (C.c_uint64 * 8)()
    assert F.hr_u32(em.emul_plan_mipmaps_compress_from_channels(*args, out)) == want, name


def test_pipeline_without_steps_is_from_ex(em):
    """channels NULL or with no step enabled: the HRESULT and the plan of dxb200_mipmaps_compress_from_ex"""
    for bf, src_kw, df in ((83, dict(), 98), (83, None, 98), (28, dict(width=5, height=5, resize_filter=0x400000), 98), (28, None, 28),
                           (71, dict(decompress_format=71), 98), (28, dict(), 98)):
        source = capi.chain_source(**src_kw) if src_kw is not None else None
        lw, lh = (source.width or 16, source.height or 16) if source is not None else (16, 16)
        base = capi.images([capi.make_image(BUF.ctypes.data, 16, 16, bf)])
        dst = _chain(lw, lh, df)
        ps = C.byref(source) if source is not None else None
        want = F.hr_u32(L.dxb200_mipmaps_compress_from_ex(base, 1, ps, 2, 0, None, df, 0, 0.5, 1.0, dst, None))
        for ch in (None, CS.steps(), CS.steps(color_key=None, swizzle=(0, 1, 2, 3))):
            pc = C.byref(ch) if ch is not None else None
            got = F.hr_u32(L.dxb200_mipmaps_compress_from_channels(base, 1, ps, pc, 2, 0, None, df, 0, 0.5, 1.0, dst, None))
            assert got == want, (bf, src_kw, df)
            out = (C.c_uint64 * 8)()
            hr = F.hr_u32(em.emul_plan_mipmaps_compress_from_channels(base, 1, ps, pc, 2, 0, None, df, 0, 0.5, 1.0, dst, out))
            if hr == 0:
                assert out[2] == 0


def test_pipeline_channel_steps_run_on_level_0(em):
    """a valid plan runs the steps on level 0's format and size: after the BC5 decompress (R8G8B8A8 for reconstruct Z) and the resize"""
    s = CS.steps(invert_y=True, reconstruct_z=True)
    base = capi.images([capi.make_image(BUF.ctypes.data, 16, 16, 83)])
    dst = _chain(8, 8, 98)
    out = (C.c_uint64 * 8)()
    assert em.emul_plan_mipmaps_compress_from_channels(base, 1, C.byref(capi.chain_source(0, 8, 8)), C.byref(s), 2, 0, None, 98, 0, 0.5, 1.0,
                                                       dst, out) == 0
    assert list(out[:7]) == [1, 1, 1, 28, 28, 8, 8]


# ---- the emulator against the reference -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("config", sorted(CS.CONFIGS))
@pytest.mark.parametrize("fmt", CS.FORMATS)
def test_emulator_equals_reference(fmt, config, ref, em):
    s = CS.steps(**CS.CONFIGS[config])
    img = CS.corpus(fmt)
    want = ref.apply(fmt, CS.W, CS.H, [img], s)[0]
    got = CS.emul_apply(em, fmt, CS.W, CS.H, [img], s)[0]
    SV.assert_same(got, want, fmt, "%d %s" % (fmt, config))


def test_emulator_equals_reference_on_arrays_in_place(ref, em):
    """an array of three images, steps written over their sources"""
    fmt, s = 28, CS.steps(**CS.CONFIGS["all"])
    imgs = [CS.corpus(fmt, 64, 32, seed=k) for k in range(3)]
    want = ref.apply(fmt, 64, 32, imgs, s)
    src = capi.images([capi.make_image(a.ctypes.data, 64, 32, fmt) for a in imgs])
    assert em.emul_apply_channel_steps(src, 3, C.byref(s), src) == 0
    for a, b in zip(imgs, want):
        SV.assert_same(a, b, fmt, "in place")
