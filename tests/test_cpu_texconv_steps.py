"""CPU suite: the argument checks and plans of texconv's -alpha (demultiply) and BC3n / RXGB layout steps in
dxb200_mipmaps_compress_from_channels_ex, dxb200_mipmaps_convert_from_ex and dxb200_levels_from_ex, without a device.  A failing
call returns E_INVALIDARG for the steps' own rules (a layout other than 0-2, a layout into anything but BC3_UNORM or on the call
without a BC target), then the HRESULT of the call without _ex's own rules, then that of the first separate call that would fail
(Decompress, PremultiplyAlpha REVERSE, Resize, ..., premultiply, the layout's TransformImage, Compress), through the library and
through the planners on the host (tests/emul/texconv_steps.cpp).  A valid call's plan says which launches a chunk runs, the
decompress format a layout picks for BC4 / BC5 and that a layout or demultiply turns levels_from's pass-through off.  NULL and
all-zero steps plan exactly as the calls without _ex."""
import ctypes as C
import os

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests.bc7_ranking_build import host_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = capi.lib
IP = C.POINTER(capi.Image)
TP = C.POINTER(capi.TexconvSteps)
E_INVALIDARG, E_POINTER, E_FAIL, E_NOT_SUPPORTED = 0x80070057, 0x80004003, 0x80004005, 0x80070032
BUF = np.zeros(1 << 22, np.uint8)
NOUT = 17
SW, UNORM = 1 << 16, 1 << 20
DXT5NM = SW | (1 << 2) | (2 << 4) | (0x4 << 8) | (0x1 << 12)        # swizzle (0, 1, 2, 0), zero B, one R
RXGB = SW | 3 | (1 << 2) | (2 << 4)                                  # swizzle (3, 1, 2, 0)
REVERSE = 1                         # the premultiply launch's reverse bit (TEX_PMALPHA_REVERSE = 0x2 in the call)
GEN_ARGS = [IP, C.c_size_t, C.POINTER(capi.ChainSource), C.POINTER(capi.ChannelSteps), C.c_size_t, C.c_uint32, C.POINTER(capi.ChainSteps),
            C.c_uint32, C.c_uint32, C.c_float, C.c_float, IP, C.POINTER(C.c_int32), TP]
CONV_ARGS = [IP, C.c_size_t, C.POINTER(capi.ChainSource), C.POINTER(capi.ChannelSteps), C.c_uint32, C.c_uint32, C.c_float, C.c_size_t,
             C.c_uint32, C.POINTER(capi.ChainSteps), IP, C.POINTER(C.c_int32), TP]
LEV_ARGS = [IP, C.c_size_t, C.c_size_t, C.POINTER(capi.ChainSource), C.POINTER(capi.ChannelSteps), C.c_uint32, C.c_uint32, C.c_uint32,
            C.c_float, C.POINTER(capi.ChainSteps), IP, C.POINTER(C.c_int32), TP]
ENTRIES = {"gen": ("dxb200_mipmaps_compress_from_channels_ex", "emul_plan_compress_from_channels_ex", GEN_ARGS),
           "conv": ("dxb200_mipmaps_convert_from_ex", "emul_plan_convert_from_ex", CONV_ARGS),
           "lev": ("dxb200_levels_from_ex", "emul_plan_levels_from_ex", LEV_ARGS)}


@pytest.fixture(scope="module")
def em(tmp_path_factory):
    E = host_lib("texconv_steps.cpp", tmp_path_factory.mktemp("texconv_steps_emul"), os.path.join(ROOT, "tests", "emul"))
    for _, name, args in ENTRIES.values():
        getattr(E, name).argtypes = args + [C.POINTER(C.c_uint64)]
        getattr(E, name).restype = C.c_int32
    return E


def _img(w, h, fmt, ptr=True):
    p = BUF.ctypes.data if ptr else None
    if fmt in F.BYTES_PER_PIXEL or fmt in F.BLOCK_BYTES:
        return capi.make_image(p, w, h, fmt)
    return capi.Image(w, h, fmt, 0, 0, p)


def _sizes(w, h, levels):
    out = []
    for _ in range(levels):
        out.append((w, h))
        w, h = max(1, w // 2), max(1, h // 2)
    return out


def _change(ims, bad):
    if bad is not None:
        i, field, value = bad
        setattr(ims[i], field, value)
    return ims


def call_args(entry, bf, w, h, items, levels, df, src_kw=None, ch_kw=None, steps=None, ts=None, base_bad=None, dst_bad=None):
    """the arguments of `entry` (without alphaAllOpaque and ts' pointer) for items of a w x h base of bf: one level 0 per item
    ("gen", "conv") or `levels` kept levels per item ("lev"); dst = the chains of df at the output size"""
    source = capi.chain_source(**src_kw) if src_kw is not None else None
    channels = capi.channel_steps(**ch_kw) if ch_kw is not None else None
    ow, oh = (source.width, source.height) if source is not None and source.width else (w, h)
    bsizes = _sizes(w, h, levels) if entry == "lev" else [(w, h)]
    base = capi.images(_change([_img(bw, bh, bf) for _ in range(items) for (bw, bh) in bsizes], base_bad))
    dst = capi.images(_change([_img(lw, lh, df) for _ in range(items) for (lw, lh) in _sizes(ow, oh, levels)], dst_bad))
    src_p = C.byref(source) if source is not None else None
    ch_p = C.byref(channels) if channels is not None else None
    st_p = C.byref(steps) if steps is not None else None
    if entry == "gen":
        return (base, items, src_p, ch_p, levels, 0, st_p, df, 0, 0.5, 1.0, dst), (source, channels, steps)
    if entry == "conv":
        return (base, items, src_p, ch_p, df, 0, 0.5, levels, 0, st_p, dst), (source, channels, steps)
    return (base, items, levels, src_p, ch_p, df, 0, 0, 0.5, st_p, dst), (source, channels, steps)


PM = capi.chain_steps(0.0, True)
DM = dict(demultiply=True)
NM, RX = dict(bc3_layout=1), dict(bc3_layout=2)
# (name, entry, base fmt, w, h, items, levels, dst fmt, source kwargs, channels kwargs, steps, texconv kwargs, base change,
#  dst change, HRESULT); a change is (image index, field, value), image index = item * levels + l of the base ("lev") or dst
CASES = [
    # the steps' own rules, before any other check
    ("layout_3", "gen", 28, 16, 16, 1, 5, 77, None, None, None, dict(bc3_layout=3), None, None, E_INVALIDARG),
    ("layout_3_levels_from", "lev", 77, 16, 16, 1, 5, 77, None, None, None, dict(bc3_layout=3), None, None, E_INVALIDARG),
    ("layout_bc3_srgb", "gen", 28, 16, 16, 1, 5, 78, None, None, None, NM, None, None, E_INVALIDARG),
    ("layout_bc7", "gen", 28, 16, 16, 1, 5, 98, None, None, None, RX, None, None, E_INVALIDARG),
    ("layout_bc7_levels_from", "lev", 77, 16, 16, 1, 5, 98, None, None, None, NM, None, None, E_INVALIDARG),
    ("layout_bc3_srgb_before_null_base_pixels", "lev", 28, 16, 16, 1, 5, 78, None, None, None, RX, (2, "pixels", None), None, E_INVALIDARG),
    ("layout_bc7_before_demultiply_r8g8", "gen", 49, 16, 16, 1, 5, 98, None, None, None, dict(demultiply=True, bc3_layout=1), None, None,
     E_INVALIDARG),
    ("layout_convert_from", "conv", 28, 16, 16, 1, 5, 28, None, None, None, NM, None, None, E_INVALIDARG),
    ("layout_convert_from_bc3_target", "conv", 28, 16, 16, 1, 5, 77, None, None, None, RX, None, None, E_INVALIDARG),
    ("layout_convert_from_before_null_base_pixels", "conv", 28, 16, 16, 2, 5, 10, None, None, None, NM, (1, "pixels", None), None,
     E_INVALIDARG),
    # the call's own rules, before the steps' checks
    ("levels_0_with_demultiply_r8g8", "lev", 49, 16, 16, 1, 0, 77, None, None, None, DM, None, None, E_INVALIDARG),
    ("coverage_with_demultiply_r8g8", "lev", 49, 16, 16, 1, 5, 77, None, None, capi.chain_steps(0.5), DM, None, None, E_INVALIDARG),
    # Decompress, then demultiply
    ("decompress_to_bc_before_demultiply", "gen", 77, 16, 16, 1, 5, 77, dict(decompress_format=71), None, None, DM, None, None, E_INVALIDARG),
    ("decompress_pixels_before_demultiply", "lev", 77, 16, 16, 1, 5, 98, None, None, None, DM, (3, "pixels", None), None, E_POINTER),
    ("demultiply_r8g8", "gen", 49, 16, 16, 1, 5, 77, None, None, None, DM, None, None, E_NOT_SUPPORTED),
    ("demultiply_r8g8_convert_from", "conv", 49, 16, 16, 1, 5, 28, None, None, None, DM, None, None, E_NOT_SUPPORTED),
    ("demultiply_r8g8_levels_from", "lev", 49, 16, 16, 1, 5, 49, None, None, None, DM, None, None, E_NOT_SUPPORTED),
    ("demultiply_bc4_default_decompress", "gen", 80, 16, 16, 1, 5, 98, dict(), None, None, DM, None, None, E_NOT_SUPPORTED),
    ("demultiply_bc4_default_decompress_levels_from", "lev", 80, 16, 16, 1, 5, 80, None, None, None, DM, None, None, E_NOT_SUPPORTED),
    ("demultiply_bc5_default_decompress", "conv", 83, 16, 16, 1, 5, 28, dict(), None, None, DM, None, None, E_NOT_SUPPORTED),
    ("demultiply_bc_base_without_source", "conv", 77, 16, 16, 1, 5, 28, None, None, None, DM, None, None, E_NOT_SUPPORTED),
    ("demultiply_before_box_resize", "gen", 49, 20, 20, 1, 3, 77, dict(width=7, height=7, resize_filter=F.TEX_FILTER_BOX), None, None, DM,
     None, None, E_NOT_SUPPORTED),
    ("demultiply_base_item1_pixels", "gen", 28, 16, 16, 2, 5, 77, None, None, None, DM, (1, "pixels", None), None, E_POINTER),
    ("demultiply_base_level2_format", "lev", 28, 16, 16, 1, 5, 98, None, None, None, DM, (2, "format", 87), None, E_INVALIDARG),
    # Resize after demultiply
    ("box_resize_after_demultiply", "gen", 28, 20, 20, 1, 3, 77, dict(width=7, height=7, resize_filter=F.TEX_FILTER_BOX), None, None, DM,
     None, None, E_FAIL),
    ("box_resize_with_layout", "gen", 83, 20, 20, 1, 3, 77, dict(width=7, height=7, resize_filter=F.TEX_FILTER_BOX), None, None, NM,
     None, None, E_FAIL),
    # premultiply before the layout, the layout's TransformImage, Compress after it
    ("premultiply_r8g8_before_layout", "gen", 49, 16, 16, 1, 5, 77, None, None, PM, NM, None, None, E_NOT_SUPPORTED),
    ("layout_base_level3_format", "lev", 28, 16, 16, 1, 5, 77, None, None, None, RX, (3, "format", 87), None, E_FAIL),
    ("layout_base_level2_pixels", "lev", 28, 16, 16, 1, 5, 77, None, None, None, NM, (2, "pixels", None), None, E_POINTER),
    ("compress_dst_level2_size_with_layout", "gen", 28, 16, 16, 1, 5, 77, None, None, None, NM, None, (2, "width", 8), E_FAIL),
    ("compress_dst_level1_pixels_with_layout", "lev", 83, 16, 16, 2, 5, 77, None, None, None, RX, None, (6, "pixels", None), E_POINTER),
    ("compress_dst_format_with_layout_and_demultiply", "lev", 77, 16, 16, 1, 5, 77, None, None, None, dict(demultiply=True, bc3_layout=1),
     None, (3, "format", 78), E_INVALIDARG),
]


def _run(entry, em, case_args, ts, opaque, out=None):
    lib_name, em_name, _ = ENTRIES[entry]
    got_lib = F.hr_u32(getattr(L, lib_name)(*case_args, opaque, ts))
    got_em = F.hr_u32(getattr(em, em_name)(*case_args, opaque, ts, out))
    return got_lib, got_em


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_hresults(case, em):
    name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, base_bad, dst_bad, want = case
    args, _keep = call_args(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, None, base_bad, dst_bad)
    ts = capi.texconv_steps(**ts_kw)
    opaque = C.c_int32(-1)
    for op in (C.byref(opaque), None):
        got_lib, got_em = _run(entry, em, args, C.byref(ts), op)
        assert (hex(got_lib), hex(got_em)) == (hex(want), hex(want)), name
    assert opaque.value == -1


def test_every_case_fixed_plans(em):
    """each case that changes an image plans once that change is undone, and each case that fails on a step fails without it: the
    table tests the check it names and no other"""
    for case in CASES:
        name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, base_bad, dst_bad, want = case
        if base_bad is None and dst_bad is None or ts_kw.get("bc3_layout", 0) > 2 or entry == "conv" and ts_kw.get("bc3_layout") \
                or ts_kw.get("bc3_layout") and df != 77 or levels == 0:
            continue
        args, _keep = call_args(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps)
        ts = capi.texconv_steps(**ts_kw)
        assert _run(entry, em, args, C.byref(ts), None)[1] == 0, name


# (name, entry, base fmt, w, h, items, levels, dst fmt, source kwargs, channels kwargs, steps, texconv kwargs,
#  { decompress, demultiply, resize, channels, convert, post, premultiply, layout, compress, decompress format, working format,
#    demultiply flags, layout word, pass-through })
PLANS = [
    ("bc5_to_bc3n", "gen", 83, 64, 64, 2, 7, 77, dict(), None, None, NM, [1, 0, 0, 0, 0, 0, 0, 1, 1, 28, 28, 0, DXT5NM | UNORM, 0]),
    ("bc5_snorm_to_rxgb", "gen", 84, 64, 64, 1, 7, 77, dict(), None, None, RX, [1, 0, 0, 0, 0, 0, 0, 1, 1, 31, 31, 0, RXGB, 0]),
    ("bc4_to_bc3n", "gen", 80, 32, 32, 1, 6, 77, dict(), None, None, NM, [1, 0, 0, 0, 0, 0, 0, 1, 1, 28, 28, 0, DXT5NM | UNORM, 0]),
    ("bc4_snorm_to_rxgb_levels", "lev", 81, 32, 32, 1, 6, 77, None, None, None, RX, [1, 0, 0, 0, 0, 0, 0, 1, 1, 31, 31, 0, RXGB, 0]),
    ("bc5_explicit_decompress_format_kept", "gen", 83, 32, 32, 1, 6, 77, dict(decompress_format=2), None, None, NM,
     [1, 0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 0, DXT5NM, 0]),
    ("bc5_invert_y_reconstruct_z_to_bc3n", "lev", 83, 32, 32, 2, 6, 77, None, dict(invert_y=True, reconstruct_z=True), None, NM,
     [1, 0, 0, 1, 0, 0, 0, 1, 1, 28, 28, 0, DXT5NM | UNORM, 0]),
    ("bc4_layout_makes_demultiply_possible", "lev", 80, 32, 32, 1, 6, 77, None, None, None, dict(demultiply=True, bc3_layout=2),
     [1, 1, 0, 0, 0, 0, 0, 1, 1, 28, 28, REVERSE, RXGB | UNORM, 0]),
    ("rgba16f_to_bc3n_premultiply", "gen", 10, 32, 32, 1, 6, 77, None, None, PM, NM, [0, 0, 0, 0, 0, 0, 1, 1, 1, 0, 10, 0, DXT5NM, 0]),
    ("r10g10b10a2_to_bc3n_coverage", "gen", 24, 32, 32, 1, 6, 77, None, None, capi.chain_steps(0.5, True), NM,
     [0, 0, 0, 0, 0, 0, 1, 1, 1, 0, 24, 0, DXT5NM | UNORM, 0]),
    ("bc3_demultiply_to_bc7", "gen", 77, 32, 32, 3, 6, 98, dict(), None, PM, DM, [1, 1, 0, 0, 0, 0, 1, 0, 1, 28, 28, REVERSE, 0, 0]),
    ("bc3_demultiply_srgb_flags", "gen", 77, 32, 32, 1, 6, 98, dict(), None, PM, dict(demultiply=True, demultiply_flags=F.TEX_FILTER_SRGB),
     [1, 1, 0, 0, 0, 0, 1, 0, 1, 28, 28, REVERSE | F.TEX_FILTER_SRGB, 0, 0]),
    ("rgba8_srgb_demultiply_resize", "gen", 29, 40, 40, 1, 5, 98, dict(width=16, height=16), None, PM, DM,
     [0, 1, 1, 0, 0, 0, 1, 0, 1, 0, 29, REVERSE | F.TEX_FILTER_SRGB, 0, 0]),
    ("rgba8_demultiply_no_front", "gen", 28, 32, 32, 1, 6, 98, None, None, None, DM, [0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 28, REVERSE, 0, 0]),
    ("a8_demultiply", "gen", 65, 32, 32, 1, 6, 77, None, None, None, DM, [0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 65, REVERSE, 0, 0]),
    ("bc7_demultiply_to_bgra8", "conv", 98, 32, 32, 1, 6, 87, dict(), None, PM, DM, [1, 1, 0, 0, 1, 0, 1, 0, 0, 28, 28, REVERSE, 0, 0]),
    ("rgba16f_demultiply_resize_to_rgba8", "conv", 10, 40, 24, 2, 4, 28, dict(width=20, height=12), None, PM, DM,
     [0, 1, 1, 0, 1, 0, 1, 0, 0, 0, 10, REVERSE, 0, 0]),
    ("rgba8_demultiply_unconverted", "conv", 28, 32, 32, 1, 6, 28, None, None, PM, DM, [0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 28, REVERSE, 0, 0]),
    ("bc3_demultiply_stops_pass_through", "lev", 77, 32, 32, 1, 6, 77, None, None, None, DM, [1, 1, 0, 0, 0, 0, 0, 0, 1, 28, 28, REVERSE, 0, 0]),
    ("bc3_layout_stops_pass_through", "lev", 77, 32, 32, 1, 6, 77, None, None, None, RX, [1, 0, 0, 0, 0, 0, 0, 1, 1, 28, 28, 0, RXGB | UNORM, 0]),
    ("bc3_pass_through_without_steps", "lev", 77, 32, 32, 1, 6, 77, None, None, None, dict(), [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 77, 0, 0, 1]),
    ("rgba8_demultiply_copied_levels", "lev", 28, 32, 32, 2, 6, 28, None, None, PM, DM, [0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 28, REVERSE, 0, 0]),
]


def _try_plan(entry, em, args, ts):
    out = (C.c_uint64 * NOUT)()
    return F.hr_u32(getattr(em, ENTRIES[entry][1])(*args, None, ts, out)), list(out)


def _plan(entry, em, args, ts):
    hr, out = _try_plan(entry, em, args, ts)
    assert hr == 0, hex(hr)
    return out


def launches_per_chunk(entry, plan, levels):
    """kernel launches of the steps in front of the mips and after them that one chunk runs, from a plan: one each for Decompress,
    the demultiply, Resize, the channel steps, Convert, the later channel steps, the layout and Compress; premultiply is one per
    level of a generated chain and one for kept levels"""
    dec, dm, rs, ch, cv, post, gen, cov, pm, lay, comp = plan[:11]
    return dec + dm + rs + ch + cv + post + lay + comp + pm * (levels if gen else 1)


@pytest.mark.parametrize("plan", PLANS, ids=[p[0] for p in PLANS])
def test_plans(plan, em):
    name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, want = plan
    args, _keep = call_args(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps)
    ts = capi.texconv_steps(**ts_kw)
    out = _plan(entry, em, args, C.byref(ts))
    got = [out[0], out[1], out[2], out[3], out[4], out[5], out[8], out[9], out[10], out[11], out[12], out[13], out[14], out[15]]
    assert got == want, (name, got)
    assert out[6] == (entry != "lev"), name
    # exactly one more launch per chunk for each step than the same call without them, where that call decompresses to the same
    # format and does not pass the chain through
    hr, bare = _try_plan(entry, em, args, None)
    if hr == 0 and bare[11] == out[11] and not bare[15]:
        extra = (1 if ts_kw.get("demultiply") else 0) + (1 if ts_kw.get("bc3_layout") else 0)
        assert launches_per_chunk(entry, out, levels) == launches_per_chunk(entry, bare, levels) + extra, name


@pytest.mark.parametrize("bf,want", [(80, 28), (81, 31), (83, 28), (84, 31), (71, 28), (77, 28), (98, 28)])
@pytest.mark.parametrize("layout", [1, 2])
def test_decompress_format_with_layout(bf, want, layout, em):
    """with a layout and no decompress format a BC4 / BC5 base decompresses to R8G8B8A8 (SNORM for the SNORM twins), as texconv
    picks it; other BC bases keep DefaultDecompress, and without a layout BC4 / BC5 keep theirs"""
    for entry in ("gen", "lev"):
        args, _keep = call_args(entry, bf, 16, 16, 1, 5, 77, dict() if entry == "gen" else None)
        ts = capi.texconv_steps(bc3_layout=layout)
        assert _plan(entry, em, args, C.byref(ts))[11] == want, (entry, bf)
        default = _plan(entry, em, args, None)
        assert default[11] == (0 if default[15] else {80: 61, 81: 63, 83: 49, 84: 51}.get(bf, 28)), (entry, bf, default)


# (entry, base fmt, items, levels, dst fmt, source kwargs, channels kwargs, steps)
SAME = [
    ("gen", 28, 2, 5, 98, None, None, None),
    ("gen", 77, 1, 5, 71, dict(), dict(invert_y=True), PM),
    ("gen", 83, 1, 4, 83, dict(width=8, height=8), dict(reconstruct_z=True), None),
    ("gen", 28, 1, 5, 77, None, None, capi.chain_steps(0.5, True)),
    ("conv", 98, 2, 5, 87, dict(), dict(swizzle=(2, 1, 0, 3)), PM),
    ("conv", 28, 1, 5, 28, None, dict(color_key=0x102030), None),
    ("lev", 77, 2, 5, 77, None, None, None),
    ("lev", 77, 1, 5, 98, None, None, PM),
    ("lev", 28, 1, 5, 10, None, dict(invert_y=True), None),
]


@pytest.mark.parametrize("case", SAME, ids=["%s_%d_%d" % (c[0], c[1], c[4]) for c in SAME])
def test_null_and_zero_steps_plan_as_the_call_without_ex(case, em):
    entry, bf, items, levels, df, src_kw, ch_kw, steps = case
    args, _keep = call_args(entry, bf, 16, 16, items, levels, df, src_kw, ch_kw, steps)
    zero = capi.texconv_steps()
    a = _plan(entry, em, args, None)
    b = _plan(entry, em, args, C.byref(zero))
    assert a == b and a[1] == 0 and a[9] == 0


def test_zero_steps_answer_as_the_calls_without_ex(em):
    """every failing case of the calls without _ex answers the same through _ex with NULL and with all-zero steps"""
    from tests import test_cpu_levels_from as lf
    zero = capi.texconv_steps()
    for case in lf.CASES:
        name, bf, sizes, items, src_kw, ch_kw, df, cf, steps, base_bad, dst_bad, levels, want = case[:13]
        args = lf._args(bf, sizes, items, src_kw, ch_kw, df, cf, 0, steps, base_bad, dst_bad, levels)
        for ts in (None, C.byref(zero)):
            assert F.hr_u32(L.dxb200_levels_from_ex(*args, None, ts)) == want, name
    for case in CASES:
        name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, base_bad, dst_bad, want = case
        args, _keep = call_args(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, None, base_bad, dst_bad)
        if _try_plan(entry, em, args, None)[0] == 0:
            continue                    # a valid call would run on a device
        plain = {"gen": L.dxb200_mipmaps_compress_from_channels, "conv": L.dxb200_mipmaps_convert_from, "lev": L.dxb200_levels_from}[entry]
        base_hr = F.hr_u32(plain(*args, None))
        for ts in (None, C.byref(zero)):
            assert F.hr_u32(getattr(L, ENTRIES[entry][0])(*args, None, ts)) == base_hr, name
