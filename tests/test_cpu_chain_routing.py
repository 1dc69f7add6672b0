"""CPU suite: what one chunk of the one-call pipelines (dxb200_mipmaps_compress_from_channels_ex, dxb200_mipmaps_convert_from_ex,
dxb200_levels_from_ex) stages and runs, without a device.  For one valid call of each routing case the planner's chunk plan
(tests/emul/texconv_steps.cpp, emul_chunk_plan) must list the planes a chunk's buffer holds, in order, with how each image travels,
and every step with the plane it reads, the plane it writes and the images it covers.

Planes are "role per-item-images copy-of-image-0 copy-of-the-rest" (U = up, D = down, N = device only); steps are
"kind source>destination cover" with cover front (the items' level 0, or every kept level), all (every image) or level (one
launch per level of a generated chain)."""
import ctypes as C
import os

import pytest

from directxtex_b200 import capi, formats as F
from tests.bc7_ranking_build import host_lib
from tests.test_cpu_texconv_steps import DM, ENTRIES, NM, PM, call_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROLES = ["base", "dec", "l0", "chain", "dst", "words"]
COPIES = "UDN"
KINDS = ["decompress", "demultiply", "resize", "copy", "channels", "convert", "post", "mips", "coverage", "premultiply", "layout",
         "compress", "scan"]
COVERS = ["front", "all", "level"]
FILTER = F.TEX_FILTER_LINEAR


@pytest.fixture(scope="module")
def em(tmp_path_factory):
    E = host_lib("texconv_steps.cpp", tmp_path_factory.mktemp("chain_routing_emul"), os.path.join(ROOT, "tests", "emul"))
    for _, name, args in ENTRIES.values():
        getattr(E, name).argtypes = args + [C.POINTER(C.c_uint64)]
        getattr(E, name).restype = C.c_int32
    E.emul_chunk_plan.argtypes = [C.POINTER(C.c_uint64), C.c_size_t]
    E.emul_chunk_plan.restype = C.c_size_t
    return E


# (name, entry, base fmt, w, h, items, levels, dst fmt, source kwargs, channels kwargs, steps, texconv kwargs, scan,
#  planes, steps, item 0's weight = the bytes of its level 0 in the chain)
CASES = [
    # a generated chain compressed from an uploaded level 0: no front step, nothing of the base is staged
    ("rgba8_to_bc3_scan", "gen", 28, 32, 32, 1, 6, 77, None, None, None, {}, True,
     "chain 6 UN, dst 6 DD, words 1 DD",
     "mips chain>chain all, compress chain>dst all, scan dst>words all", 4096),
    # demultiply without Decompress runs on the uploaded level 0
    ("rgba8_demultiply_to_bc7", "gen", 28, 32, 32, 1, 6, 98, None, None, None, DM, False,
     "chain 6 UN, dst 6 DD",
     "demultiply chain>chain front, mips chain>chain all, compress chain>dst all", 4096),
    # Decompress writes level 0 of the chain; demultiply in place there; coverage, premultiply one launch per level
    ("bc3_demultiply_coverage_premultiply_to_bc7", "gen", 77, 32, 32, 2, 6, 98, {}, None, capi.chain_steps(0.5, True), DM, False,
     "base 1 UU, chain 6 NN, dst 6 DD",
     "decompress base>chain front, demultiply chain>chain front, mips chain>chain all, coverage chain>chain all, "
     "premultiply chain>chain level, compress chain>dst all", 4096),
    # Decompress then Resize: the decompressed image has a plane of its own
    ("bc5_resize_invert_y_to_bc3n_scan", "gen", 83, 40, 40, 1, 6, 77, dict(width=32, height=32), dict(invert_y=True), None, NM, True,
     "base 1 UU, dec 1 NN, chain 6 NN, dst 6 DD, words 1 DD",
     "decompress base>dec front, resize dec>chain front, channels chain>chain front, mips chain>chain all, layout chain>chain all, "
     "compress chain>dst all, scan dst>words all", 4096),
    ("rgba16f_resize_swizzle_to_bc7", "gen", 10, 64, 64, 2, 6, 98, dict(width=32, height=32), dict(swizzle=(2, 1, 0, 3)), None, {}, False,
     "base 1 UU, chain 6 NN, dst 6 DD",
     "resize base>chain front, channels chain>chain front, mips chain>chain all, compress chain>dst all", 8192),
    # an uncompressed output: the chain is dst; a front step and a Convert leave level 0 in a plane of its own
    ("bc7_demultiply_convert_color_key_premultiply_scan", "conv", 98, 32, 32, 1, 6, 87, {}, dict(color_key=0x102030), PM, DM, True,
     "base 1 UU, l0 1 NN, dst 6 DD, words 1 DD",
     "decompress base>l0 front, demultiply l0>l0 front, convert l0>dst front, post dst>dst front, mips dst>dst all, "
     "premultiply dst>dst level, scan dst>words all", 4096),
    ("bc1_resize_convert_scan", "conv", 71, 64, 64, 1, 6, 10, dict(width=32, height=32), None, None, {}, True,
     "base 1 UU, dec 1 NN, l0 1 NN, dst 6 DD, words 1 DD",
     "decompress base>dec front, resize dec>l0 front, convert l0>dst front, mips dst>dst all, scan dst>words all", 8192),
    # a Convert without a front step reads the base; the swizzle runs in place on it
    ("rgba16f_swizzle_convert", "conv", 10, 32, 32, 2, 5, 28, None, dict(swizzle=(2, 1, 0, 3)), None, {}, False,
     "base 1 UU, dst 5 DD",
     "channels base>base front, convert base>dst front, mips dst>dst all", 4096),
    # no step writes level 0: the base is copied into it, demultiply runs on the base before
    ("rgba8_demultiply_copy_color_key_premultiply", "conv", 28, 32, 32, 1, 6, 28, None, dict(color_key=0x102030), PM, DM, False,
     "base 1 UU, dst 6 DD",
     "demultiply base>base front, copy base>dst front, channels dst>dst front, mips dst>dst all, premultiply dst>dst level", 4096),
    # kept levels: every level of the base goes up where the generated chains hold level 0
    ("bc3_pass_through", "lev", 77, 32, 32, 1, 6, 77, None, None, None, {}, False,
     "base 6 UU, dst 6 DD",
     "copy base>dst front", 1024),
    ("rgba8_premultiply_to_bc7_scan", "lev", 28, 32, 32, 2, 6, 98, None, None, PM, {}, True,
     "chain 6 UU, dst 6 DD, words 1 DD",
     "premultiply chain>chain front, compress chain>dst all, scan dst>words all", 4096),
    ("bc3_to_bc7", "lev", 77, 32, 32, 1, 6, 98, None, None, None, {}, False,
     "base 6 UU, chain 6 NN, dst 6 DD",
     "decompress base>chain front, compress chain>dst all", 4096),
    ("bc3_swizzle_convert_color_key", "lev", 77, 32, 32, 1, 6, 87, None, dict(swizzle=(2, 1, 0, 3), color_key=0x102030), None, {}, False,
     "base 6 UU, l0 6 NN, dst 6 DD",
     "decompress base>l0 front, channels l0>l0 front, convert l0>dst front, post dst>dst front", 4096),
    ("rgba8_demultiply_convert", "lev", 28, 16, 16, 1, 5, 10, None, None, None, DM, False,
     "base 5 UU, dst 5 DD",
     "demultiply base>base front, convert base>dst front", 2048),
    ("rgba8_resize_to_bc1", "lev", 28, 40, 40, 1, 1, 71, dict(width=20, height=20), None, None, {}, False,
     "base 1 UU, chain 1 NN, dst 1 DD",
     "resize base>chain front, compress chain>dst all", 1600),
]


def _chunk_plan(em):
    out = (C.c_uint64 * 256)()
    n = em.emul_chunk_plan(out, len(out))
    w = list(out[:n])
    nplanes, nsteps, per, filt, weight = w[:5]
    planes = [w[5 + 4 * i: 9 + 4 * i] for i in range(nplanes)]
    steps = [w[5 + 4 * nplanes + 4 * i: 9 + 4 * nplanes + 4 * i] for i in range(nsteps)]
    assert n == 5 + 4 * (nplanes + nsteps)
    return (", ".join("%s %d %s%s" % (ROLES[r], p, COPIES[a], COPIES[b]) for r, p, a, b in planes),
            ", ".join("%s %s>%s %s" % (KINDS[k], ROLES[s], ROLES[d], COVERS[c]) for k, s, d, c in steps), per, filt, weight)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_chunk_routing(case, em):
    name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, scan, want_planes, want_steps, want_weight = case
    args, _keep = call_args(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps)
    args = list(args)
    if entry != "lev":
        args[5 if entry == "gen" else 8] = FILTER             # GenerateMipMaps' filter
    ts = capi.texconv_steps(**ts_kw)
    opaque = C.c_int32(-1)
    hr = getattr(em, ENTRIES[entry][1])(*args, C.byref(opaque) if scan else None, C.byref(ts), None)
    assert hr == 0, (name, hex(F.hr_u32(hr)))
    planes, steps_, per, filt, weight = _chunk_plan(em)
    assert planes == want_planes, (name, planes)
    assert steps_ == want_steps, (name, steps_)
    assert per == (levels if entry == "lev" else 1), name
    assert filt == (0 if entry == "lev" else FILTER), name
    assert weight == want_weight, name
