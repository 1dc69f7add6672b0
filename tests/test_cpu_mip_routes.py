"""CPU suite for the mip / resize kernel routes (no GPU needed).

- The specialised mip kernel instantiations compiled into the library (family x UNORM twin of a hot format x filter mode x
  sRGB x LIN, read from its kernel entry points) are exactly those the cases of the GPU route table in
  tests/test_gpu_mip_routes.py reach, so a new instantiation cannot go untested and none is compiled that no call selects.
- k_mip_sep's fp32 tap coordinates, run as the kernel runs them, stay inside the image and inside its shared-memory tile
  buffers up to the extent limit the launcher gives it.
- The host emulator of the mip arithmetic (the inline code every mip kernel runs) against the oracle under TEX_FILTER_SRGB,
  SRGB_IN and SRGB_OUT, for every supported pixel format and filter.  Both run glibc's powf here, so they agree bit for bit;
  the GPU suite holds the device's powf to the one-code / one-ulp / 2^-20 rule of DESIGN.md section 3."""
import os
import re

import numpy as np
import pytest

from directxtex_b200 import formats as F
from tests import oracle_lib, test_gpu_mip_routes as R
from tests.kernel_routes import kernel_entries

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compiled_instantiations():
    """{(family, format, mode, sRGB, LIN)} of every k_mip_box3 / k_mip_tail / k_mip_sep / k_mip_tile kernel compiled into the
    library, in the form of test_gpu_mip_routes.instantiations"""
    out = set()
    for fam, insts in kernel_entries().items():
        for args in insts:
            if fam == "k_mip_box3":                       # <FMT, SRGB, LIN>
                out.add(("box3", args[0], 0, args[1], args[2]))
            elif fam == "k_mip_sep":                      # <FMT, SRGB>
                out.add(("sep", args[0], 0, args[1], False))
            elif fam in ("k_mip_tail", "k_mip_tile"):     # <FMT, MODE, SRGB>
                out.add((fam[len("k_mip_"):], args[0], args[1], args[2], False))
    return out


def test_route_table_reaches_exactly_the_compiled_instantiations():
    """the route table's cases reach every specialised mip kernel in the library and no other, and the kernels are compiled on
    the UNORM twins of the hot formats only"""
    compiled = compiled_instantiations()
    assert len(compiled) == 108, len(compiled)                 # 6 twins x (box3 4 + tail 6 + sep 2 + tile 6)
    assert {fmt for (_, fmt, _, _, _) in compiled} == {R.TWIN.get(f, f) for f in R.HOT}
    reached = set().union(*(R.instantiations(c) for c in R.CASES))
    assert not reached - compiled, sorted(reached - compiled)
    assert not compiled - reached, sorted(compiled - reached)


def test_route_table_cases_are_well_formed():
    seen = set()
    for c in R.CASES:
        assert R.case_id(c) not in seen, R.case_id(c)
        seen.add(R.case_id(c))
        assert c.fams and c.fams <= set(R.FAMILIES), c
        assert c.layout == "host" or c.layout in R.LAYOUTS, c
        assert c.layout != "mixed" or c.items >= 2, c
        n = c.items * sum(F.compute_pitch(c.fmt, w, h)[1] for (w, h) in R.levels_of(c))
        assert n < 100 << 20 or c.items > 3, (R.case_id(c), n)       # host-side buffers of one case stay under 100 MB
    # the items, filters, sRGB variants and shapes the route table promises
    assert {c.items for c in R.CASES} >= {1, 3, 70000}
    assert {R.mode_of(c) for c in R.CASES} == {R.BOX, R.LIN, R.CUB, R.TRI, R.PT}
    assert {c.fl & R.SRGB for c in R.CASES} >= {0, R.SRGB, R.SRGB_IN}
    assert {c.layout for c in R.CASES} == {"host"} | set(R.LAYOUTS)
    assert any(c.fmt not in R.HOT for c in R.CASES)


def _sep_constants():
    src = open(os.path.join(ROOT, "directxtex_b200", "csrc", "dxb_k_rows.cu")).read()
    get = lambda name: re.search(r"#define %s (.+)" % name, src).group(1).split("//")[0].strip()
    tw, th = int(get("DXB_SEP_TW")), int(get("DXB_SEP_TH"))
    assert get("DXB_SEP_MAXC") == "(DXB_SEP_TW * 3 + 4)" and get("DXB_SEP_MAXR") == "(DXB_SEP_TH * 3 + 4)"
    m = re.fullmatch(r"\(1u << (\d+)\)", get("DXB_SEP_MAX_EXTENT"))
    return tw, th, tw * 3 + 4, th * 3 + 4, 1 << int(m.group(1))


def sep_violations(source, dest, tile, slots):
    """dxb_sep_entry's statements in fp32 for every destination coordinate of one axis: (bases outside [0, source - 1],
    tiles of `tile` coordinates whose taps base - 1 .. base + 2 need more than `slots` buffer slots)"""
    u = np.arange(dest, dtype=np.uint32)
    scale = np.float32(source) / np.float32(dest)
    t = (u.astype(np.float32) + np.float32(0.5)) * scale
    base = np.trunc(t - np.float32(0.5)).astype(np.int64)
    outside = int(((base < 0) | (base > source - 1)).sum())
    first = base[::tile]
    last = base[np.minimum(np.arange(tile - 1, dest + tile - 1, tile), dest - 1)]
    return outside, int((last + 2 - (first - 1) + 1 > slots).sum())


def test_sep_extent_limit_keeps_taps_in_the_image_and_the_tile_buffers():
    """the launcher takes k_mip_sep only when every extent is <= DXB_SEP_MAX_EXTENT and source <= 3 x destination; at that bound
    (largest rounding errors) the base tap stays a source pixel and a tile's columns / rows fit rowbuf / H, for same size, the 3:1
    limit, 2:1, upscales and seeded pairs.  Above it they can fail: a same-size row of 12 582 912 pixels rounds its last base to
    the width (the other example of dxb_k_rows.cu, 132 columns in a tile, needs a 179-million-pixel row and is not run here)"""
    tw, th, maxc, maxr, lim = _sep_constants()
    assert lim == 1 << 22
    pairs = [(s_, d) for s_ in (lim, lim - 1, lim - 3) for d in (s_, s_ - 1, -(-s_ // 3), s_ // 3 + 1, -(-s_ // 2), s_ // 2 + 1, (2 * s_) // 3)]
    pairs += [(s_, lim) for s_ in (lim // 3, lim // 2 + 1, lim - 5, 3)] + [(lim, lim - 7), (lim // 3 * 2, lim)]
    rng = np.random.default_rng(22)
    for _ in range(12):
        d = int(rng.integers(lim // 3, lim + 1))
        pairs.append((int(rng.integers(1, min(3 * d, lim) + 1)), d))
    for s_, d in pairs:
        assert s_ <= 3 * d and max(s_, d) <= lim
        assert sep_violations(s_, d, tw, maxc) == (0, 0), (s_, d)
        assert sep_violations(s_, d, th, maxr) == (0, 0), (s_, d)
    assert sep_violations(12582912, 12582912, tw, maxc)[0] > 0          # base rounded up to the width


@pytest.mark.parametrize("sflag", [F.TEX_FILTER_SRGB, F.TEX_FILTER_SRGB_IN, F.TEX_FILTER_SRGB_OUT])
def test_emulator_srgb_mips_match_oracle(oracle, emul, sflag):
    rng = np.random.default_rng(sflag >> 24)
    for fmt in sorted(F.BYTES_PER_PIXEL):
        for mode in (F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, F.TEX_FILTER_POINT):
            for (w, h) in ((32, 16), (16, 2)):
                src = oracle_lib.random_image(fmt, w, h, rng)
                hr, want = oracle.generate_mipmaps(src, w, h, fmt, mode | sflag)
                he, got = emul.generate_mipmaps(src, w, h, fmt, mode | sflag)
                assert hr == 0 and he == 0, (fmt, hex(mode), hex(hr), hex(he))
                assert np.array_equal(got, want), (fmt, hex(mode | sflag), w, h)
