"""CPU suite for the dense sweep of Resize and GenerateMipMaps extents (tests/resize_sweep.py), no GPU needed.

- The host emulator of the mip arithmetic (the inline code every mip kernel runs) equals the oracle bit for bit on every case of
  the sweep, resize and chains, and fails with it where BOX does not halve exactly.  Both run glibc's powf, so sRGB cases are
  bit-exact here too.
- k_mip_sep's fp32 tap coordinates, run as the kernel runs them, stay inside the image and inside its shared-memory tile buffers
  on every axis of every level the sweep expects on k_mip_sep.
- resize_sweep.route() restates dxb_launch_mip_chain: its predicates are pinned to dxb_k_rows.cu here, and it gives the families
  of every case of the route tables of tests/test_gpu_mip_routes.py and tests/address_modes.py, which the GPU suites assert.
- The sweep reaches both sides of the edges it is there for, and stays within its device-time and host-memory budget."""
import collections
import os
import re

import numpy as np
import pytest

from directxtex_b200 import formats as F
from tests import address_modes as A, resize_sweep as S, test_gpu_mip_routes as R
from tests.test_cpu_mip_routes import sep_violations

HOT_SWEPT = (2, 28)


def test_case_counts():
    """prints the case count per operation, filter, format, sRGB and expected families"""
    n = collections.Counter((S.group_id(S.group_key(c)), ",".join(sorted(f[len("k_mip_"):] for f in c.fams)) or "E_FAIL")
                            for c in S.cases())
    for (g, fams), k in sorted(n.items()):
        print("%-28s %-18s %6d" % (g, fams, k))
    print("resize %d, mips %d, device %d" % (len(S.resize_cases()), len(S.chain_cases()), len(S.device_cases())))
    ids = [R.case_id(c) for c in S.cases()]
    assert len(set(ids)) == len(ids)
    assert sum(map(len, S.host_groups().values())) == len(ids) and all(S.host_groups().values())
    assert sum(map(len, S.device_groups().values())) == len(S.device_cases()) and all(S.device_groups().values())


# ---- the route rule ------------------------------------------------------------------------------------------------------
def test_route_rule_is_the_launchers():
    """the predicates route() restates, as they stand in dxb_k_rows.cu: a change to any of them must change route() too"""
    src = open(os.path.join(S.ROOT, "directxtex_b200", "csrc", "dxb_k_rows.cu")).read()
    flat = re.sub(r"\s+", " ", src)
    for text in (
            "if (n > 65535u) return false;",                                               # uniform_batch
            "if ((a0.sw & 7u) || (a0.sh & 7u) || a0.sw < 8u || a0.sh < 8u || !uniform_batch(hj, items)) return false;",
            "if (a.dw != a.sw / 2 || a.dh != a.sh / 2 || b.dw != a.sw / 4 || b.dh != a.sh / 4 || c.dw != a.sw / 8 || c.dh != a.sh / 8) return false;",
            "if (!vec_aligned(a.src, a.srcPitch, 8 * B) || !vec_aligned(a.dst, a.dstPitch, 4 * B) || !vec_aligned(b.dst, b.dstPitch, 2 * B) || !vec_aligned(c.dst, c.dstPitch, B)) return false;",
            "if (lin && (a0.sw > (1u << 23) || a0.sh > (1u << 23))) return false;",
            "const dim3 g((a0.sw / 8 + 31) / 32, (a0.sh / 8 + 7) / 8, items); if (g.y > 65535u) return false;",
            "if (special && uniform_batch(hj, P.njobs))",
            "pixAligned = pixAligned && vec_aligned(hj[i].src, hj[i].srcPitch, dxb_bytes_per_pixel(P.format));",
            "const dim3 gs((j0.dw + DXB_SEP_TW - 1) / DXB_SEP_TW, (j0.dh + DXB_SEP_TH - 1) / DXB_SEP_TH, P.njobs);",
            "const bool sepExtent = j0.sw <= DXB_SEP_MAX_EXTENT && j0.dw <= DXB_SEP_MAX_EXTENT && j0.sh <= DXB_SEP_MAX_EXTENT && j0.dh <= DXB_SEP_MAX_EXTENT;",
            "if (P.mode == DXB_FILTER_CUBIC && pixAligned && sepExtent && j0.sw <= 3u * j0.dw && j0.sh <= 3u * j0.dh && gs.y <= 65535u &&",
            "const uint32_t rowsPerCta = (P.mode == DXB_FILTER_CUBIC) ? 8u * DXB_CUBIC_KY : 8u;",
            "const dim3 g((j0.dw + 31) / 32, (j0.dh + rowsPerCta - 1) / rowsPerCta, P.njobs); if (g.y <= 65535u)",
            "const bool srgb = (P.lflags == (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT));",
            "const bool special = !genericOnly && (srgb || P.lflags == 0) && on_mip_format(P.format, none) && on_mip_mode(P.mode, none);",
            "if (hostJobs[(size_t)(l - 1) * items].sw <= 64 && hostJobs[(size_t)(l - 1) * items].sh <= 64) { tailStart = l; break; }",
            "const bool tail = special && levels - tailStart >= 2 && items <= 0x7FFFFFFFu;",
            "const bool fused = special && P.mode != DXB_FILTER_CUBIC && levels >= 4;",
            "if (fused && l + 2 < levels && (hj[0].sw > 64 || hj[0].sh > 64) && launch_box3(stream, jobs + at, hj, items, P, srgb))",
            "return dxb_on_value<28, 29, 10, 2, 61, 41, 87>(fmt,",
            "return dxb_on_value<DXB_FILTER_BOX, DXB_FILTER_LINEAR, DXB_FILTER_CUBIC>(mode, fn);"):
        assert text in flat, text
    assert (S.SEP_TW, S.SEP_TH, S.CUBIC_KY, S.SEP_MAX_EXTENT) == (32, 16, 4, 1 << 22)
    assert R.HOT == (28, 29, 10, 2, 61, 41, 87)


def test_route_rule_gives_the_route_tables_families():
    """route() on every case and word of the two route tables the GPU suites check against the launch counters"""
    for c in R.CASES:
        assert S.families(c) == c.fams, (R.case_id(c), sorted(S.families(c)), sorted(c.fams))
        assert S.families(c, option=1) == {R.LEVEL}, R.case_id(c)
    n = 0
    for c in A.CASES + A.TRI_GRID:
        for word in c.words:
            for lay in ("host", "pad16"):
                rc = A.route_case(c, word, lay)
                assert S.families(rc) == rc.fams, (R.case_id(rc), sorted(S.families(rc)), sorted(rc.fams))
                n += 1
    assert n > 1000


# ---- the emulator against the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", S.GROUP_KEYS, ids=S.group_id)
def test_emulator_matches_oracle(oracle, emul, key):
    bad = []
    group = S.host_groups()[key]
    for c in group:
        src = R.sources(c)[0]
        if c.resize:
            (ho, want), (he, got) = [x.resize(src, c.w, c.h, c.fmt, c.resize[0], c.resize[1], c.fl) for x in (oracle, emul)]
        else:
            (ho, want), (he, got) = [x.generate_mipmaps(src, c.w, c.h, c.fmt, c.fl) for x in (oracle, emul)]
        if (ho, he) != ((0, 0) if c.fams else (F.E_FAIL, F.E_FAIL)):
            bad.append("%s: HRESULT oracle 0x%08X, emulator 0x%08X" % (R.case_id(c), ho, he))
        elif c.fams and not np.array_equal(got, want):
            bad.append("%s: %d bytes differ" % (R.case_id(c), int((got != want).sum())))
    assert not bad, "%d of %d cases failed:\n%s" % (len(bad), len(group), "\n".join(bad[:40]))


# ---- k_mip_sep's windows -------------------------------------------------------------------------------------------------
def sep_axes():
    """{(source, destination)} of the U axes and of the V axes of every level the sweep runs on k_mip_sep"""
    u, v = set(), set()
    for c in S.cases() + S.device_cases():
        sizes = R.levels_of(c)
        for fam, l, k in S.route(c):
            if fam == R.SEP:
                (sw, sh), (dw, dh) = sizes[l - 1], sizes[l]
                u.add((sw, dw))
                v.add((sh, dh))
    return u, v


def test_sep_taps_stay_in_the_image_and_the_tile_buffers():
    """dxb_sep_entry's fp32 statements on every axis the sweep expects on k_mip_sep: every base tap inside [0, source - 1]
    and every 32-column tile within rowbuf, every 16-row tile within H"""
    u, v = sep_axes()
    assert len(u) > 2000 and len(v) > 2000, (len(u), len(v))
    for s, d in sorted(u):
        assert s <= 3 * d and sep_violations(s, d, S.SEP_TW, S.SEP_MAXC) == (0, 0), (s, d)
    for s, d in sorted(v):
        assert s <= 3 * d and sep_violations(s, d, S.SEP_TH, S.SEP_MAXR) == (0, 0), (s, d)


# ---- what the sweep reaches ----------------------------------------------------------------------------------------------
def swept_axes(c):
    """the (source, destination) pairs of case c's two axes at every level"""
    sizes = R.levels_of(c)
    return [((a[0], b[0]), (a[1], b[1])) for a, b in zip(sizes, sizes[1:])]


def test_sweep_reaches_every_family_per_filter_and_format():
    """each filter on each swept hot format reaches every family the launcher has for it, and the generic format only
    k_mip_level; filter 0 and LINEAR reach k_mip_level on hot formats through the grid's y limit"""
    want = {R.PT: {R.LEVEL}, R.TRI: {R.LEVEL}, R.CUB: {R.SEP, R.TILE, R.TAIL}, R.LIN: {R.BOX3, R.TILE, R.TAIL, R.LEVEL},
            0: {R.BOX3, R.TILE, R.TAIL, R.LEVEL}, R.BOX: {R.BOX3, R.TILE, R.TAIL}}
    reached = collections.defaultdict(set)
    for c in S.cases():
        reached[(S.filter_of(c), c.fmt, S.srgb_of(c))] |= c.fams
    for flt, fams in want.items():
        for fmt in HOT_SWEPT:
            assert reached[(flt, fmt, False)] == fams, (flt, fmt, reached[(flt, fmt, False)])
        assert reached[(flt, 10, False)] <= fams and reached[(flt, 24, False)] == {R.LEVEL}, flt
        assert reached[(flt, 28, True)] and reached[(flt, 28, True)] <= fams, flt
    # every chain shape under BOX either halves (pow2) or fails; every other filter runs every shape
    for c in S.chain_cases():
        assert bool(c.fams) == (S.filter_of(c) != R.BOX or (R.ispow2(c.w) and R.ispow2(c.h))), R.case_id(c)


def test_sweep_reaches_both_sides_of_each_edge():
    for fmt in HOT_SWEPT:
        cub = [c for c in S.resize_cases() if c.fmt == fmt and S.filter_of(c) == R.CUB and not c.fl & ~R.MODE_MASK]
        axes = lambda fam: {swept_axes(c)[0] for c in cub if fam in c.fams}
        sep, tile = axes(R.SEP), axes(R.TILE)
        # exactly 3:1 on k_mip_sep, 3:1 + 1 (and ceil(s / 3) - 1) on k_mip_tile, on both axes
        for k in (0, 1):
            assert any(p[k][0] == 3 * p[k][1] for p in sep), (fmt, k)
            assert any(p[k][0] == 3 * p[k][1] + 1 for p in tile), (fmt, k)
            assert any(p[k][1] == -(-p[k][0] // 3) - 1 and p[k][0] > 48 for p in tile), (fmt, k)
        # destination extents on both sides of k_mip_sep's 32 x 16 tiles and k_mip_tile's 32 x 32 (CUBIC) and 32 x 8 tiles
        assert {p[0][1] for p in sep} >= {31, 32, 33, 63, 64, 65} and {p[1][1] for p in sep} >= {15, 16, 17, 31, 32, 33}
        assert {p[0][1] for p in tile} >= {31, 32, 33} and {p[1][1] for p in tile} >= {31, 32, 33}
        lin = {swept_axes(c)[0] for c in S.resize_cases() if c.fmt == fmt and S.filter_of(c) == R.LIN and R.TILE in c.fams}
        assert {p[1][1] for p in lin} >= {7, 8, 9, 15, 16, 17}
        # chains: k_mip_box3 declined on sizes that are not multiples of 8, the tail from 64 x 64 and odd halvings
        chains = [c for c in S.chain_cases() if c.fmt == fmt]
        assert any(R.BOX3 in c.fams for c in chains if S.filter_of(c) == R.LIN)
        assert any(R.BOX3 not in c.fams and c.w > 64 and c.w % 8 == 0 and c.h % 8 for c in chains if S.filter_of(c) == R.LIN)
        assert any(c.fams == {R.TAIL} and max(c.w, c.h) == 64 for c in chains)
        assert any(c.fams == {R.TILE, R.TAIL} and max(c.w, c.h) == 65 for c in chains)
        pairs = {p for c in chains for lv in swept_axes(c) for p in lv}
        assert {(3, 1), (7, 3), (5, 2), (129, 64)} <= pairs
    # the long thin pairs: POINT's 16.16 step beyond 32 bits, on both axes, up and down
    pt = [c for c in S.resize_cases() if S.filter_of(c) == R.PT]
    for s in S.LONG:
        assert any(c.w == s and c.resize[0] > s for c in pt) and any(c.h == s and c.resize[1] < s for c in pt), s
    # BOX runs on the long rows that halve (65536 -> 32768 over 2 -> 1), on both axes, and fails on the others
    box = [c for c in S.resize_cases() if S.filter_of(c) == R.BOX and max(c.w, c.h) in S.LONG]
    assert {(c.w, c.h) for c in box if c.fams} == {(65536, 2), (2, 65536)}, sorted({(c.w, c.h) for c in box if c.fams})


def test_small_pairs_run_under_every_word():
    """every one-axis pair with an extent of 5 or less runs under every address word of tests/address_modes.py (0 included), on
    each axis, for LINEAR, CUBIC, TRIANGLE and filter 0: the 1-, 2- and 3-pixel sources enlarged under wrap and mirror among them"""
    seen = set()
    for c in S.resize_cases():
        if c.fmt not in HOT_SWEPT or S.srgb_of(c):
            continue
        flt, word = S.filter_of(c), c.fl & ~R.MODE_MASK
        fixed = S.fixed_pair(flt)
        if (c.h, c.resize[1]) == fixed:
            seen.add((flt, 0, (c.w, c.resize[0]), word))
        if (c.w, c.resize[0]) == fixed:
            seen.add((flt, 1, (c.h, c.resize[1]), word))
    small = sorted({p for p in S.DENSE + S.BOUNDARY + S.RANDOM if min(p) <= 5})
    assert {(1, 2), (1, 3), (2, 3), (3, 1), (5, 48), (48, 5)} <= set(small) and len(small) >= 455
    missing = [(S.FILTER_NAME[f], axis, p, hex(w)) for f in S.WORD_FILTERS for axis in (0, 1) for p in small for w in A.WORDS
               if (f, axis, p, w) not in seen]
    assert not missing, (len(missing), missing[:20])


def test_device_cases_cover_the_layouts():
    """the device tenth runs every filter at pad16 and off4; at off4 8- and 16-byte pixels leave k_mip_sep for k_mip_tile"""
    dev = S.device_cases()
    assert {(S.filter_of(c), c.layout) for c in dev} == {(f, lay) for f in S.FILTERS for lay in ("pad16", "off4")}
    moved = [c for c in dev if c.layout == "off4" and c.fmt == 2 and R.SEP in S.with_layout(c, "host").fams]
    assert len(moved) > 100 and all(R.SEP not in c.fams and R.TILE in c.fams for c in moved)
    assert any(c.layout == "pad16" and c.fmt == 2 and R.SEP in c.fams for c in dev)


# ---- budget ----------------------------------------------------------------------------------------------------------------
# Cost of one case of test_gpu_resize_sweep.py (option 0, option 1 and the oracle; device cases also the host API once): per
# launched case, per E_FAIL case, per device case and per pixel of every level.  The model gives 151 s for the sweep as it
# stands; the file took 151 s on one NVIDIA H100 80GB HBM3 at its 700 W power limit.
SECONDS_PER_CASE, SECONDS_PER_FAIL, SECONDS_PER_DEVICE_CASE, SECONDS_PER_PIXEL = 5e-4, 1e-4, 2e-3, 2e-8
BUDGET_SECONDS = 300


def test_budget():
    run = [c for c in S.cases() if c.fams]
    dev = list(S.device_cases())
    pixels = sum(sum(w * h for (w, h) in R.levels_of(c)) for c in run + dev + dev)
    est = (len(run) * SECONDS_PER_CASE + (len(S.cases()) - len(run)) * SECONDS_PER_FAIL + len(dev) * SECONDS_PER_DEVICE_CASE +
           pixels * SECONDS_PER_PIXEL)
    print("cases %d (%d fail), device %d, pixels %d: estimated %.0f s" % (len(S.cases()), len(S.cases()) - len(run), len(dev), pixels, est))
    assert est <= BUDGET_SECONDS
    big = max(list(S.cases()) + dev, key=S.host_bytes)
    assert S.host_bytes(big) < 100 << 20, R.case_id(big)
