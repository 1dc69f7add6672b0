"""CPU suite for the per-axis address modes of GenerateMipMaps and Resize (no GPU needed); the case table is
tests/address_modes.py.

- Teeth: on the reference alone, every word of every case gives the result of another word exactly when address_modes.acting
  says the two read the same taps, for 0, the U/V swap, the word without either axis's bits and without each one bit.  This is
  what lets the GPU suite see a route that swaps, ORs or drops an axis.
- The host emulator of the mip arithmetic (dxb_mips.cuh, the TRIANGLE gather lists of dxb_plan.h, planned as the library plans
  a call) against the reference, bit for bit, for every case and word, mips and resize.
- Route coverage: the table reaches every specialised kernel family on every hot format with a word that is asymmetric
  between U and V, and where the family can see it, one whose U/V swap changes the reference's result."""
import functools

import numpy as np
import pytest

from tests import address_modes as A


@functools.lru_cache(maxsize=None)
def _ref(oracle, c, word):
    return A.oracle_result(oracle, c, word, A.sources(c)[0])


def check_teeth(oracle, c):
    """every word of c against its variants on the reference; returns how many pairs were compared"""
    n = 0
    for word in c.words:
        for v in A.variants(word):
            same = A.same_taps(c, word, v)
            if same is None:
                continue
            eq = np.array_equal(_ref(oracle, c, word), _ref(oracle, c, v))
            assert eq == same, (A.case_id(c), "word %#x vs %#x: the reference's results are %s" % (word, v, "equal" if eq else "different"))
            n += 1
    return n


@pytest.mark.parametrize("c", A.CASES, ids=A.case_id)
def test_reference_tells_the_words_apart(oracle, c):
    assert check_teeth(oracle, c) > 0


def test_reference_tells_the_words_apart_on_triangle_grid(oracle):
    n = sum(check_teeth(oracle, c) for c in A.TRI_GRID)
    assert n > 0


def test_wrap_wins_over_mirror_on_one_axis(oracle):
    """bounduvw takes wrap when both bits of an axis are set: WRAP_U | MIRROR_U reads like WRAP_U, not like MIRROR_U, on CUBIC
    where both act (enlarging U)"""
    c = A.case(28, 7, 5, A.CUB, (A.SEP,), resize=(20, 13))
    assert A.acting(c)[A.WU] and A.acting(c)[A.MU]
    both = _ref(oracle, c, A.WU | A.MU)
    assert np.array_equal(both, _ref(oracle, c, A.WU))
    assert not np.array_equal(both, _ref(oracle, c, A.MU))
    assert not np.array_equal(_ref(oracle, c, A.MU), _ref(oracle, c, 0))


def check_emulator(oracle, emul, c):
    for word in c.words:
        rc = A.route_case(c, word)
        for k, src in enumerate(A.sources(c)):
            if c.resize:
                he, got = emul.resize(src, c.w, c.h, c.fmt, c.resize[0], c.resize[1], rc.fl)
                hr, want = oracle.resize(src, c.w, c.h, c.fmt, c.resize[0], c.resize[1], rc.fl)
            else:
                he, got = emul.generate_mipmaps(src, c.w, c.h, c.fmt, rc.fl)
                hr, want = oracle.generate_mipmaps(src, c.w, c.h, c.fmt, rc.fl)
            assert hr == 0 and he == 0, (A.case_id(c), hex(word), hex(hr), hex(he))
            assert np.array_equal(got, want), (A.case_id(c), "word %#x item %d: emulator != reference" % (word, k))


@pytest.mark.parametrize("c", A.CASES, ids=A.case_id)
def test_emulator_matches_oracle(oracle, emul, c):
    check_emulator(oracle, emul, c)


def test_emulator_matches_oracle_on_triangle_grid(oracle, emul):
    for c in A.TRI_GRID:
        check_emulator(oracle, emul, c)


def test_case_table_is_well_formed():
    ids = [A.case_id(c) for c in A.CASES + A.TRI_GRID]
    assert len(ids) == len(set(ids))
    for c in A.CASES + A.TRI_GRID:
        assert 0 in c.words and c.fams and c.fams <= set(A.R.FAMILIES), A.case_id(c)
        assert set(c.words) >= {A.swap_uv(w) for w in c.words}, A.case_id(c)        # closed under the U/V swap
    assert set().union(*(c.words for c in A.CASES)) == set(A.WORDS)
    assert {c.fmt for c in A.CASES} >= set(A.HOT) | {88, 24}
    assert {A.R.mode_of(A.route_case(c, 0)) for c in A.CASES} == {A.BOX, A.LIN, A.CUB, A.TRI, A.PT}
    assert any(c.fl & A.SRGB and c.fmt == 28 for c in A.CASES) and any(c.items > 1 for c in A.CASES)
    # 1-, 2-, 3- and 5-pixel axes, 1 x N and N x 1, enlarging resizes
    short = {min(c.w, c.h) for c in A.CASES} | {min(c.resize) for c in A.CASES if c.resize}
    assert short >= {1, 2, 3, 5}
    assert any(c.w == 1 and c.h > 1 for c in A.CASES) and any(c.h == 1 and c.w > 1 for c in A.CASES)
    assert any(c.resize and c.resize[0] > c.w and c.resize[1] > c.h for c in A.CASES)
    # the TRIANGLE grid: every source and destination extent 1 .. 9 on each axis
    assert {(c.w, c.resize[0]) for c in A.TRI_GRID if c.h == 6} == {(s, d) for s in range(1, 10) for d in range(1, 10)}
    assert {(c.h, c.resize[1]) for c in A.TRI_GRID if c.w == 6} == {(s, d) for s in range(1, 10) for d in range(1, 10)}


def _reaches(fam, fmt, strict):
    """a case of format fmt on family fam with an asymmetric word; strict: one whose U/V swap changes the reference's result"""
    for c in A.CASES:
        if c.fmt == fmt and fam in c.fams:
            for w in c.words:
                if A.asymmetric(w) and (not strict or A.same_taps(c, w, A.swap_uv(w)) is False):
                    return True
    return False


@pytest.mark.parametrize("fmt", A.HOT)
def test_every_hot_format_sees_asymmetric_words_on_every_family(fmt):
    """k_mip_box3 (BOX, or LINEAR at 2:1) reads no address bit, so it is reached with asymmetric words that must not change its
    result; k_mip_sep, k_mip_tile and k_mip_tail with words whose U/V swap does change it.  Every case also runs on k_mip_level
    with DXB200_OPT_MIP_KERNELS = 1."""
    assert _reaches(A.BOX3, fmt, strict=False)
    for fam in (A.SEP, A.TILE, A.TAIL):
        assert _reaches(fam, fmt, strict=True), (fam, fmt)


def test_generic_kernel_sees_asymmetric_words_on_every_filter():
    """k_mip_level under option 0: a format without specialised kernels and TRIANGLE, each with a word whose swap matters"""
    for fmt in (88, 24):
        assert _reaches(A.LEVEL, fmt, strict=True), fmt
    for mode in (A.CUB, A.LIN, A.TRI):
        assert any(A.LEVEL in c.fams and A.R.mode_of(A.route_case(c, 0)) == mode and
                   any(A.same_taps(c, w, A.swap_uv(w)) is False for w in c.words) for c in A.CASES), mode
