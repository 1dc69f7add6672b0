"""CPU suite: BC6H and BC7 compression from every implemented source format, with every sRGB flag, anchored on the reference's
own encoder input (tests/bc67_sources_lib.py).  For every case the source's blocks equal the blocks of X, the RGBA32F image of
the floats CompressBC hands the encoder, byte for byte:

  (R) on the reference, for the case's target and, for BC7, its bit-exact BC3 twin: the recipe that builds X is right;
  (E) on the host emulator, which runs the library's planner, load, conversion and encoders: the library turns every source
      format into the reference's encoder input.

The BC6H / BC7 encoders are not bit-exact with the reference's, so only relations like these can pin the conversion layer in
front of them; device == emulator cannot see a mistake in code the two share.  A completeness check keeps the case table
spanning every source format the library's planner accepts.  No GPU needed."""
import numpy as np
import pytest

from directxtex_b200 import formats as F
from tests import bc67_sources_lib as L


def _by_source(sf):
    return [c for c in L.CASES if c.sf == sf]


def test_case_table_spans_every_implemented_source_target_and_srgb_flag(emul):
    """The sources the library's planner (plan_compress, through the emulator) accepts for BC7 are exactly the table's, and the
    table has every one of them into every BC6H / BC7 target with every sRGB flag at both sizes: a newly implemented format
    cannot go untested.  The extra flag sets run on the sources their class names."""
    buf = np.zeros(4 * 4 * 16, np.uint8)
    accepted = {fmt for fmt in range(1, 192) if emul.compress(buf, 4, 4, fmt, 98)[0] == 0}
    assert accepted == set(F.BYTES_PER_PIXEL) == set(L.SOURCES), sorted(accepted ^ set(L.SOURCES))
    for T in L.TARGETS:
        assert {fmt for fmt in range(1, 192) if emul.compress(buf, 4, 4, fmt, T)[0] == 0} == accepted, T
    have = set(L.CASES)
    missing = [L.Case(sf, T, f, w, h) for sf in L.SOURCES for T in L.TARGETS for f in L.SRGB_FLAGS for (w, h) in L.SIZES
               if L.Case(sf, T, f, w, h) not in have]
    assert not missing, [L.case_id(c) for c in missing[:8]]
    assert len(have) == len(L.CASES)
    for sf in L.DITHER_SOURCES:
        assert {c.T for c in L.CASES if c.sf == sf and c.flags & L.DITHER_UNIFORM == L.DITHER_UNIFORM} == set(L.TARGETS)
    S = L.S
    cls = L.BC7_CLASS_SOURCES
    assert cls["SNORM"] in S.SNORM_FORMATS and cls["sRGB"] in S.SRGB_FORMATS and cls["POS_ONLY float"] in (26, 67)
    assert cls["packed BGR"] in S.PACKED16 and cls["R only"] in (41, 54, 56, 58, 61, 63) and cls["no alpha"] in (6, 26, 67, 85, 88, 93)
    for sf in cls.values():
        for f in (L.QUICK, L.THREE):
            assert {c.T for c in L.CASES if c.sf == sf and c.flags & f} == {98, 99}, (sf, f)


@pytest.mark.parametrize("sf", L.SOURCES)
def test_reference_blocks_from_source_equal_blocks_from_its_encoder_input(oracle, sf):
    """(R): oracle.compress(src, sf -> T, f) == oracle.compress(X, RGBA32F -> T', f_X) for every case of this source, and the
    same for BC7's BC3 twin."""
    cases = _by_source(sf)
    srcs = [L.case_source(c) for c in cases]
    results = L.parallel_map(lambda cs: L.reference_relation(oracle, *cs), list(zip(cases, srcs)))
    bad = ["%s as %d: %d blocks differ" % (L.case_id(c), T, L.differing_blocks(a, b))
           for c, res in zip(cases, results) for (T, a, b) in res if not np.array_equal(a, b)]
    assert not bad, "%d of %d cases differ; first: %s" % (len(bad), len(cases), "; ".join(bad[:6]))


@pytest.mark.parametrize("sf", L.SOURCES)
def test_emulator_blocks_from_source_equal_blocks_from_the_reference_encoder_input(oracle, emul, sf):
    """(E): emul.compress(src, sf -> T, f) == emul.compress(X, RGBA32F -> T', f_X), X built by the reference."""
    bad, cases = [], _by_source(sf)
    for c in cases:
        src = L.case_source(c)
        x, Tx, fx = L.encoder_input(oracle, src, c.w, c.h, c.sf, c.T, c.flags)
        he1, direct = emul.compress(src, c.w, c.h, c.sf, c.T, c.flags)
        he2, via_x = emul.compress(x, c.w, c.h, 2, Tx, fx)
        assert he1 == 0 and he2 == 0, L.case_id(c)
        if not np.array_equal(direct, via_x):
            bad.append("%s: %d blocks differ" % (L.case_id(c), L.differing_blocks(direct, via_x)))
    assert not bad, "%d of %d cases differ; first: %s" % (len(bad), len(cases), "; ".join(bad[:6]))
