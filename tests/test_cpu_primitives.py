"""The host branches of the shared arithmetic headers against exact references (tests/probe/probe.cu, host build).

The host emulator (tests/emul) is the GPU's stand-in in every CPU quality measurement; where a primitive has a device-only branch the
emulator runs the host branch, so both branches must equal one exact reference.  This module checks the host branch; the device
branch is checked by tests/test_gpu_primitives.py against the same references on the same domains.

Domains up to 2^23 inputs run whole.  Larger ones (up to 2^34, all run whole by the GPU module) run a deterministic subset here, which
keeps the module near 40 s of CPU time on 8 cores: the 2^24 - 1 reciprocals at a stride of 3, the 2^26 exhaustive one-channel palette
searches (nearest1) and the 2^26 random cases of nearest4 and simd at a stride of 9.  The subset is every (2^k + 1)-th index (an odd
stride, so every low mantissa bit pattern occurs) plus, for the float-pattern domains, 2 x 512 patterns around every power of two of either sign (every
exponent boundary, which contains every rounding and clamp boundary of these primitives: 0.5, 1, 2^22, 2^23, 2^31, 2^32, the binary16
limits) and around the values the primitives clamp or round at (0.5 / 255, 254.5 / 255, 65504, 65520, 255, 2^22 - 1/2)."""
import os

import numpy as np
import pytest

from tests import probe_lib

BUDGET = 1 << 23
WINDOW = 512


@pytest.fixture(scope="module")
def probe():
    if not os.path.exists(probe_lib.HOST_SO):
        pytest.fail("tests/probe/_build/libdxb_probe_host.so missing: run __graft_entry__.build()")
    p = probe_lib.Probe(probe_lib.HOST_SO)
    assert not p.on_device
    return p


def _f32_bits(v):
    return int(np.array([v], np.float32).view(np.uint32)[0])


def _boundary_patterns():
    pats = set()
    for e in range(256):
        for s in (0, 1):
            pats.add((s << 31) | (e << 23))
    for v in (0.5 / 255, 254.5 / 255, 1.0 - 0.5 / 255, 65504.0, 65520.0, 255.0, 4194303.5, 254.5, 2.0 ** 24 - 1):
        for s in (1.0, -1.0):
            pats.add(_f32_bits(s * v))
    return sorted(pats)


def _windows(name, begin, count):
    """(begin, count) index windows around the boundary patterns that lie inside a float-pattern domain"""
    npos = probe_lib.FLOAT_NPOS.get(name)
    if npos is None and name != "unorm8":
        return []
    out = []
    for pat in _boundary_patterns():
        if name == "unorm8":
            idxs = [pat + (k << 32) for k in range(4)]
        elif pat < npos:
            idxs = [pat]
        elif pat >= 0x80000000 and npos + (pat - 0x80000000) < begin + count and npos < (1 << 32):
            idxs = [npos + (pat - 0x80000000)]
        else:
            continue
        for i in idxs:
            lo, hi = max(begin, i - WINDOW), min(begin + count, i + WINDOW)
            if lo < hi:
                out.append((lo, hi - lo))
    return out


def _runs(name, begin, count):
    if count <= BUDGET:
        return [(begin, count, 1)]
    k = 1
    while count // ((1 << k) + 1) > BUDGET:
        k += 1
    step = (1 << k) + 1
    return [(begin, (count + step - 1) // step, step)] + [(b, c, 1) for (b, c) in _windows(name, begin, count)]


@pytest.mark.parametrize("name,arg,begin,count", probe_lib.domains(), ids=lambda v: str(v))
def test_host_primitive_equals_reference(probe, name, arg, begin, count):
    """Call sites and why their arguments lie inside each domain are listed in tests/test_gpu_primitives.py; the host build must
    equal the reference on the whole domain."""
    bad, first = 0, []
    for (b, c, s) in _runs(name, begin, count):
        n, recs = probe.run(name, arg, b, c, s)
        bad += n
        first += recs
    assert bad == 0, probe_lib.describe(name, arg, bad, first[:16])


def test_host_outside_preconditions(probe):
    """Outside the preconditions the host keeps the C semantics: a float in (-1, 0) truncates to 0.  An out-of-range float to int32
    conversion gives x86's 0x80000000 where the device saturates: recorded, not required."""
    for (name, arg, begin, count) in probe_lib.RECORDED:
        bad = 0
        for (b, c, s) in _runs(name, begin, count):
            bad += probe.run(name, arg, b, c, s)[0]
        if name == "f2i_out_of_range":
            print("host f2i outside int32: %d of the sampled inputs differ from saturation" % bad)
        else:
            assert bad == 0, name


def test_unknown_check_is_refused(probe):
    import ctypes as C
    out = (C.c_ulonglong * 49)()
    assert probe.L.probe_run(len(probe.ids), 0, 0, 1, 1, C.cast(out, C.c_void_p)) == -1
