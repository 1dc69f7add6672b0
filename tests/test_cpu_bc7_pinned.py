"""BC7 blocks pinned bit for bit (tests/golden/golden_bc7_blocks_v1.npz, written by tests/golden/make_golden_bc7_blocks.py).

The encoder is not bit-exact against the reference, so its tolerance tests pass many block streams.  A change that must keep the
blocks exactly (a faster packer, a different data flow between the stages) is checked here on the host emulator, which the GPU
tests hold equal to the device: every LDR content class with the default flags, USE_3SUBSETS and QUICK, to BC7_UNORM and
BC7_UNORM_SRGB, a crop of the benchmark's image and an image with partial blocks.

Stage 4 packs the winner's fields and p-bits from the decoder's endpoint bytes.  A field of B bits, p-bit included, decodes as
(full << (8 - B)) | (full >> (2 B - 8)), so full = deq >> (8 - B), the field is full >> 1 and the p-bit full & 1 (with a p-bit) or
the field is full (without): checked exhaustively for the field widths and p-bit kinds of every mode."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_bc7_blocks as G  # noqa: E402

# (colour bits, alpha bits, p-bit) of BC7 modes 0..7 (the format's mode table)
BC7_FIELDS = [(4, 0, 1), (6, 0, 1), (5, 0, 0), (7, 0, 1), (5, 6, 0), (7, 8, 0), (7, 7, 1), (5, 5, 1)]
CASES = G.bc7_block_cases()


@pytest.fixture(scope="module")
def golden():
    return np.load(G.OUT)


def test_golden_covers_every_case(golden):
    keys = {k for c in CASES for k in (c[0] + "_in", c[0] + "_out")}
    assert keys == set(golden.files)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_emulator_blocks_equal_pinned(emul, golden, case):
    key, (w, h), make, dst, flags = case
    img = make()
    assert np.array_equal(G.sha1(img), golden[key + "_in"]), "the input generator changed: %s" % key
    hr, blocks = emul.compress(img, w, h, 2, dst, flags)
    assert hr == 0 and np.array_equal(G.sha1(blocks), golden[key + "_out"]), key


def dequantise(full, B):
    """the decoder's byte of a B-bit endpoint value (p-bit included; D3DX_BC7::Unquantize)"""
    return ((full << (8 - B)) | (full >> (2 * B - 8))) & 0xFF


@pytest.mark.parametrize("mode", range(8))
def test_fields_and_pbits_follow_from_the_dequantised_byte(mode):
    cb, ab, p = BC7_FIELDS[mode]
    for bits in {cb, ab} - {0}:
        B = bits + p
        for full in range(1 << B):
            deq = dequantise(full, B)
            assert deq >> (8 - B) == full, (mode, bits, full)
            assert deq >> (8 - bits) == full >> p, (mode, bits, full)          # the field: the byte's top `bits` bits
            if p:
                assert (deq >> (7 - bits)) & 1 == full & 1, (mode, bits, full)  # the p-bit: the bit below them
