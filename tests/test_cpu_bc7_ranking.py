"""BC7 stage-1 shape ranking (dxb_bc7.cuh, dxb_bc7_encode_pair): the ranking runs part B of dxb_bc7_shape_h1 (the index-quantisation
term) only for the shapes whose residual lower bound can still reach a selected key.  The shapes it selects must be exactly those
of the exhaustive ranking: the 2 (opaque block) / 3 (alpha block) smallest keys (bits(dxb_bc7_shape_h1) & ~63) | shape over all 64
two-subset shapes.  tests/bc7_ranking/rank_host.cpp (the host emulator plus the encoder's host-only stage-1 record) returns, per
block, the shapes it selected, whether the block is opaque and the key of every shape; its blocks must equal the emulator's.  The
device runs the same source and is held to the emulator by the GPU parity tests."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import formats as F, synth
from tests import bc7_ranking_build as B
from tests import special_values as S

BC7 = 98


@pytest.fixture(scope="module")
def rank(tmp_path_factory):
    L = B.host_lib("rank_host.cpp", tmp_path_factory.mktemp("bc7_rank_host"))
    L.rank_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4
    L.rank_compress.restype = C.c_int32
    return L


def _ranking(rank, emul, src, w, h, src_fmt, flags):
    """(selected shapes + opaque flag [blocks, 4], keys [blocks, 64], part-B rounds per block pair)"""
    src = np.ascontiguousarray(src)
    nb = ((w + 3) // 4) * ((h + 3) // 4)
    sel = np.full((nb, 4), -1, np.int32)
    key = np.zeros((nb, 64), np.uint32)
    rounds = np.full((nb + 1) // 2, -1, np.int32)
    blocks = np.zeros(nb * 16, np.uint8)
    hr = rank.rank_compress(src.ctypes.data, w, h, src_fmt, flags, blocks.ctypes.data, sel.ctypes.data, key.ctypes.data, rounds.ctypes.data)
    assert hr == 0
    hr, want = emul.compress(src, w, h, src_fmt, BC7, flags)
    assert hr == 0 and np.array_equal(blocks, want)                              # recording changes nothing
    return sel, key, rounds


def _check(rank, emul, src, w, h, src_fmt, flags=0, ctx=""):
    sel, key, rounds = _ranking(rank, emul, src, w, h, src_fmt, flags)
    assert np.all(sel >= 0) and np.all(rounds >= 0), ctx
    assert np.all(np.sort(key & 63, axis=1) == np.arange(64)), ctx              # one key per shape
    best = (np.sort(key, axis=1) & 63).astype(np.int32)
    for opaque, n in ((1, 2), (0, 3)):                                           # sel[2] is read for alpha blocks only
        m = sel[:, 3] == opaque
        bad = np.nonzero(np.any(sel[m, :n] != best[m, :n], axis=1))[0]
        assert bad.size == 0, "%s: %d %s blocks select other shapes than the exhaustive ranking; block %d: %s, exhaustive %s" % (
            ctx, bad.size, "opaque" if opaque else "alpha", np.nonzero(m)[0][bad[0]], sel[m][bad[0], :n].tolist(), best[m][bad[0], :n].tolist())
    if flags & F.TEX_COMPRESS_BC7_QUICK:
        assert np.all(rounds == 0), ctx                                          # every key is the shape: no part runs
    else:
        assert rounds.min() >= 1 and rounds.max() <= 4, ctx                      # round 0 + at most 48 survivors / 16
    return sel, rounds


@pytest.mark.parametrize("kind", synth.LDR_CLASSES)
def test_selected_shapes_equal_exhaustive_ranking(rank, emul, kind):
    img = synth.content_ldr(kind, 256, 256)
    sel, rounds = _check(rank, emul, img, 256, 256, 2, 0, kind)
    if kind in ("alpha_uncorr", "alpha_photo", "cutout"):
        assert np.any(sel[:, 3] == 0), kind                                      # the alpha path is exercised


def test_selected_shapes_equal_exhaustive_ranking_special_values(rank, emul):
    """The fp32 edge corpus, the corpus x 1000 and every half pattern (the inputs of the BC7 special-value parity test)."""
    base = S.edge_image(64, 20, seed=BC7)
    with np.errstate(over="ignore"):
        big = (base * np.float32(1000.0)).astype(np.float32)
    himg, hh = S.half_image(10, 256)
    for src, w, h, sf, name in ((base, 64, 20, 2, "edges"), (big, 64, 20, 2, "edges x 1000"), (himg, 256, hh, 10, "half patterns")):
        _check(rank, emul, src, w, h, sf, 0, name)


def test_quick_selects_the_first_shapes(rank, emul):
    """BC7_QUICK keys every shape by its index alone: shapes 0, 1, 2, and no part of the estimate runs."""
    img = synth.content_ldr("photo", 64, 64)
    sel, _ = _check(rank, emul, img, 64, 64, 2, F.TEX_COMPRESS_BC7_QUICK, "quick")
    assert np.all(sel[:, :3] == [0, 1, 2])


def test_odd_block_count_and_partial_blocks(rank, emul):
    """A last pair with one block (the other half encodes a padding block) and partial edge blocks."""
    img = synth.content_ldr("text", 37, 21)
    _check(rank, emul, img, 37, 21, 2, 0, "37 x 21")
