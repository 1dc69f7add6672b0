"""Every BC6H and BC7 block the encoders emit, checked one by one against the reference decoder (D3DXDecodeBC6H / D3DXDecodeBC7),
and the decoders on every mode.

The contract against the reference encoder (tests/tolerance.py) is statistical, and the emulator and the device share their packers
and tables, so a packing or mode-choice mistake that touches a few blocks of a rare mode passes both.  Here the host emulator
records, per block, what the encoder chose and the texels its indices select from its palette (tests/bc67_blocks/record_host.cpp),
and every block must
  (a) decode, in the reference decoder, to exactly those texels;
  (b) carry in its bit stream, read by an independent reader of the format, the recorded mode, partition, rotation, index selector
      and indices;
  (c) hold in every index the exhaustive nearest entry of its palette (BC7: and decode with no more error than the stage-3 error
      it was chosen by);
on the contract classes, the special-value corpus, partial blocks, a structured corpus, and (d) every forced mode / partition /
rotation / index-selector cell and, for BC6H, every end of every endpoint and delta field.  (e) The host emulator's decoders equal the oracle's bit for bit on random streams stratified by
mode and endpoint order."""
import numpy as np
import pytest

from directxtex_b200 import formats as F, synth
from tests import bc67_blocks_lib as BL, oracle_lib, special_values as S, tolerance

QUICK, THREE = F.TEX_COMPRESS_BC7_QUICK, F.TEX_COMPRESS_BC7_USE_3SUBSETS


@pytest.fixture(scope="module")
def rec(tmp_path_factory):
    return BL.load(tmp_path_factory.mktemp("bc67_record_host"))


@pytest.fixture(scope="module")
def tables(oracle):
    return BL.Tables(oracle)


def _bc7(rec, emul, oracle, T, img, w, h, sf=2, flags=0, ctx=""):
    blocks, r = BL.record(rec, emul, img, w, h, sf, BL.BC7, flags)
    px = None
    if sf == 2:
        px, full = BL.block_pixels(oracle_lib.bc7_ldr(img), w, h)
        if not full.all():                                      # partial blocks: (c) on the full ones
            R = BL.check_bc7(oracle, T, blocks, r, None, ctx)
            BL.check_bc7(oracle, T, blocks.reshape(-1, 16)[full].reshape(-1), r[full], px[full], ctx)
            return R
    return BL.check_bc7(oracle, T, blocks, r, px, ctx)


def _bc6h(rec, emul, oracle, T, img, w, h, fmt, sf=2, ctx=""):
    blocks, r = BL.record(rec, emul, img, w, h, sf, fmt)
    src = np.asarray(img, np.float32)
    px, full = BL.block_pixels(oracle_lib.bc6h_to_int(src[..., :3], fmt == BL.SF16), w, h)
    R = BL.check_bc6h(oracle, T, blocks, r, fmt, None, ctx)
    BL.check_bc6h(oracle, T, blocks.reshape(-1, 16)[full].reshape(-1), r[full], fmt, px[full], ctx)
    return R


# ---- (a)-(c) on the contract classes, QUICK, special values, partial blocks and the structured corpus ---------------------------
@pytest.mark.parametrize("kind,flags", tolerance.bc7_cases())
def test_bc7_blocks_decode_to_record(rec, emul, oracle, tables, kind, flags):
    n = 128
    _bc7(rec, emul, oracle, tables, synth.content_ldr(kind, n, n, tolerance.SEED), n, n, 2, flags, "%s %#x" % (kind, flags))


def test_bc7_quick_special_values_and_partial_blocks(rec, emul, oracle, tables):
    _bc7(rec, emul, oracle, tables, synth.content_ldr("photo", 64, 64, 3), 64, 64, 2, QUICK, "QUICK")
    base = S.edge_image(64, 20, seed=BL.BC7)
    with np.errstate(over="ignore"):
        big = (base * np.float32(1000.0)).astype(np.float32)
    himg, hh = S.half_image(10, 256)
    for src, w, h, sf, name in ((base, 64, 20, 2, "edges"), (big, 64, 20, 2, "edges x 1000"), (himg, 256, hh, 10, "half patterns")):
        for flags in (0, THREE):
            _bc7(rec, emul, oracle, tables, src, w, h, sf, flags, "%s %#x" % (name, flags))
    _bc7(rec, emul, oracle, tables, synth.content_ldr("text", 37, 21, 2), 37, 21, 2, THREE, "37 x 21")


@pytest.mark.parametrize("alpha", [False, True])
def test_bc7_structured_blocks(rec, emul, oracle, tables, alpha):
    """flat colours and lines on one, two and three subsets of every partition, near-equal colours, opaque / with alpha"""
    modes = np.zeros(8, np.int64)
    for seed, flags in ((1, 0), (2, THREE)):
        px = BL.structured_ldr(tables, 4096, seed + 10 * alpha, alpha)
        img = BL.blocks_to_image(px, 64, 64)
        R = _bc7(rec, emul, oracle, tables, img, 256, 256, 2, flags, "structured alpha=%d %#x" % (alpha, flags))
        modes += np.bincount(R["mode"], minlength=8)
    reached = set(np.nonzero(modes)[0].tolist())
    assert reached >= ({4, 5, 6, 7} if alpha else {0, 1, 2, 3, 4, 5, 6}), modes.tolist()


@pytest.mark.parametrize("kind,fmt", tolerance.bc6h_cases())
def test_bc6h_blocks_decode_to_record(rec, emul, oracle, tables, kind, fmt):
    n = 128
    _bc6h(rec, emul, oracle, tables, synth.content_hdr(kind, n, n, tolerance.SEED), n, n, fmt, 2, kind)


@pytest.mark.parametrize("fmt", [BL.UF16, BL.SF16])
def test_bc6h_special_values_partial_and_structured_blocks(rec, emul, oracle, tables, fmt):
    base = S.edge_image(64, 20, seed=fmt)
    with np.errstate(over="ignore"):
        big = (base * np.float32(1000.0)).astype(np.float32)
    himg, hh = S.half_image(10, 256)
    for src, w, h, sf, name in ((base, 64, 20, 2, "edges"), (big, 64, 20, 2, "edges x 1000"), (himg, 256, hh, 10, "half patterns")):
        blocks, r = BL.record(rec, emul, src, w, h, sf, fmt)
        f32 = src.view(np.float16).astype(np.float32).reshape(h, w, 4) if sf == 10 else src
        px, full = BL.block_pixels(oracle_lib.bc6h_to_int(np.nan_to_num(f32[..., :3], nan=0.0), fmt == BL.SF16), w, h)
        # (c) needs the encoder's INT pixels: the half conversion of a NaN is a NaN pattern, not 0, so blocks with a NaN skip it
        ok = full & ~np.isnan(BL.block_pixels(f32[..., :3], w, h)[0]).any(axis=(1, 2))
        BL.check_bc6h(oracle, tables, blocks, r, fmt, None, name)
        BL.check_bc6h(oracle, tables, blocks.reshape(-1, 16)[ok].reshape(-1), r[ok], fmt, px[ok], name)
    _bc6h(rec, emul, oracle, tables, synth.content_hdr("edges", 37, 21, 2), 37, 21, fmt, 2, "37 x 21")
    modes = np.zeros(14, np.int64)
    for seed in range(3):
        px = BL.structured_hdr(tables, 4096, 10 * seed + fmt, fmt == BL.SF16)
        R = _bc6h(rec, emul, oracle, tables, BL.blocks_to_image(px, 64, 64), 256, 256, fmt, 2, "structured %d" % seed)
        modes += np.bincount(R["mode"], minlength=14)
    assert np.all(modes > 0), modes.tolist()                                           # every mode, unforced


# ---- (d) forced coverage -------------------------------------------------------------------------------------------------------
def test_bc7_every_forced_cell(rec, emul, oracle, tables):
    """Every partition of modes 0, 1, 2, 3 and 7, modes 4 and 5 at every rotation, mode 4 at both index selectors, mode 6, on opaque
    and alpha content; each forced block is emitted in its cell and passes (a)-(c); both p-bit values of every endpoint in every
    mode that has p-bits; and every subset of the three-subset modes stored both as fitted and mirrored by the anchor fix-up."""
    force, px = BL.bc7_forced_cells(tables, per=2, seed=5)
    n = px.shape[0]
    nbx = 64
    nby = (n + nbx - 1) // nbx
    pad = np.concatenate([px, np.ones((nbx * nby - n, 16, 4), np.float32)])
    fpad = np.concatenate([force, np.full((nbx * nby - n, 5), -1, np.int32)])
    img = BL.blocks_to_image(pad, nbx, nby)
    blocks, r = BL.record(rec, emul, img, 4 * nbx, 4 * nby, 2, BL.BC7, THREE, force=fpad)
    lp, _ = BL.block_pixels(oracle_lib.bc7_ldr(img), 4 * nbx, 4 * nby)
    R = BL.check_bc7(oracle, tables, blocks, r, lp, "forced")
    R = {k: v[:n] for k, v in R.items()}
    missed = []
    for i, (m, rot, isel, s2, s3) in enumerate(force):
        got = (R["mode"][i], R["rot"][i] if rot >= 0 else -1, R["idx"][i] if isel >= 0 else -1,
               R["shape"][i] if s2 >= 0 else -1, R["shape"][i] if s3 >= 0 else -1)
        if got != (m, rot, isel, s2, s3):
            missed.append((i, (m, rot, isel, s2, s3), got))
    cells = {tuple(f) for f in force.tolist()}
    reached = {tuple(force[i].tolist()) for i in range(n)} - {tuple(c[1]) for c in missed}
    # every forced block must be emitted in its cell (a cell with one stray block counts as not reached)
    assert reached == cells, "%d of %d forced cells not reached: %s" % (len(cells - reached), len(cells), sorted(cells - reached)[:8])
    for m, epb in ((0, 1), (1, 0), (3, 1), (6, 1), (7, 1)):
        sel = R["mode"] == m
        pb = R["pb"][sel][:, :BL.BC7_MODES[m][0]]
        for e in range(2 if epb else 1):
            seen = set(((pb >> e) & 1).reshape(-1).tolist())
            assert seen == {0, 1}, (m, e, seen)
    for m in (0, 2):
        sel = np.nonzero(R["mode"] == m)[0]
        ib = BL.BC7_MODES[m][8]
        for j in range(3):
            a = tables.anchor3[R["shape"][sel], j] if j else np.zeros(sel.size, np.int64)
            msb = (R["idxC"][sel, a] >> (ib - 1)) & 1
            assert set(msb.tolist()) == {0, 1}, ("anchor flips of mode %d subset %d" % (m, j), set(msb.tolist()))


@pytest.mark.parametrize("fmt", [BL.UF16, BL.SF16])
def test_bc6h_every_forced_cell(rec, emul, oracle, tables, fmt):
    """All 14 modes, every two-region mode at each of the 32 shapes: each cell is emitted and passes (a)-(c)."""
    signed = fmt == BL.SF16
    force, px = BL.bc6h_forced_cells(tables, signed, per=3, seed=7)
    n = px.shape[0]
    nbx = 64
    nby = (n + nbx - 1) // nbx
    pad = np.concatenate([px, np.ones((nbx * nby - n, 16, 4), np.float32)])
    fpad = np.concatenate([force, np.full((nbx * nby - n, 2), -1, np.int32)])
    img = BL.blocks_to_image(pad, nbx, nby)
    blocks, r = BL.record(rec, emul, img, 4 * nbx, 4 * nby, 2, fmt, 0, force=fpad)
    ip, _ = BL.block_pixels(oracle_lib.bc6h_to_int(img[..., :3], signed), 4 * nbx, 4 * nby)
    R = BL.check_bc6h(oracle, tables, blocks, r, fmt, ip, "forced")
    R = {k: v[:n] for k, v in R.items()}
    # a cell is reached when one of its blocks is emitted in it
    hit = (R["mode"] == force[:, 0]) & ((force[:, 1] < 0) | (R["shape"] == force[:, 1]))
    cells = {tuple(f) for f in force.tolist()}
    reached = {tuple(force[i].tolist()) for i in np.nonzero(hit)[0]}
    assert reached == cells, "%d of %d forced cells not reached: %s" % (len(cells - reached), len(cells), sorted(cells - reached)[:8])


@pytest.mark.parametrize("fmt", [BL.UF16, BL.SF16])
def test_bc6h_endpoint_range_cells(rec, emul, oracle, tables, fmt):
    """The ends of every field: in every transformed mode and channel an emitted delta of -2^(n-1) and of 2^(n-1) - 1, and in every
    mode and channel the base endpoint at the lowest code, 0 and the highest code (bc6h_edge_cells).  Blocks are built from chosen
    codes and the mode is forced; every block passes (a)-(c), and a cell is reached when one of its four blocks emits it."""
    signed = fmt == BL.SF16
    force, px, cells = BL.bc6h_edge_cells(tables, signed, variants=4, seed=3)
    n = px.shape[0]
    nbx = 64
    nby = (n + nbx - 1) // nbx
    pad = np.concatenate([px, np.ones((nbx * nby - n, 16, 4), np.float32)])
    fpad = np.concatenate([force, np.full((nbx * nby - n, 2), -1, np.int32)])
    img = BL.blocks_to_image(pad, nbx, nby)
    blocks, r = BL.record(rec, emul, img, 4 * nbx, 4 * nby, 2, fmt, 0, force=fpad)
    ip, _ = BL.block_pixels(oracle_lib.bc6h_to_int(img[..., :3], signed), 4 * nbx, 4 * nby)
    R = BL.check_bc6h(oracle, tables, blocks, r, fmt, ip, "endpoint range")
    R = {k: v[:n] for k, v in R.items()}
    owner = np.array([hash(c) for c in cells])
    missed = [c for c in sorted(set(cells)) if not np.any(BL.bc6h_edge_reached(R, c) & (owner == hash(c)))]
    transformed = sum(1 for m in BL.BC6H_MODES if m[3][0])
    assert len(set(cells)) == transformed * 6 + 14 * 3 * (3 if signed else 2)
    assert not missed, "%d of %d endpoint-range cells not reached: %s" % (len(missed), len(set(cells)), missed[:8])


# ---- (e) the decoders on every mode ---------------------------------------------------------------------------------------------
DECODE_CASES = [(98, 28), (98, 2), (95, 2), (95, 10), (96, 2), (96, 10), (71, 28), (77, 28), (80, 61), (81, 63), (83, 49), (84, 51),
                (80, 2), (81, 2), (84, 2)]


@pytest.mark.parametrize("bc,df", DECODE_CASES)
def test_decoders_on_every_mode(oracle, emul, bc, df):
    """random payloads with the mode field (BC6H, BC7) or the endpoint order (BC1, BC3, BC4, BC5) set: the emulator's decoder equals
    the oracle's bit for bit in every stratum, at a partial-block size"""
    w, h = 26, 18
    nb = ((w + 3) // 4) * ((h + 3) // 4)
    for label, blocks in BL.decoder_streams(bc, nb, seed=bc * 7 + df):
        hr, want = oracle.decompress(blocks, w, h, bc, df)
        he, got = emul.decompress(blocks, w, h, bc, df)
        assert hr == 0 and he == 0, (bc, df, label)
        S.assert_same(got, want, df, "decompress %d -> %d %s" % (bc, df, label))
