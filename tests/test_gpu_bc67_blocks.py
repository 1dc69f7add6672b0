"""The sm_90a BC6H and BC7 encoders and the decoders, block by block (see tests/test_cpu_bc67_blocks.py for the checks).

Encoders: the structured corpus, the special-value corpus and the contents of the forced cells (here unforced) through
k_compress_bc7 and k_compress_bc7_tma (DXB200_OPT_BC7_FEED 0 and 1) and k_compress_bc6h from RGBA32F and RGBA16F.  The device's
blocks equal the host emulator's, block for block, and the reference decoder returns the texels the emulator recorded for each.  The
corpus must keep reaching every BC7 mode, every BC6H mode, and the BC7 rotation / index-selector cells listed below.
Decoders: random block streams stratified by mode and endpoint order through the host API and through a padded device destination,
on k_decompress_t and on k_decompress: bit for bit the oracle."""
import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import bc67_blocks_lib as BL, oracle_lib, special_values as S
from tests.kernel_routes import launched
from tests.test_gpu_bc_formats import decompress_kernel, device_call

pytestmark = pytest.mark.gpu
THREE = F.TEX_COMPRESS_BC7_USE_3SUBSETS
BC7_KERNELS = ("k_compress_bc7_tma", "k_compress_bc7")
DEC_KERNELS = ("k_decompress_t", "k_decompress")
# (mode, rotation, index selector) cells of modes 4 and 5: the unforced corpus reaches all twelve
BC7_ROT_CELLS = {(4, 0, 0), (4, 0, 1), (4, 1, 0), (4, 1, 1), (4, 2, 0), (4, 2, 1), (4, 3, 0), (4, 3, 1), (5, 0, 0), (5, 1, 0), (5, 2, 0), (5, 3, 0)}


@pytest.fixture(scope="module", autouse=True)
def _init():
    assert capi.lib.dxb200_init(0) == 0


@pytest.fixture(scope="module")
def rec(tmp_path_factory):
    return BL.load(tmp_path_factory.mktemp("bc67_record_host"))


@pytest.fixture(scope="module")
def tables(oracle):
    return BL.Tables(oracle)


def _square(px):
    """[n, 16, C] blocks -> an image 64 blocks wide, padded with copies of the first block"""
    n = px.shape[0]
    nby = (n + 63) // 64
    pad = np.concatenate([px, np.repeat(px[:1], 64 * nby - n, 0)])
    return BL.blocks_to_image(pad, 64, nby), 256, 4 * nby


def bc7_corpus(T):
    """(name, RGBA32F image, w, h, flags)"""
    out = []
    for alpha in (False, True):
        for flags in (0, THREE):
            img, w, h = _square(BL.structured_ldr(T, 4096, 3 + alpha + 2 * flags // THREE, alpha))
            out.append(("structured alpha=%d" % alpha, img, w, h, flags))
    _, px = BL.bc7_forced_cells(T, per=2, seed=5)
    img, w, h = _square(px)
    out += [("forced-cell content", img, w, h, 0), ("forced-cell content", img, w, h, THREE)]
    base = S.edge_image(64, 20, seed=BL.BC7)
    with np.errstate(over="ignore"):
        big = (base * np.float32(1000.0)).astype(np.float32)
    out += [("edges", base, 64, 20, THREE), ("edges x 1000", big, 64, 20, 0)]
    return out


def test_bc7_blocks_on_both_kernels(rec, emul, oracle, tables):
    modes, cells = np.zeros(8, np.int64), set()
    feed = capi.lib.dxb200_get_option(capi.OPT_BC7_FEED)
    try:
        for name, img, w, h, flags in bc7_corpus(tables):
            blocks, r = BL.record(rec, emul, img, w, h, 2, BL.BC7, flags)
            R = BL.check_bc7(oracle, tables, blocks, r, None, name)
            modes += np.bincount(R["mode"], minlength=8)
            sep = np.isin(R["mode"], (4, 5))
            cells |= set(zip(R["mode"][sep].tolist(), R["rot"][sep].tolist(), R["idx"][sep].tolist()))
            for f, kernel in ((0, "k_compress_bc7"), (1, "k_compress_bc7_tma")):
                assert capi.lib.dxb200_set_option(capi.OPT_BC7_FEED, f) == 0
                got, ran = launched(BC7_KERNELS, capi.compress, img, w, h, 2, BL.BC7, flags)
                assert ran == {kernel}, (name, flags, ran)
                nd = np.nonzero(np.any(got.reshape(-1, 16) != blocks.reshape(-1, 16), axis=1))[0]
                assert nd.size == 0, "%s %#x on %s: %d blocks differ from the emulator, first %d (mode %d)" % (
                    name, flags, kernel, nd.size, nd[0], R["mode"][nd[0]])
    finally:
        capi.lib.dxb200_set_option(capi.OPT_BC7_FEED, feed)
    print("BC7 modes on the device:", modes.tolist(), "rotation / index-selector cells:", sorted(cells))
    assert np.all(modes > 0), modes.tolist()
    assert cells >= BC7_ROT_CELLS, sorted(BC7_ROT_CELLS - cells)


@pytest.mark.parametrize("fmt", [BL.UF16, BL.SF16])
def test_bc6h_blocks_from_f32_and_f16(rec, emul, oracle, tables, fmt):
    signed = fmt == BL.SF16
    modes = np.zeros(14, np.int64)
    corpus = []
    for seed in range(3):
        img, w, h = _square(BL.structured_hdr(tables, 4096, 10 * seed + fmt, signed))
        corpus.append(("structured %d" % seed, img, w, h))
    _, px = BL.bc6h_forced_cells(tables, signed, per=1, seed=7)
    img, w, h = _square(px)
    corpus.append(("forced-cell content", img, w, h))
    _, px, _ = BL.bc6h_edge_cells(tables, signed, variants=1, seed=3)
    img, w, h = _square(px)
    corpus.append(("endpoint-range content", img, w, h))
    base = S.edge_image(64, 20, seed=fmt)
    corpus.append(("edges", base, 64, 20))
    for name, img, w, h in corpus:
        with np.errstate(over="ignore"):                        # the edge corpus holds values beyond the half range
            f16 = np.ascontiguousarray(img.astype(np.float16))
        for sf, src in ((2, img), (10, f16)):
            blocks, r = BL.record(rec, emul, src, w, h, sf, fmt)
            R = BL.check_bc6h(oracle, tables, blocks, r, fmt, None, "%s from %d" % (name, sf))
            if sf == 2:
                modes += np.bincount(R["mode"], minlength=14)
            got, ran = launched(("k_compress_bc6h",), capi.compress, src, w, h, sf, fmt)
            assert ran == {"k_compress_bc6h"}, ran
            nd = np.nonzero(np.any(got.reshape(-1, 16) != blocks.reshape(-1, 16), axis=1))[0]
            assert nd.size == 0, "%s from %d: %d blocks differ from the emulator, first %d (mode %d)" % (name, sf, nd.size, nd[0], R["mode"][nd[0]])
    print("BC6H %d modes on the device:" % fmt, modes.tolist())
    assert np.all(modes > 0), modes.tolist()


DEVICE_DECODE = [(98, 28), (95, 2), (96, 2), (71, 28), (77, 28), (80, 61), (81, 63), (83, 49), (84, 51),
                 (98, 2), (95, 10), (96, 10), (81, 2), (84, 2)]


@pytest.mark.parametrize("bc,df", DEVICE_DECODE)
def test_decoders_on_every_mode(oracle, bc, df):
    w, h = 26, 18
    nb = ((w + 3) // 4) * ((h + 3) // 4)
    row = w * F.BYTES_PER_PIXEL[df]
    want_kernel = decompress_kernel(bc, df)
    for label, blocks in BL.decoder_streams(bc, nb, seed=bc * 7 + df):
        hr, want = oracle.decompress(blocks, w, h, bc, df)
        assert hr == 0
        for path, (got, ran) in (("host", launched(DEC_KERNELS, capi.decompress, blocks, w, h, bc, df)),
                                 ("device", launched(DEC_KERNELS, device_call, capi.lib.dxb200_decompress_device, (df,), blocks, w, h, bc, df,
                                                     dpitch=((row + 15) & ~15) + 16))):
            assert ran == {want_kernel}, (bc, df, path, ran)
            S.assert_same(got, want, df, "decompress %d -> %d %s on %s" % (bc, df, label, path))
