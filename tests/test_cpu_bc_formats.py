"""CPU mirror of tests/test_gpu_bc_formats.py: the host lock-step emulator of our kernels against the oracle over every source
format into every BC1-BC5 target (sRGB targets and flags included), every BC source into every destination, and the
BC7_UNORM_SRGB contract against the reference encoder; plus a check that the GPU suite's kernel pair lists name exactly the
specialised instantiations compiled into the library.  No GPU needed."""
import numpy as np
import pytest

from directxtex_b200 import formats as F, synth
from tests import special_values as S, tolerance
from tests import test_gpu_bc_formats as G, test_gpu_mip_routes as R
from tests.kernel_routes import kernel_entries

def twins(pairs):
    """the instantiations the launchers run (a, b) pairs on: each format replaced by its UNORM twin (dxb_make_linear)"""
    return {(R.TWIN.get(a, a), R.TWIN.get(b, b)) for a, b in pairs}


def test_gpu_pair_lists_equal_the_compiled_specialised_kernels():
    """the GPU suite's pair lists name exactly the k_compress_bc15_t and k_decompress_t instantiations compiled into the library:
    a new instantiation cannot go untested, and none is compiled that the lists do not route to"""
    k = kernel_entries()
    assert twins(G.BC15_PAIRS) == k["k_compress_bc15_t"], sorted(twins(G.BC15_PAIRS) ^ k["k_compress_bc15_t"])
    assert twins(G.DEC_PAIRS) == k["k_decompress_t"], sorted(twins(G.DEC_PAIRS) ^ k["k_decompress_t"])
    assert k["k_compress_bc15_t"] <= set(G.BC15_ALIAS_CASES)
    assert k["k_decompress_t"] <= set(G.DECOMPRESS_PAIRS)
    # the sRGB aliases the launchers remap onto the specialised kernels are in the lists too
    for d, s in ((72, 29), (72, 91), (75, 29), (75, 91), (78, 29), (78, 91)):
        assert (d, s) in G.BC15_ALIAS_CASES
    for bc, df in G.EXACT_SRGB_DECOMPRESS + [(72, 28), (78, 28), (99, 28), (99, 2)]:
        assert (bc, df) in G.DECOMPRESS_PAIRS


def test_srgb_resolution_and_exact_pairs():
    """the flags each case resolves to: sRGB on both sides cancels (exact), one side converts (powf)"""
    IN, OUT = F.TEX_FILTER_SRGB_IN, F.TEX_FILTER_SRGB_OUT
    for bc, df in G.EXACT_SRGB_DECOMPRESS:
        assert S.powf_direction(0, bc, df) == 0, (bc, df)
    assert S.powf_direction(0, 72, 28) == IN and S.powf_direction(0, 99, 2) == IN and S.powf_direction(0, 99, 31) == IN
    assert S.powf_direction(0, 28, 72) == OUT and S.powf_direction(0, 2, 99) == OUT and S.powf_direction(0, 29, 95) == IN
    assert S.powf_direction(IN, 28, 72) == 0 and S.powf_direction(F.TEX_COMPRESS_SRGB, 28, 71) == 0
    assert S.powf_direction(IN, 31, 71) == 0 and S.powf_direction(OUT, 31, 71) == OUT and S.powf_direction(OUT, 28, 81) == 0
    assert S.powf_direction(IN, 65, 71) == 0 and S.powf_direction(0, 29, 91) == 0


@pytest.mark.parametrize("fmt", sorted(F.BYTES_PER_PIXEL))
def test_srgb_safe_image(fmt):
    """right size, deterministic, and at least a quarter of the candidate values kept (every value without a GPU)"""
    for d in (F.TEX_FILTER_SRGB_IN, F.TEX_FILTER_SRGB_OUT):
        a = S.srgb_safe_image(fmt, d, 22, 14, seed=5)
        assert a.dtype == np.uint8 and a.size == 22 * 14 * F.BYTES_PER_PIXEL[fmt]
        assert np.array_equal(a, S.srgb_safe_image(fmt, d, 22, 14, seed=5))
        kept, total = S.SRGB_SAFE_FRACTIONS[(fmt, d)]
        assert total == 0 or kept >= 0.25 * total


@pytest.mark.parametrize("sf", sorted(F.BYTES_PER_PIXEL))
def test_compress_every_source_into_every_bc15_target(oracle, emul, sf):
    n = 0
    for df in G.BC15_TARGETS:
        for fl in G.COMPRESS_FLAGS:
            for (w, h) in G.SIZES:
                src = G.compress_source(sf, df, fl, w, h, seed=w + df)
                hr, want = oracle.compress(src, w, h, sf, df, fl)
                he, got = emul.compress(src, w, h, sf, df, fl)
                assert hr == 0 and he == 0, (sf, df, hex(fl))
                S.assert_same(got, want, df, "BC %d from %d flags %#x %dx%d" % (df, sf, fl, w, h))
                n += 1
    assert n == len(G.BC15_TARGETS) * len(G.COMPRESS_FLAGS) * len(G.SIZES)


@pytest.mark.parametrize("bc", sorted(F.BLOCK_BYTES))
def test_decompress_every_bc_source_into_every_destination(oracle, emul, bc):
    """bit for bit everywhere: the emulator and the oracle share glibc's powf"""
    for (w, h) in ((13, 9), (32, 16)):
        for kind, blocks in G.bc_streams(oracle, bc, w, h, seed=bc * 31 + w):
            for df in sorted(F.BYTES_PER_PIXEL):
                hr, want = oracle.decompress(blocks, w, h, bc, df)
                he, got = emul.decompress(blocks, w, h, bc, df)
                assert hr == 0 and he == 0, (bc, df)
                S.assert_same(got, want, df, "decompress %d -> %d %s %dx%d" % (bc, df, kind, w, h))


@pytest.mark.parametrize("kind", ["photo", "gradient", "alpha_photo"])
def test_bc7_srgb_contract_emulator_vs_reference(oracle, emul, kind):
    """the emulator's RGBA32F -> BC7_UNORM_SRGB stream meets the BC7 contract against the live reference encoder's, both
    measured against the reference's sRGB encoding of the source (the GPU suite checks the device the same way)"""
    n = tolerance.SIZE
    img = synth.content_ldr(kind, n, n, tolerance.SEED)
    he, got = emul.compress(img, n, n, 2, 99)
    hr, ref = oracle.compress(img, n, n, 2, 99)
    assert he == 0 and hr == 0
    ratio = G.check_bc7_srgb_contract(oracle, got, ref, img, kind)
    print("BC7_UNORM_SRGB %s: MSE %.3f x the reference's" % (kind, ratio))
