"""GPU suite: BC6H and BC7 compression from every implemented source format, with every sRGB flag, anchored on the reference's
own encoder input (tests/bc67_sources_lib.py; the CPU half checks the recipe on the reference and the emulator).

(D) For every case the device's blocks from the source equal its blocks from X (the RGBA32F image of the floats the reference's
CompressBC hands the encoder) and the emulator's blocks from the source, byte for byte, through the host API and through
dxb200_compress_device with padded rows at an unaligned base pointer.  Sources come from special_values.srgb_safe_image where a
powf step runs, so that the device's sRGB steps see values on which CUDA's and glibc's powf agree.  Non-RGBA32F sources run
k_compress_bc7 or k_compress_bc6h (the gather of their own that these kernels restate); X of full blocks also runs on
k_compress_bc7_tma, with the same blocks as the direct kernel.  An array of three images of one non-float source, and the fused
mip-and-compress and own-levels paths on four sources, equal the separate calls (D) anchors."""
import contextlib

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import bc67_sources_lib as L
from tests.kernel_routes import launched
from tests.test_gpu_bc_formats import device_call

pytestmark = pytest.mark.gpu
KERNELS = ("k_compress_bc7", "k_compress_bc7_tma", "k_compress_bc6h")


@pytest.fixture(scope="module", autouse=True)
def _init():
    assert capi.lib.dxb200_init(0) == 0


def kernel(T):
    return "k_compress_bc6h" if T in L.BC6H else "k_compress_bc7"


@contextlib.contextmanager
def bc7_feed(mode):
    old = capi.lib.dxb200_get_option(capi.OPT_BC7_FEED)
    assert capi.lib.dxb200_set_option(capi.OPT_BC7_FEED, mode) == 0
    try:
        yield
    finally:
        capi.lib.dxb200_set_option(capi.OPT_BC7_FEED, old)


def _report(bad, total):
    assert not bad, "%d of %d cases differ; first: %s" % (len(bad), total, "; ".join(bad[:6]))


@pytest.mark.parametrize("sf", L.SOURCES)
def test_device_blocks_from_source_equal_blocks_from_the_reference_encoder_input(oracle, emul, sf):
    """(D) for every case of this source: host API from the source == host API from X == emulator from the source; the device
    API from a copy of the source with rows 4 bytes longer than tight at a base pointer 4 bytes past an aligned one gives the same
    blocks; every call of the source runs k_compress_bc7 / k_compress_bc6h.  For BC7 at 32 x 16, X on k_compress_bc7_tma
    (DXB200_OPT_BC7_FEED 1) and on the direct kernel (0) gives the same blocks."""
    bad, cases = [], [c for c in L.CASES if c.sf == sf]
    for c in cases:
        ctx = L.case_id(c)
        src = L.case_source(c)
        x, Tx, fx = L.encoder_input(oracle, src, c.w, c.h, c.sf, c.T, c.flags)
        he, em = emul.compress(src, c.w, c.h, c.sf, c.T, c.flags)
        assert he == 0, ctx
        got, ran = launched(KERNELS, capi.compress, src, c.w, c.h, c.sf, c.T, c.flags)
        via_x, ran_x = launched(KERNELS, capi.compress, x, c.w, c.h, 2, Tx, fx)
        row = c.w * F.BYTES_PER_PIXEL[c.sf]
        dev, ran_dev = launched(KERNELS, device_call, capi.lib.dxb200_compress_device, (c.T, c.flags, 0.5, 1.0), src, c.w, c.h,
                                c.sf, c.T, row + 4, 4)
        if not np.array_equal(got, em):
            bad.append("%s: %d blocks differ from the emulator" % (ctx, L.differing_blocks(got, em)))
        if not np.array_equal(got, via_x):
            bad.append("%s: %d blocks differ from X's" % (ctx, L.differing_blocks(got, via_x)))
        if not np.array_equal(dev, got):
            bad.append("%s: device layout: %d blocks differ" % (ctx, L.differing_blocks(dev, got)))
        if ran != {kernel(c.T)} or ran_dev != {kernel(c.T)} or ran_x != {kernel(c.T)}:
            bad.append("%s: ran %s / %s / X %s" % (ctx, sorted(ran), sorted(ran_dev), sorted(ran_x)))
        if c.T in (98, 99) and (c.w, c.h) == (32, 16):
            with bc7_feed(1):
                tma, ran_t = launched(KERNELS, capi.compress, x, c.w, c.h, 2, Tx, fx)
            with bc7_feed(0):
                direct, ran_d = launched(KERNELS, capi.compress, x, c.w, c.h, 2, Tx, fx)
            if ran_t != {"k_compress_bc7_tma"} or ran_d != {"k_compress_bc7"} or not np.array_equal(tma, via_x) or not np.array_equal(direct, via_x):
                bad.append("%s: X on %s / %s: %d / %d blocks differ" % (ctx, sorted(ran_t), sorted(ran_d), L.differing_blocks(tma, via_x),
                                                                        L.differing_blocks(direct, via_x)))
    _report(bad, len(cases))


@pytest.mark.parametrize("T", L.TARGETS)
def test_array_of_three_non_float_images(oracle, emul, T):
    """Three R10G10B10A2_UNORM images in one call, with every sRGB flag, at both sizes: each image's blocks equal the device's
    blocks from its X and the emulator's from the image, on k_compress_bc7 / k_compress_bc6h."""
    bad, total = [], 0
    for f in L.SRGB_FLAGS:
        for (w, h) in L.SIZES:
            srcs = [L.source(24, T, f, w, h, seed=77 + 5 * i + w) for i in range(3)]
            outs, ran = launched(KERNELS, capi.compress_array, srcs, w, h, 24, T, f)
            if ran != {kernel(T)}:
                bad.append("flags %#x %dx%d ran %s" % (f, w, h, sorted(ran)))
            for i, (src, got) in enumerate(zip(srcs, outs)):
                total += 1
                x, Tx, fx = L.encoder_input(oracle, src, w, h, 24, T, f)
                he, em = emul.compress(src, w, h, 24, T, f)
                assert he == 0
                if not np.array_equal(got, capi.compress(x, w, h, 2, Tx, fx)) or not np.array_equal(got, em):
                    bad.append("flags %#x %dx%d image %d" % (f, w, h, i))
    _report(bad, total)


# the fused paths on one source per class: UNORM 16-bit, packed UNORM into an sRGB target, SNORM into signed BC6H, shared exponent
FUSED = [(11, 98), (24, 99), (13, 96), (67, 95)]


@pytest.mark.parametrize("sf,T", FUSED)
def test_mipmaps_compress_equals_separate_calls(sf, T):
    """dxb200_mipmaps_compress of two images == dxb200_generate_mipmaps then one dxb200_compress per level, byte for byte"""
    w, h = 40, 24
    srcs = [L.S.source_image(sf, w, h, seed=91 + i) for i in range(2)]
    outs = capi.mipmaps_compress(srcs, w, h, sf, T)
    for i, (src, got) in enumerate(zip(srcs, outs)):
        chain, layout = capi.generate_mipmaps(src, w, h, sf, 0)
        two = np.concatenate([capi.compress(chain[off:off + sl], lw, lh, sf, T) for (off, lw, lh, row, sl) in layout])
        assert np.array_equal(got, two), "%d -> %d image %d: %d blocks differ" % (sf, T, i, L.differing_blocks(got, two))


@pytest.mark.parametrize("sf,T", FUSED)
def test_levels_from_equals_one_compress_over_all_levels(sf, T):
    """dxb200_levels_from of two items with three levels of their own == one dxb200_compress of each item's levels as an array"""
    sizes = [(22, 14), (11, 7), (5, 3)]
    items = [[L.S.source_image(sf, lw, lh, seed=13 * i + l) for l, (lw, lh) in enumerate(sizes)] for i in range(2)]
    outs, _ = capi.levels_from(items, sizes, sf, T)
    for i, item in enumerate(items):
        want = capi.compress_images(item, sizes, sf, T)
        for l, (got, wl) in enumerate(zip(outs[i], want)):
            assert np.array_equal(got, wl), "%d -> %d item %d level %d: %d blocks differ" % (sf, T, i, l, L.differing_blocks(got, wl))
