"""GPU suite: dxb200_mipmaps_compress_ex, texconv's GenerateMipMaps -> ScaleMipMapsAlphaForCoverage -> PremultiplyAlpha -> Compress
with the chains kept in device memory, and the coverage search that runs on the device for a whole batch.

Every result equals the separate library calls (generate_mipmaps, scale_mipmaps_alpha_for_coverage per item, premultiply_alpha per
image, compress per image) bit for bit, and where the reference's own composed calls are bit-exact, those too."""
import ctypes as C
import re

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import oracle_lib, special_values as S, staging_cases as SC
from tests.test_cpu_capi import KERNELS

pytestmark = pytest.mark.gpu
L = capi.lib
BC67 = (94, 95, 96, 97, 98, 99)
FILTERS = (F.TEX_FILTER_POINT, F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, 0)
SOURCES = (28, 29, 87, 2, 10)
# (alpha reference, premultiply flags or None): coverage 0.5 / 0.25 / off x premultiply off / 0 / IGNORE_SRGB / REVERSE
COMBOS = [(ref, pm) for ref in (0.5, 0.25, 0.0) for pm in (None, 0, 0x1, 0x2)]


@pytest.fixture(autouse=True)
def one_device():
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0


def steps_of(ref, pm):
    return capi.chain_steps(ref, pm is not None, pm or 0)


def ex_call(srcs, w, h, sf, df, filter, steps, extras=None):
    """dxb200_mipmaps_compress_ex of equally sized host images, level 0 rows `extras[i]` bytes wider than tight; (hr, chains)"""
    levels = F.count_mips(w, h)
    extras = extras or [0] * len(srcs)
    row, _ = F.compute_pitch(sf, w, h)
    layout, total = capi.texture_layout(df, w, h, 1, levels)
    bases, outs = [], [np.zeros(total, np.uint8) for _ in srcs]
    for src, e in zip(srcs, extras):
        a = np.full((h, row + e), 0xA5, np.uint8)
        a[:, :row] = np.ascontiguousarray(src).view(np.uint8).reshape(h, row)
        bases.append(a)
    s = capi.images([capi.Image(w, h, sf, row + e, (row + e) * h, a.ctypes.data) for a, e in zip(bases, extras)])
    d = capi.images([capi.Image(lw, lh, df, r, sp, o.ctypes.data + off) for o in outs for (off, lw, lh, r, sp) in layout])
    hr = L.dxb200_mipmaps_compress_ex(s, len(srcs), levels, filter, C.byref(steps), df, 0, 0.5, 1.0, d)
    return F.hr_u32(hr), outs


def separate_chains(srcs, w, h, sf, filter, ref, pm):
    """the uncompressed chains after the separate calls: generate_mipmaps, scale_mipmaps_alpha_for_coverage per item,
    premultiply_alpha per image"""
    chains = capi.generate_mipmaps_images(srcs, w, h, sf, filter)
    layout, _ = F.mip_chain_layout(sf, w, h, 0)
    out = []
    for chain in chains:
        if ref > 0:
            chain = capi.scale_mipmaps_alpha_for_coverage(chain, w, h, sf, ref)
        if pm is not None:
            chain = np.concatenate([capi.premultiply_alpha(chain[off:off + sl], lw, lh, sf, pm) for (off, lw, lh, row, sl) in layout])
        out.append(chain)
    return out, layout


def compress_chain(chain, layout, sf, df):
    return np.concatenate([capi.compress(chain[off:off + sl], lw, lh, sf, df) for (off, lw, lh, row, sl) in layout])


def reference_blocks(oracle, src, w, h, sf, df, filter, ref, pm):
    """the reference's GenerateMipMaps [-> ScaleMipMapsAlphaForCoverage] [-> PremultiplyAlpha] -> Compress of one item"""
    if ref > 0:
        hr, _, chain = oracle.mips_alpha_coverage(src, w, h, sf, ref, filter)
    else:
        hr, chain = oracle.generate_mipmaps(src, w, h, sf, filter)
    assert hr == 0
    layout, _ = F.mip_chain_layout(sf, w, h, 0)
    if pm is not None:
        chain = np.concatenate([oracle.premultiply_alpha(chain[off:off + sl], lw, lh, sf, pm)[1] for (off, lw, lh, row, sl) in layout])
    return np.concatenate([oracle.compress(chain[off:off + sl], lw, lh, sf, df)[1] for (off, lw, lh, row, sl) in layout])


def alpha_image(sf, w, h, rng):
    """random colour, alpha with edges around 0.25 and 0.5 so that every coverage step has work"""
    img = oracle_lib.random_image(sf, w, h, rng)
    yy, xx = np.mgrid[0:h, 0:w]
    a = np.clip(0.4 + 0.4 * np.sin(xx * 0.5) * np.cos(yy * 0.35) + rng.normal(0, 0.1, (h, w)), 0, 1)
    if sf in (28, 29, 87):
        img = img.reshape(h, w, 4)
        img[..., 3] = (a * 255).astype(np.uint8)
    else:
        dt = np.float16 if sf == 10 else np.float32
        img = img.view(dt).reshape(h, w, 4)
        img[..., 3] = a.astype(dt)
    return np.ascontiguousarray(img)


def test_ex_equals_separate_calls_every_target_source_filter(oracle):
    """Every BC target x sources 28 / 29 / 87 / 2 / 10 x filters POINT / BOX / LINEAR / CUBIC / TRIANGLE / 0, two items at 64 x 16
    and 40 x 24, each call with one of coverage 0.5 / 0.25 / off x premultiply off / 0 / IGNORE_SRGB / REVERSE (every pair on every
    source): bit for bit the separate calls, and for BC1-BC5 without a powf step the reference's composed calls."""
    bad, total, k = [], 0, 0
    for sf in SOURCES:
        rng = np.random.default_rng(sf)
        for (w, h) in ((64, 16), (40, 24)):
            srcs = [alpha_image(sf, w, h, rng) for _ in range(2)]
            for fl in FILTERS:
                ref, pm = COMBOS[k % len(COMBOS)]
                k += 1
                ctx = "%d %dx%d filter %#x coverage %g pm %s" % (sf, w, h, fl, ref, pm)
                if fl == F.TEX_FILTER_BOX and (w, h) == (40, 24):
                    hr, _ = ex_call(srcs, w, h, sf, 71, fl, steps_of(ref, pm))
                    assert hr == F.E_FAIL, (ctx, hex(hr))           # BOX needs power-of-two sizes (GenerateMipMaps)
                    continue
                chains, layout = separate_chains(srcs, w, h, sf, fl, ref, pm)
                for df in sorted(F.BLOCK_BYTES):
                    hr, outs = ex_call(srcs, w, h, sf, df, fl, steps_of(ref, pm))
                    assert hr == 0, (ctx, df, hex(hr), capi.last_error())
                    for i, (src, chain, got) in enumerate(zip(srcs, chains, outs)):
                        total += 1
                        if not np.array_equal(got, compress_chain(chain, layout, sf, df)):
                            bad.append("%s -> %d item %d != separate calls" % (ctx, df, i))
                            continue
                        # the reference: BC1-BC5 from the linear sources without a powf step in Compress (an sRGB source has one in
                        # its mips and its premultiply, where the contract is one code)
                        if df in BC67 or sf == 29 or S.powf_direction(0, sf, df):
                            continue
                        if not np.array_equal(got, reference_blocks(oracle, src, w, h, sf, df, fl, ref, pm)):
                            bad.append("%s -> %d item %d != reference" % (ctx, df, i))
    assert k == len(SOURCES) * 12
    assert not bad, "%d of %d differ; first: %s" % (len(bad), total, "; ".join(bad[:6]))


@pytest.mark.parametrize("sf,df,w,h,items,fl,extras,nchunks", [
    (28, 77, 1024, 1024, 12, 0, (0, 64, 4), 2),                     # eleven chains per chunk, then one
    (2, 98, 2048, 2048, 2, F.TEX_FILTER_CUBIC, (64, 16), 2),        # each chain larger than a chunk
    (10, 95, 512, 128, 3, F.TEX_FILTER_BOX, (8, 0, 136), 1)])       # a non-square chain down to height 1
def test_ex_arrays_over_chunks_with_wide_level0(sf, df, w, h, items, fl, extras, nchunks):
    """Coverage 0.5 and premultiply on arrays of chains over several 80 MiB chunks, single chains larger than a chunk and a
    single-chunk array, level 0 at row pitches wider than tight: every item equals the separate calls."""
    levels = F.count_mips(w, h)
    ex = [extras[i % len(extras)] for i in range(items)]
    chunks, _ = SC.chain_chunks(sf, df, w, h, items, levels, max(ex))
    assert len(chunks) == nchunks, chunks
    rng = np.random.default_rng(w + items)
    srcs = [alpha_image(sf, w, h, rng) for _ in range(items)]
    hr, outs = ex_call(srcs, w, h, sf, df, fl, steps_of(0.5, 0), ex)
    assert hr == 0, (hex(hr), capi.last_error())
    for i, (src, got) in enumerate(zip(srcs, outs)):
        (chain,), layout = separate_chains([src], w, h, sf, fl, 0.5, 0)
        assert np.array_equal(got, compress_chain(chain, layout, sf, df)), (sf, df, w, h, i)


def launches(fn, *args):
    before = {k: capi.kernel_launch_count(k) for k in KERNELS}
    out = fn(*args)
    return out, {k: capi.kernel_launch_count(k) - before[k] for k in KERNELS if capi.kernel_launch_count(k) != before[k]}


def family(kernel):
    return "k_mip" if kernel.startswith("k_mip") else re.sub(r"_(t|vec|tma)$", "", kernel)


@pytest.mark.parametrize("w,h,items", [(2048, 2048, 1), (1024, 1024, 12)])
def test_ex_routes(w, h, items):
    """Each chunk of an _ex call runs the coverage search of all its chains as exactly 10 k_alpha_coverage launches and one
    k_scale_alpha (a 12-level chain; twelve 11-level chains in two chunks); the per-item call runs 10 + 1 whatever its level count;
    the mip, premultiply and compress kernel families are the ones the separate calls take."""
    levels = F.count_mips(w, h)
    chunks, _ = SC.chain_chunks(28, 77, w, h, items, levels)
    rng = np.random.default_rng(items)
    srcs = [alpha_image(28, w, h, rng) for _ in range(items)]
    (hr, outs), ran = launches(ex_call, srcs, w, h, 28, 77, 0, steps_of(0.5, 0))
    assert hr == 0
    assert ran["k_alpha_coverage"] == 10 * len(chunks) and ran["k_scale_alpha"] == len(chunks), (ran, chunks)
    chains, layout = separate_chains(srcs[:1], w, h, 28, 0, 0.0, None)
    got, ran1 = launches(capi.scale_mipmaps_alpha_for_coverage, chains[0], w, h, 28, 0.5)
    assert ran1 == {"k_alpha_coverage": 10, "k_scale_alpha": 1}, ran1
    sep = set()
    for fn, args in ((capi.generate_mipmaps_images, (srcs, w, h, 28, 0)),):
        sep |= set(launches(fn, *args)[1])
    for (off, lw, lh, row, sl) in layout:
        sep |= set(launches(capi.premultiply_alpha, got[off:off + sl], lw, lh, 28, 0)[1])
        sep |= set(launches(capi.compress, got[off:off + sl], lw, lh, 28, 77)[1])
    fused = {family(k) for k in ran} - {"k_alpha_coverage", "k_scale_alpha"}
    assert fused == {family(k) for k in sep}, (sorted(ran), sorted(sep))


def test_ex_sharded_equals_one_device():
    """With every GPU initialised, _ex shards items over the devices and equals one device's result."""
    n = L.dxb200_device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    rng = np.random.default_rng(9)
    srcs = [alpha_image(28, 256, 256, rng) for _ in range(4 * n)]
    hr, one = ex_call(srcs, 256, 256, 28, 77, 0, steps_of(0.5, 0))
    assert hr == 0
    capi.init_devices(list(range(n)))
    try:
        hr, many = ex_call(srcs, 256, 256, 28, 77, 0, steps_of(0.5, 0))
    finally:
        L.dxb200_shutdown()
        assert L.dxb200_init(0) == 0
    assert hr == 0
    for a, b in zip(one, many):
        assert np.array_equal(a, b)


def test_float_alpha_corpus_through_both_entries(oracle):
    """Alpha of +Inf, -0, denormals, 0, 1 and the reference value +-1 ulp in RGBA32F and RGBA16F: the per-item entry equals the
    reference's ScaleMipMapsAlphaForCoverage and _ex (coverage only, BC3) equals the reference's composed calls."""
    rng = np.random.default_rng(71)
    for fmt, (w, h) in ((2, (48, 20)), (2, (32, 32)), (10, (40, 24))):
        dt = np.float16 if fmt == 10 else np.float32
        for ref in (0.5, 0.25):
            r = dt(ref)
            tiny = np.finfo(dt).smallest_subnormal
            alphas = np.array([0, 1, np.inf, -0.0, tiny, 4 * tiny, r, np.nextafter(r, dt(0)), np.nextafter(r, dt(1))], dt)
            img = S.edge_image(w, h, seed=w)
            with np.errstate(over="ignore"):
                img = img.astype(dt)
            img[..., 3] = alphas[rng.integers(0, len(alphas), (h, w))]
            img = np.ascontiguousarray(img)
            hr, plain, want = oracle.mips_alpha_coverage(img, w, h, fmt, ref)
            assert hr == 0
            got = capi.scale_mipmaps_alpha_for_coverage(plain, w, h, fmt, ref)
            S.assert_same(got, want, fmt, "per-item coverage fmt %d %dx%d ref %g" % (fmt, w, h, ref))
            hr, (blocks,) = ex_call([img], w, h, fmt, 77, 0, steps_of(ref, None))
            assert hr == 0
            assert np.array_equal(blocks, reference_blocks(oracle, img, w, h, fmt, 77, 0, ref, None)), (fmt, w, h, ref)
