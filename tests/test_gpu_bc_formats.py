"""GPU suite at the format boundary of Compress and Decompress: every source format into every BC1-BC5 target (the sRGB ones
included) with every sRGB flag; every specialised kernel pair k_compress_bc15_t<DF,SF> and the sRGB aliases the launcher maps
onto it, with padded and unaligned source rows; BC7_UNORM_SRGB and BC6H from sRGB sources, on the direct and the TMA-fed BC7
kernel; every BC source into every destination through the host API and through padded, unaligned device destinations; and mip
chains compressed to sRGB targets.  Results are compared bit for bit with the oracle (BC6H / BC7: with the host emulator, and
BC7_UNORM_SRGB also against the reference encoder's quality).  Where a compress runs powf, the sources come from
special_values.srgb_safe_image, on which glibc's and CUDA's powf agree, so that bit for bit stays meaningful; decompress keeps
the one-code rule where it converts between sRGB and linear (DESIGN.md section 3)."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F, synth
from tests import oracle_lib, special_values as S, tolerance
from tests.kernel_routes import launched

pytestmark = pytest.mark.gpu

PIXEL_FORMATS = sorted(F.BYTES_PER_PIXEL)
BC_FORMATS = sorted(F.BLOCK_BYTES)
BC15_TARGETS = (71, 72, 74, 75, 77, 78, 80, 81, 83, 84)
COMPRESS_FLAGS = (0, F.TEX_COMPRESS_SRGB_IN, F.TEX_COMPRESS_SRGB_OUT, F.TEX_COMPRESS_SRGB, F.TEX_COMPRESS_DITHER, F.TEX_COMPRESS_UNIFORM)
# 22 x 14: partial blocks and rows that are not 16-byte aligned (the scalar gather); 32 x 16: full blocks, aligned rows (the vector gather)
SIZES = ((22, 14), (32, 16))

# the (target, source) pairs dxb_launch_bc15 routes to k_compress_bc15_t (dxb_k_bc15.cu) and the (source, target) pairs
# dxb_launch_decompress routes to k_decompress_t (dxb_k_decode.cu); test_cpu_bc_formats checks them against the instantiations
# compiled into the library
BC15_PAIRS = [(71, 28), (71, 87), (71, 10), (71, 2), (74, 28), (74, 87), (74, 10), (74, 2), (77, 28), (77, 87), (77, 10), (77, 2),
              (80, 61), (80, 28), (80, 41), (80, 2), (81, 61), (81, 28), (81, 41), (81, 2),
              (83, 49), (83, 28), (83, 16), (83, 2), (84, 49), (84, 28), (84, 16), (84, 2)]
DEC_PAIRS = [(71, 28), (74, 28), (77, 28), (98, 28), (80, 61), (81, 63), (83, 49), (84, 51), (95, 2), (96, 2)]
DECOMPRESS_PAIRS = [(bc, df) for bc in BC_FORMATS for df in PIXEL_FORMATS]
SRGB_TWIN = {71: 72, 74: 75, 77: 78, 98: 99, 28: 29, 87: 91}
# each specialised pair with every sRGB variant of its two formats: the launcher maps 72 / 75 / 78 onto 71 / 74 / 77 and 29 / 91
# onto 28 / 87; where both sides are sRGB (or neither) the resolved flags are the default ones and the specialised kernel runs
BC15_ALIAS_CASES = sorted({(d, s) for (df, sf) in BC15_PAIRS for d in {df, SRGB_TWIN.get(df, df)} for s in {sf, SRGB_TWIN.get(sf, sf)}})
# decompress pairs whose sRGB sides cancel (no powf): exact, and 72 / 75 / 78 / 99 -> 29 take k_decompress_t after the remap
EXACT_SRGB_DECOMPRESS = [(bc, df) for bc in S.SRGB_BLOCK_FORMATS for df in S.SRGB_FORMATS]
UNORM_TWIN = {s: u for u, s in SRGB_TWIN.items()}
BC15_KERNELS = ("k_compress_bc15_t", "k_compress_bc15")
DEC_KERNELS = ("k_decompress_t", "k_decompress")


def bc15_kernel(sf, df, flags):
    """the kernel dxb_launch_bc15 takes: k_compress_bc15_t for a listed pair of UNORM twins without DITHER or UNIFORM whose
    resolved sRGB steps cancel (the default flag set), else k_compress_bc15"""
    hot = ((UNORM_TWIN.get(df, df), UNORM_TWIN.get(sf, sf)) in BC15_PAIRS and not flags & (F.TEX_COMPRESS_DITHER | F.TEX_COMPRESS_UNIFORM)
           and not S.resolve_srgb(flags, sf, df))
    return "k_compress_bc15_t" if hot else "k_compress_bc15"


def decompress_kernel(bc, df):
    """the kernel dxb_launch_decompress takes: k_decompress_t for a listed pair of UNORM twins without an sRGB step, else k_decompress"""
    hot = (UNORM_TWIN.get(bc, bc), UNORM_TWIN.get(df, df)) in DEC_PAIRS and not S.resolve_srgb(0, bc, df)
    return "k_decompress_t" if hot else "k_decompress"


@pytest.fixture(scope="module", autouse=True)
def _init():
    assert capi.lib.dxb200_init(0) == 0


def _rows(fmt, w, h):
    row, sl = F.compute_pitch(fmt, w, h)
    return row, sl // row


def _round16(n):
    return (n + 15) & ~15


def device_call(entry, mid, src, w, h, sf, df, spitch=0, soff=0, dpitch=0, doff=0):
    """entry(src image, 1, *mid, dst image, stream) on a device copy of `src` (tightly packed host bytes) with the given row
    pitches (0: tight) and base pointers `soff` / `doff` bytes past a fresh allocation; returns the tightly packed result"""
    torch = pytest.importorskip("torch")
    srow, sn = _rows(sf, w, h)
    drow, dn = _rows(df, w, h)
    spitch, dpitch = spitch or srow, dpitch or drow
    a = np.zeros(soff + sn * spitch, np.uint8)
    a[soff:].reshape(sn, spitch)[:, :srow] = np.ascontiguousarray(src).view(np.uint8).reshape(sn, srow)
    d_in = torch.from_numpy(a).cuda()
    d_out = torch.zeros(doff + dn * dpitch, dtype=torch.uint8, device="cuda")
    s = capi.images([capi.Image(w, h, sf, spitch, spitch * sn, d_in.data_ptr() + soff)])
    d = capi.images([capi.Image(w, h, df, dpitch, dpitch * dn, d_out.data_ptr() + doff)])
    hr = entry(s, 1, *mid, d, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert hr == 0, (hex(F.hr_u32(hr)), capi.last_error())
    torch.cuda.synchronize()
    return np.ascontiguousarray(d_out.cpu().numpy()[doff:].reshape(dn, dpitch)[:, :drow]).reshape(-1)


def compress_source(sf, df, flags, w, h, seed):
    """srgb_safe_image where the resolved flags run powf, the special-value sources (source_image) everywhere else"""
    d = S.powf_direction(flags, sf, df)
    return S.srgb_safe_image(sf, d, w, h, seed) if d else S.source_image(sf, w, h, seed)


def _fail_report(bad, total):
    assert not bad, "%d of %d cases differ; first: %s" % (len(bad), total, "; ".join(bad[:6]))


# ---- Compress: every source into every BC1-BC5 target -----------------------------------------------------------------------
@pytest.mark.parametrize("sf", PIXEL_FORMATS)
def test_compress_every_source_into_every_bc15_target(oracle, sf):
    """Each source format into BC1-BC5 and their sRGB variants with no flag, SRGB_IN, SRGB_OUT, both, DITHER and UNIFORM, at
    22 x 14 and 32 x 16, through the host API: bit for bit the oracle, on the kernel bc15_kernel names."""
    bad, total = [], 0
    for df in BC15_TARGETS:
        for fl in COMPRESS_FLAGS:
            for (w, h) in SIZES:
                src = compress_source(sf, df, fl, w, h, seed=w + df)
                hr, want = oracle.compress(src, w, h, sf, df, fl)
                assert hr == 0
                got, ran = launched(BC15_KERNELS, capi.compress, src, w, h, sf, df, fl)
                total += 1
                if S.mismatches(got, want, df).any() or ran != {bc15_kernel(sf, df, fl)}:
                    bad.append("%d -> %d flags %#x %dx%d on %s" % (sf, df, fl, w, h, sorted(ran)))
    _fail_report(bad, total)


@pytest.mark.parametrize("df,sf", BC15_ALIAS_CASES)
def test_bc15_kernel_pairs_and_srgb_aliases_on_device_layouts(oracle, df, sf):
    """Every k_compress_bc15_t pair and its sRGB aliases through the device API with the source row pitch tight, tight + 16 and
    tight + 4 and with the base pointer 4 bytes past an aligned one (the vector and the scalar paths of dxb_gather_block_t):
    bit for bit the oracle, on k_compress_bc15_t where the sRGB sides agree or cancel and on k_compress_bc15 where a powf step
    remains."""
    bad, total = [], 0
    for (w, h) in SIZES:
        src = compress_source(sf, df, 0, w, h, seed=3 * w + sf)
        hr, want = oracle.compress(src, w, h, sf, df)
        assert hr == 0
        row = w * F.BYTES_PER_PIXEL[sf]
        for spitch, soff in ((row, 0), (row + 16, 0), (row + 4, 0), (row, 4)):
            got, ran = launched(BC15_KERNELS, device_call, capi.lib.dxb200_compress_device, (df, 0, 0.5, 1.0), src, w, h, sf, df, spitch, soff)
            total += 1
            if S.mismatches(got, want, df).any() or ran != {bc15_kernel(sf, df, 0)}:
                bad.append("%d -> %d %dx%d pitch %d offset %d on %s" % (sf, df, w, h, spitch, soff, sorted(ran)))
    _fail_report(bad, total)


# ---- BC7_UNORM_SRGB and BC6H from sRGB sources -------------------------------------------------------------------------------
def _equal_blocks(got, em, ctx):
    nd = int((got.reshape(-1, 16) != em.reshape(-1, 16)).any(1).sum())
    assert nd == 0, "%s: %d of %d blocks differ from the emulator" % (ctx, nd, got.size // 16)


@pytest.mark.parametrize("sf", [2, 10, 28, 29, 91])
def test_bc7_srgb_target_equals_emulator(emul, sf):
    """BC7_UNORM_SRGB from RGBA32F / RGBA16F / RGBA8 (linear -> sRGB before the encoder) and from RGBA8_SRGB / BGRA8_SRGB (no
    conversion), with DEFAULT, QUICK and USE_3SUBSETS, on the direct kernel: device == emulator bit for bit."""
    for flags in (0, F.TEX_COMPRESS_BC7_QUICK, F.TEX_COMPRESS_BC7_USE_3SUBSETS):
        for (w, h) in ((22, 14), (64, 20)):
            src = compress_source(sf, 99, flags, w, h, seed=w + flags % 97)
            got = capi.compress(src, w, h, sf, 99, flags)
            he, em = emul.compress(src, w, h, sf, 99, flags)
            assert he == 0
            _equal_blocks(got, em, "BC7_SRGB from %d flags %#x %dx%d" % (sf, flags, w, h))


@pytest.mark.parametrize("bc", [95, 96])
def test_bc6h_from_srgb_source_equals_emulator(emul, bc):
    """R8G8B8A8_UNORM_SRGB into BC6H: sRGB -> linear before the encoder; device == emulator bit for bit."""
    for (w, h) in ((22, 14), (64, 20)):
        src = compress_source(29, bc, 0, w, h, seed=w)
        got = capi.compress(src, w, h, 29, bc)
        he, em = emul.compress(src, w, h, 29, bc)
        assert he == 0
        _equal_blocks(got, em, "BC6H %d from 29 %dx%d" % (bc, w, h))


def test_bc7_srgb_tma_fed_array_equals_emulator(emul):
    """An array of RGBA32F images made of full blocks, compressed to BC7_UNORM_SRGB, lies at a constant stride in the staging
    buffer and goes through k_compress_bc7_tma, which converts each pixel with the resolved sRGB flags: both instantiations
    (DEFAULT, USE_3SUBSETS) == emulator, and the TMA launch counter moves."""
    w, h, n = 72, 20, 3
    imgs = [S.srgb_safe_image(2, F.TEX_FILTER_SRGB_OUT, w, h, seed=40 + i) for i in range(n)]
    before, feed = capi.tma_launch_count(), capi.lib.dxb200_get_option(capi.OPT_BC7_FEED)
    assert capi.lib.dxb200_set_option(capi.OPT_BC7_FEED, 1) == 0
    try:
        for flags in (0, F.TEX_COMPRESS_BC7_USE_3SUBSETS):
            outs = capi.compress_array(imgs, w, h, 2, 99, flags)
            for i, (img, got) in enumerate(zip(imgs, outs)):
                he, em = emul.compress(img, w, h, 2, 99, flags)
                assert he == 0
                _equal_blocks(got, em, "TMA BC7_SRGB flags %#x image %d" % (flags, i))
    finally:
        capi.lib.dxb200_set_option(capi.OPT_BC7_FEED, feed)
    assert capi.tma_launch_count() >= before + 2


def srgb_stage(oracle, img):
    """what the reference BC7 encoder is given for a BC7_UNORM_SRGB target: the source converted linear -> sRGB by the
    reference's own Convert (alpha untouched), staged to 0..255 as its encoder stages LDR input (BC6HBC7.cpp:2794-2797)"""
    h, w = img.shape[:2]
    hr, rgb = oracle.convert(img, w, h, 2, 6, F.TEX_FILTER_SRGB_OUT)
    assert hr == 0
    rgba = np.concatenate([rgb.view(np.float32).reshape(h, w, 3), img[..., 3:]], -1)
    return oracle_lib.bc7_ldr(rgba).astype(np.float64)


def bc7_srgb_block_sse(oracle, blocks, stage):
    n = stage.shape[0]
    dec = oracle.decode_blocks(99, blocks, n, n).astype(np.float64) * 255.0
    return ((dec - stage) ** 2).reshape(n // 4, 4, n // 4, 4, 4).sum((1, 3, 4))


def check_bc7_srgb_contract(oracle, ours_blocks, ref_blocks, img, ctx):
    """the two inequalities of tests/tolerance.py, both streams measured against the reference's sRGB encoding of the source"""
    stage = srgb_stage(oracle, img)
    ours, theirs = bc7_srgb_block_sse(oracle, ours_blocks, stage), bc7_srgb_block_sse(oracle, ref_blocks, stage)
    ratio = ours.sum() / max(theirs.sum(), 1e-9)
    bad = float((ours > 2.0 * theirs + 16.0).mean())
    assert ours.sum() <= 1.02 * theirs.sum() + 1e-6, (ctx, ratio)
    assert bad < 0.01, (ctx, bad)
    return ratio


@pytest.mark.parametrize("kind", ["photo", "gradient", "alpha_photo"])
def test_bc7_srgb_contract_vs_reference(oracle, kind):
    """RGBA32F -> BC7_UNORM_SRGB at 256 x 256 on the device and on the reference encoder, live: the device stream is within
    the BC7 contract of the reference's against the sRGB encoding of the source.  Device == emulator cannot see an sRGB flag
    lost in code the two share; this can."""
    n = tolerance.SIZE
    img = synth.content_ldr(kind, n, n, tolerance.SEED)
    got = capi.compress(img, n, n, 2, 99)
    hr, ref = oracle.compress(img, n, n, 2, 99)
    assert hr == 0
    check_bc7_srgb_contract(oracle, got, ref, img, kind)


# ---- Decompress: every BC source into every destination ----------------------------------------------------------------------
def bc_streams(oracle, bc, w, h, seed):
    """random bytes (every mode, and the invalid ones, of the format) and a stream the reference encoder made"""
    rng = np.random.default_rng(seed)
    nb = ((w + 3) // 4) * ((h + 3) // 4)
    yield "random", rng.integers(0, 256, nb * F.BLOCK_BYTES[bc], dtype=np.uint8)
    src = rng.random((h, w, 4)).astype(np.float32) * (4.0 if bc in (95, 96) else 1.0) - (1.0 if bc in (81, 84, 96) else 0.0)
    hr, blocks = oracle.compress(src, w, h, 2, bc, 0)
    assert hr == 0
    yield "encoded", blocks


def decompress_matches(oracle, got, want, w, h, bc, df):
    """bit for bit, except the one-code rule where the resolved flags convert between sRGB and linear"""
    if S.powf_direction(0, bc, df):
        try:
            S.assert_within_one_code(oracle, got, want, w, h, df)
        except AssertionError:
            return False
        return True
    return not S.mismatches(got, want, df).any()


@pytest.mark.parametrize("bc", BC_FORMATS)
def test_decompress_every_bc_source_into_every_destination(oracle, bc):
    """Each BC format (72 / 75 / 78 / 99 included) into every destination at 13 x 9 and 32 x 16, random and encoded streams,
    through the host API and through the device API with the destination pitch padded to 16 bytes + 16 (the table-driven and
    the row-store paths of k_decompress_t) and with pitch + 4 at a base pointer 4 bytes off (the scalar stores); each call on
    the kernel decompress_kernel names."""
    bad, total = [], 0
    for (w, h) in ((13, 9), (32, 16)):
        for kind, blocks in bc_streams(oracle, bc, w, h, seed=bc * 31 + w):
            for df in PIXEL_FORMATS:
                hr, want = oracle.decompress(blocks, w, h, bc, df)
                assert hr == 0
                row = w * F.BYTES_PER_PIXEL[df]
                outs = (("host", launched(DEC_KERNELS, capi.decompress, blocks, w, h, bc, df)),
                        ("device pitch %d" % (_round16(row) + 16),
                         launched(DEC_KERNELS, device_call, capi.lib.dxb200_decompress_device, (df,), blocks, w, h, bc, df, dpitch=_round16(row) + 16)),
                        ("device pitch %d offset 4" % (row + 4),
                         launched(DEC_KERNELS, device_call, capi.lib.dxb200_decompress_device, (df,), blocks, w, h, bc, df, dpitch=row + 4, doff=4)))
                for path, (got, ran) in outs:
                    total += 1
                    if not decompress_matches(oracle, got, want, w, h, bc, df) or ran != {decompress_kernel(bc, df)}:
                        bad.append("%d -> %d %s %dx%d %s on %s" % (bc, df, kind, w, h, path, sorted(ran)))
    _fail_report(bad, total)


# ---- GenerateMipMaps + Compress to sRGB targets ------------------------------------------------------------------------------
@pytest.mark.parametrize("sf,df", [(29, 78), (28, 72)])
def test_mipmaps_compress_to_srgb_targets(oracle, sf, df):
    """dxb200_mipmaps_compress == dxb200_generate_mipmaps + dxb200_compress on the GPU, bit for bit.  The chain keeps its rule
    against the reference's (R8G8B8A8_UNORM_SRGB filters in linear light: one code).  29 -> 78 converts nothing, so its blocks
    also equal the oracle's compression of the GPU's own chain levels, bit for bit."""
    rng = np.random.default_rng(61 + df)
    for (w, h, n) in ((64, 64, 2), (96, 40, 2)):
        srcs = [oracle_lib.random_image(sf, w, h, rng) for _ in range(n)]
        outs = capi.mipmaps_compress(srcs, w, h, sf, df)
        for i, (src, got) in enumerate(zip(srcs, outs)):
            ctx = "%d -> %d %dx%d image %d" % (sf, df, w, h, i)
            chain, layout = capi.generate_mipmaps(src, w, h, sf, 0)
            hr, rchain = oracle.generate_mipmaps(src, w, h, sf, 0)
            assert hr == 0
            if sf == 29:
                S.assert_within_one_code(oracle, chain, rchain, 0, 0, sf, ctx)
            else:
                assert np.array_equal(chain, rchain), ctx
            levels = [chain[off:off + sl] for (off, lw, lh, row, sl) in layout]
            two = np.concatenate([capi.compress(lv, lw, lh, sf, df) for lv, (off, lw, lh, row, sl) in zip(levels, layout)])
            assert np.array_equal(got, two), ctx
            if not S.powf_direction(0, sf, df):
                want = np.concatenate([oracle.compress(lv, lw, lh, sf, df)[1] for lv, (off, lw, lh, row, sl) in zip(levels, layout)])
                assert np.array_equal(got, want), ctx
