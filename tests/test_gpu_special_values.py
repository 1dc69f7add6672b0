"""GPU suite on the special-value corpus (tests/special_values.py): the CUDA kernels against the oracle (or, for BC6H / BC7,
against the host lock-step emulator) at the values where kernels go wrong -- +-0, denormals, the half overflow points,
+-Inf next to -Inf, FLT_MAX, the rounding ties of every store -- and at the widths, pitches and batch shapes that select
each kernel variant.  Outputs are compared bit for bit except that any NaN matches any NaN in a float destination
(special_values.mismatches); sRGB paths keep the +-1 code rule."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import special_values as S
from tests.kernel_routes import launched

pytestmark = pytest.mark.gpu

PIXEL_FORMATS = sorted(F.BYTES_PER_PIXEL)
CORPUS_SOURCES = S.F32_FORMATS + S.F16_FORMATS + S.PACKED16 + (26, 67)
CONVERT_FLAGS = (0, F.TEX_FILTER_FLOAT_X2BIAS, F.TEX_FILTER_RGB_COPY_RED, F.TEX_FILTER_RGB_COPY_GREEN, F.TEX_FILTER_RGB_COPY_BLUE,
                 F.TEX_FILTER_DITHER, F.TEX_FILTER_DITHER_DIFFUSION, F.TEX_FILTER_SRGB_IN, F.TEX_FILTER_SRGB_OUT, F.TEX_FILTER_SRGB)
# the (source, destination) pairs dxb_launch_convert routes to k_convert_vec and the formats dxb_launch_pmalpha routes to
# k_pmalpha_vec (dxb_k_rows.cu); test_cpu_special_values checks them against the instantiations compiled into the library
VEC_PAIRS = [(61, 41), (41, 61), (28, 2), (2, 28), (10, 2), (2, 10), (28, 10), (10, 28), (28, 87), (87, 28),
             (61, 28), (28, 61), (11, 2), (2, 11), (41, 2), (2, 41), (29, 2), (2, 29), (29, 28), (28, 29)]
PMALPHA_VEC_FORMATS = (28, 29, 87, 91, 10, 2)
CONVERT_KERNELS = ("k_convert_vec", "k_convert", "k_convert_diffuse")
PMALPHA_KERNELS = ("k_pmalpha_vec", "k_pmalpha")


@pytest.fixture(scope="module", autouse=True)
def _init():
    assert capi.lib.dxb200_init(0) == 0


# ---- device-pointer calls with chosen row pitches ------------------------------------------------------------------------
def _rows(fmt, w, h):
    row, sl = F.compute_pitch(fmt, w, h)
    return row, sl // row


def _upload(torch, buf, fmt, w, h, pitch):
    row, n = _rows(fmt, w, h)
    a = np.zeros((n, pitch), np.uint8)
    a[:, :row] = np.ascontiguousarray(buf).view(np.uint8).reshape(n, row)
    return torch.from_numpy(a.reshape(-1)).cuda()


def device_call(entry, mid, srcs, sizes, sf, df, spitches=None, dpitches=None):
    """entry(src images, n, *mid, dst images, stream) on device copies of `srcs` (tightly packed host buffers) with the given
    row pitches (default: tight); returns the tightly packed results"""
    torch = pytest.importorskip("torch")
    spitches = spitches or [_rows(sf, w, h)[0] for (w, h) in sizes]
    dpitches = dpitches or [_rows(df, w, h)[0] for (w, h) in sizes]
    d_in = [_upload(torch, b, sf, w, h, p) for b, (w, h), p in zip(srcs, sizes, spitches)]
    d_out = [torch.zeros(p * _rows(df, w, h)[1], dtype=torch.uint8, device="cuda") for (w, h), p in zip(sizes, dpitches)]
    s = capi.images([capi.Image(w, h, sf, p, p * _rows(sf, w, h)[1], t.data_ptr()) for t, (w, h), p in zip(d_in, sizes, spitches)])
    d = capi.images([capi.Image(w, h, df, p, p * _rows(df, w, h)[1], t.data_ptr()) for t, (w, h), p in zip(d_out, sizes, dpitches)])
    hr = entry(s, len(srcs), *mid, d, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert hr == 0, (hex(F.hr_u32(hr)), capi.last_error())
    torch.cuda.synchronize()
    out = []
    for t, (w, h), p in zip(d_out, sizes, dpitches):
        row, n = _rows(df, w, h)
        out.append(np.ascontiguousarray(t.cpu().numpy().reshape(n, p)[:, :row]).reshape(-1))
    return out


def convert_device(src, w, h, sf, df, flags=0, spitch=None, dpitch=None):
    return device_call(capi.lib.dxb200_convert_device, (df, flags, 0.5), [src], [(w, h)], sf, df,
                       spitches=[spitch] if spitch else None, dpitches=[dpitch] if dpitch else None)[0]


def check(oracle, got, want, w, h, sf, df, flags, ctx):
    if S.involves_srgb(sf, df, flags):
        S.assert_within_one_code(oracle, got, want, w, h, df, ctx)
    else:
        S.assert_same(got, want, df, ctx)


def _ppt(sf, df):
    return 16 // max(F.BYTES_PER_PIXEL[sf], F.BYTES_PER_PIXEL[df])


def _round16(n):
    return (n + 15) & ~15


# ---- Convert ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf", PIXEL_FORMATS)
def test_convert_every_pair_widths(oracle, sf):
    """Every (src, dst) pair at widths 1, PPT-1, PPT, PPT+1, 257 and 1031 (PPT = pixels per 16-byte vector of the wider side),
    3 rows, through the device API with both row pitches rounded up to 16 bytes.  Per convert_vec_ok that takes k_convert_vec
    for the VEC_PAIRS pairs -- its vector body, its ragged end (widths that are not a multiple of PPT) and, at 1031 pixels of
    16 bytes, two CTAs per row -- and k_convert for every other pair."""
    for df in PIXEL_FORMATS:
        if df == sf:
            continue
        ppt = _ppt(sf, df)
        for w in sorted({1, ppt - 1, ppt, ppt + 1, 257, 1031} - {0}):
            h = 3
            src = S.source_image(sf, w, h, seed=w)
            hr, want = oracle.convert(src, w, h, sf, df)
            assert hr == 0
            got, ran = launched(CONVERT_KERNELS, convert_device, src, w, h, sf, df, 0, _round16(w * F.BYTES_PER_PIXEL[sf]),
                                _round16(w * F.BYTES_PER_PIXEL[df]))
            check(oracle, got, want, w, h, sf, df, 0, "convert %d -> %d width %d" % (sf, df, w))
            assert ran == {"k_convert_vec" if (sf, df) in VEC_PAIRS else "k_convert"}, (sf, df, w, ran)


@pytest.mark.parametrize("sf,df", VEC_PAIRS)
def test_convert_vec_pairs_vector_and_generic_kernel(oracle, sf, df):
    """Each k_convert_vec pair twice through the device API: pitches rounded up to 16 bytes (convert_vec_ok holds:
    k_convert_vec) and both pitches padded by 4 more bytes (the wider side moves 16-byte vectors, so the padded pitch fails
    convert_vec_ok: the generic k_convert).  Widths give several CTAs per row for every PPT; both results equal the oracle."""
    ppt = _ppt(sf, df)
    sb, db = F.BYTES_PER_PIXEL[sf], F.BYTES_PER_PIXEL[df]
    for w in (ppt + 1, 257, 1024 * ppt + ppt + 1):
        h = 5
        src = S.source_image(sf, w, h, seed=7 * w)
        hr, want = oracle.convert(src, w, h, sf, df)
        assert hr == 0
        for pad in (0, 4):
            got, ran = launched(CONVERT_KERNELS, convert_device, src, w, h, sf, df, 0, _round16(w * sb) + pad, _round16(w * db) + pad)
            check(oracle, got, want, w, h, sf, df, 0, "convert %d -> %d width %d pad %d" % (sf, df, w, pad))
            assert ran == {"k_convert_vec" if pad == 0 else "k_convert"}, (sf, df, w, pad, ran)


def _corpus_source(fmt):
    if fmt in S.F32_FORMATS:
        return S.f32_image(fmt, 64, 20).view(np.uint8).reshape(-1), 64, 20
    if fmt in S.F16_FORMATS:
        img, h = S.half_image(fmt, 256)
        return img.view(np.uint8).reshape(-1), 256, h
    return S.source_image(fmt, 256, 256), 256, 256


@pytest.mark.parametrize("sf", CORPUS_SOURCES)
def test_convert_flags_special_values(oracle, sf):
    """The fp32 corpus (R32G32B32A32 / R32G32B32 / R32G32 / R32), every half pattern and the packed-source patterns to every
    destination with each flag family, through the host API.  Refused pairs (dithered stores to 85 / 86 / 115) must be
    refused.  DITHER_DIFFUSION runs k_convert_diffuse, every other flag one of the other two convert kernels.  sRGB with error
    diffusion is left to the CPU suite: diffusion carries powf's last-place difference between glibc and CUDA into later
    pixels, beyond the one-code rule."""
    src, w, h = _corpus_source(sf)
    for df in PIXEL_FORMATS:
        if df == sf:
            continue
        for fl in CONVERT_FLAGS:
            if S.convert_refused(df, fl):
                with pytest.raises(capi.DxTexError) as e:
                    capi.convert(src, w, h, sf, df, fl)
                assert e.value.hr == F.HRESULT_E_NOT_SUPPORTED
                continue
            if S.involves_srgb(sf, df, fl) and fl & F.TEX_FILTER_DITHER_DIFFUSION:
                continue
            hr, want = oracle.convert(src, w, h, sf, df, fl)
            assert hr == 0
            got, ran = launched(CONVERT_KERNELS, capi.convert, src, w, h, sf, df, fl)
            check(oracle, got, want, w, h, sf, df, fl, "convert %d -> %d flags %#x" % (sf, df, fl))
            diffuse = bool(fl & F.TEX_FILTER_DITHER_DIFFUSION)
            assert ran and ("k_convert_diffuse" in ran) == diffuse and (not diffuse or len(ran) == 1), (sf, df, hex(fl), ran)


# ---- mips, resize, premultiplied alpha, alpha coverage ---------------------------------------------------------------------
def _float_source(fmt, w, h, seed):
    if fmt in (2, 41):
        return S.f32_image(fmt, w, h, seed).view(np.uint8).reshape(-1)
    if fmt == 10:
        with np.errstate(over="ignore"):                        # beyond 65504 -> half Inf: part of the corpus
            return S.edge_image(w, h, seed).astype(np.float16).view(np.uint8).reshape(-1)
    return S.source_image(fmt, w, h, seed)


@pytest.mark.parametrize("fmt", [2, 10, 28, 41, 61, 29])
def test_mips_kernel_families_special_values(oracle, fmt):
    """Corpus chains through every mip kernel family: 128 x 64 BOX / LINEAR (fused k_mip_box3 for the top levels, then
    k_mip_tail), 100 x 60 LINEAR (k_mip_tile) and CUBIC (k_mip_sep), 37 x 19 odd sizes, TRIANGLE / POINT / WRAP / MIRROR (the
    generic k_mip_level).  R8G8B8A8_UNORM_SRGB goes through powf: +-1 code."""
    filters = (F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, F.TEX_FILTER_POINT, 0,
               F.TEX_FILTER_LINEAR | F.TEX_FILTER_WRAP, F.TEX_FILTER_CUBIC | F.TEX_FILTER_MIRROR, F.TEX_FILTER_TRIANGLE | F.TEX_FILTER_WRAP)
    for (w, h) in ((128, 64), (100, 60), (37, 19)):
        src = _float_source(fmt, w, h, seed=w)
        for fl in filters:
            if (fl & 0xF00000) == F.TEX_FILTER_BOX and (w & (w - 1) or h & (h - 1)):
                continue
            hr, want = oracle.generate_mipmaps(src, w, h, fmt, fl)
            got, _ = capi.generate_mipmaps(src, w, h, fmt, fl)
            assert hr == 0
            ctx = "mips fmt %d %dx%d filter %#x" % (fmt, w, h, fl)
            if fmt == 29:
                S.assert_within_one_code(oracle, got, want, 0, 0, fmt, ctx)
            else:
                S.assert_same(got, want, fmt, ctx)


@pytest.mark.parametrize("fmt", [2, 10, 41])
def test_resize_special_values(oracle, fmt):
    cases = ((64, 20, 32, 10), (37, 19, 50, 7), (64, 20, 128, 41))
    filters = (F.TEX_FILTER_POINT, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, F.TEX_FILTER_BOX, 0,
               F.TEX_FILTER_LINEAR | F.TEX_FILTER_WRAP, F.TEX_FILTER_CUBIC | F.TEX_FILTER_MIRROR)
    for (w, h, nw, nh) in cases:
        src = _float_source(fmt, w, h, seed=nw)
        for fl in filters:
            if (fl & 0xF00000) == F.TEX_FILTER_BOX and (nw * 2 != w or nh * 2 != h):
                continue
            hr, want = oracle.resize(src, w, h, fmt, nw, nh, fl)
            assert hr == 0
            S.assert_same(capi.resize(src, w, h, fmt, nw, nh, fl), want, fmt, "resize fmt %d %dx%d -> %dx%d filter %#x" % (fmt, w, h, nw, nh, fl))


@pytest.mark.parametrize("flags", [0, 2])
def test_premultiply_alpha_special_values(oracle, flags):
    """Inf x alpha 0, Inf x Inf, division by denormal alphas and by alpha near 0 (reverse), on the vector kernel (aligned
    rows) and the generic one (odd widths)"""
    for fmt in (2, 10):
        for (w, h) in ((64, 20), (37, 19)):
            src = _float_source(fmt, w, h, seed=w + flags)
            hr, want = oracle.premultiply_alpha(src, w, h, fmt, flags)
            assert hr == 0
            S.assert_same(capi.premultiply_alpha(src, w, h, fmt, flags), want, fmt, "pmalpha fmt %d %dx%d flags %d" % (fmt, w, h, flags))


# (format, TEX_PMALPHA flags, resolved sRGB steps): both directions (0x2 = REVERSE); sRGB steps both (29 / 91, or
# TEX_PMALPHA_SRGB = 0x3000000), none (no flag, or IGNORE_SRGB = 0x1) or one (0x1000000 / 0x2000000: k_pmalpha only)
PMALPHA_ROUTES = [(28, 0, 0), (28, 2, 0), (28, 0x3000000, 3), (28, 0x3000002, 3), (28, 0x1000000, 1), (28, 0x2000002, 2),
                  (29, 0, 3), (29, 2, 3), (29, 1, 0), (29, 3, 0), (87, 0x3000002, 3), (91, 0, 3), (91, 3, 0),
                  (10, 0, 0), (10, 2, 0), (2, 0, 0), (2, 2, 0)]


@pytest.mark.parametrize("fmt,flags,srgb", PMALPHA_ROUTES)
def test_premultiply_alpha_vector_and_generic_kernel(oracle, fmt, flags, srgb):
    """257 x 3 through the device API with both row pitches rounded up to 16 bytes (k_pmalpha_vec when the resolved sRGB steps
    are both or none, k_pmalpha for one) and padded by 4 more bytes (k_pmalpha): the oracle bit for bit, or within one code
    where an sRGB step runs powf."""
    w, h = 257, 3
    pitch = _round16(w * F.BYTES_PER_PIXEL[fmt])
    src = _float_source(fmt, w, h, seed=fmt + flags)
    hr, want = oracle.premultiply_alpha(src, w, h, fmt, flags)
    assert hr == 0
    for pad in (0, 4):
        (got,), ran = launched(PMALPHA_KERNELS, device_call, capi.lib.dxb200_premultiply_alpha_device, (flags,), [src], [(w, h)], fmt, fmt,
                               [pitch + pad], [pitch + pad])
        ctx = "pmalpha fmt %d flags %#x pad %d" % (fmt, flags, pad)
        if srgb:
            assert np.abs(got.astype(np.int32) - want.astype(np.int32)).max() <= 1, ctx
        else:
            S.assert_same(got, want, fmt, ctx)
        assert ran == {"k_pmalpha_vec" if pad == 0 and srgb in (0, 3) else "k_pmalpha"}, (ctx, ran)


def test_scale_mipmaps_alpha_for_coverage_threshold_values(oracle):
    """alpha made of 0, 1 and the reference value +-1 ulp (in the format's own precision); RGB from the corpus"""
    rng = np.random.default_rng(53)
    for fmt, (w, h) in ((2, (48, 20)), (2, (32, 32)), (10, (40, 24))):
        for ref in (0.5, 0.25):
            dt = np.float16 if fmt == 10 else np.float32
            r = dt(ref)
            alphas = np.array([0, 1, r, np.nextafter(r, dt(0)), np.nextafter(r, dt(1))], dt)
            img = S.edge_image(w, h, seed=w)
            with np.errstate(over="ignore"):
                img = img.astype(dt)
            img[..., 3] = alphas[rng.integers(0, len(alphas), (h, w))]
            hr, plain, want = oracle.mips_alpha_coverage(img, w, h, fmt, ref)
            assert hr == 0
            got = capi.scale_mipmaps_alpha_for_coverage(plain, w, h, fmt, ref)
            S.assert_same(got, want, fmt, "alpha coverage fmt %d %dx%d ref %g" % (fmt, w, h, ref))


# ---- block compression -----------------------------------------------------------------------------------------------------
def _bc_sources():
    out = [(S.f32_image(sf, 64, 20, seed=sf).view(np.uint8).reshape(-1), 64, 20, sf) for sf in S.F32_FORMATS]
    img, h = S.half_image(10, 256)
    out.append((img.view(np.uint8).reshape(-1), 256, h, 10))
    return out


@pytest.mark.parametrize("bc", [71, 74, 77, 80, 81, 83, 84])
def test_bc15_special_values(oracle, bc):
    for src, w, h, sf in _bc_sources():
        for flags in (0, F.TEX_COMPRESS_UNIFORM, F.TEX_COMPRESS_DITHER):
            hr, want = oracle.compress(src, w, h, sf, bc, flags)
            assert hr == 0
            S.assert_same(capi.compress(src, w, h, sf, bc, flags), want, bc, "BC %d from %d flags %#x" % (bc, sf, flags))


@pytest.mark.parametrize("bc,flags", [(95, 0), (96, 0), (98, 0), (98, F.TEX_COMPRESS_BC7_QUICK), (98, F.TEX_COMPRESS_BC7_USE_3SUBSETS)])
def test_bc6h_bc7_special_values_equal_emulator(oracle, emul, bc, flags):
    """Device == host emulator bit for bit on the fp32 corpus, the corpus x 1000 and every half pattern (negative values into
    UF16, beyond 65504, +-Inf, denormals); every pixel whose input is finite decodes (reference decoder) to finite values."""
    base = S.edge_image(64, 20, seed=bc + flags)
    with np.errstate(over="ignore"):
        big = (base * np.float32(1000.0)).astype(np.float32)
    himg, hh = S.half_image(10, 256)
    for src, w, h, sf, f32 in ((base, 64, 20, 2, base), (big, 64, 20, 2, big), (himg, 256, hh, 10, himg.view(np.float16).astype(np.float32))):
        got = capi.compress(src, w, h, sf, bc, flags)
        he, em = emul.compress(src, w, h, sf, bc, flags)
        assert he == 0
        nd = int((got.reshape(-1, 16) != em.reshape(-1, 16)).any(1).sum())
        assert nd == 0, "BC %d flags %#x from %d (%dx%d): %d of %d blocks differ from the emulator" % (bc, flags, sf, w, h, nd, got.size // 16)
        dec = oracle.decode_blocks(bc, got, w, h)
        assert np.isfinite(dec[np.isfinite(f32.reshape(h, w, 4)).all(-1)]).all(), (bc, flags, sf)


# ---- mixed-size batches ----------------------------------------------------------------------------------------------------
MIXED = [(1, 1), (2, 3), (4, 4), (5, 7), (64, 4), (257, 3), (128, 128)]


def _mixed_sources(fmt=2):
    out = []
    for i, (w, h) in enumerate(MIXED):
        img = S.edge_image(w, h, seed=100 + i)
        if fmt == 10:
            with np.errstate(over="ignore"):
                img = img.astype(np.float16)
        out.append(np.ascontiguousarray(img).view(np.uint8).reshape(-1))
    return out


def _both_paths(host_fn, entry, mid, srcs, sf, df):
    """the host-pointer array entry and the device-pointer entry on the same mixed batch"""
    return [("host", host_fn()), ("device", device_call(entry, mid, srcs, MIXED, sf, df))]


@pytest.mark.parametrize("bc", [71, 74, 77, 80, 81, 83, 84, 95, 96, 98])
def test_mixed_size_batch_compress(oracle, emul, bc):
    """One call over 1x1, 2x3, 4x4, 5x7, 64x4, 257x3 and 128x128 images (every unit finds its image by dxb_find_job): the
    first images hold one block each, so BC6H / BC7 block pairs straddle two images of different widths.  BC1-BC5 equal the
    oracle, BC6H / BC7 the emulator, and every image equals its single-image result."""
    srcs = _mixed_sources()
    for path, outs in _both_paths(lambda: capi.compress_images(srcs, MIXED, 2, bc), capi.lib.dxb200_compress_device, (bc, 0, 0.5, 1.0), srcs, 2, bc):
        for i, ((w, h), s_, o) in enumerate(zip(MIXED, srcs, outs)):
            if bc in (95, 96, 98):
                he, want = emul.compress(s_, w, h, 2, bc)
                assert he == 0
            else:
                hr, want = oracle.compress(s_, w, h, 2, bc)
                assert hr == 0
            S.assert_same(o, want, bc, "%s batch BC %d image %d (%dx%d)" % (path, bc, i, w, h))
            assert np.array_equal(o, capi.compress(s_, w, h, 2, bc)), (path, bc, i)


@pytest.mark.parametrize("sf,df,fl", [(2, 28, 0), (2, 10, 0), (10, 2, 0), (2, 41, 0), (2, 31, F.TEX_FILTER_DITHER), (2, 28, F.TEX_FILTER_DITHER_DIFFUSION)])
def test_mixed_size_batch_convert(oracle, sf, df, fl):
    """A batch of different sizes fails convert_vec_ok (equal sizes required), so the generic k_convert (or the per-image
    diffusion kernel) runs with a job table; every image equals the oracle and its single-image result."""
    srcs = _mixed_sources(sf)
    host = lambda: capi.convert_images(srcs, MIXED, sf, df, fl)
    for path, outs in _both_paths(host, capi.lib.dxb200_convert_device, (df, fl, 0.5), srcs, sf, df):
        for i, ((w, h), s_, o) in enumerate(zip(MIXED, srcs, outs)):
            hr, want = oracle.convert(s_, w, h, sf, df, fl)
            assert hr == 0
            S.assert_same(o, want, df, "%s batch convert %d -> %d flags %#x image %d (%dx%d)" % (path, sf, df, fl, i, w, h))
            assert np.array_equal(o, capi.convert(s_, w, h, sf, df, fl)), (path, i)


@pytest.mark.parametrize("bc,df", [(71, 28), (77, 2), (80, 41), (84, 2), (95, 10), (96, 2), (98, 28)])
def test_mixed_size_batch_decompress(oracle, bc, df):
    srcs = _mixed_sources()
    blocks = []
    for (w, h), s_ in zip(MIXED, srcs):
        hr, b = oracle.compress(s_, w, h, 2, bc)
        assert hr == 0
        blocks.append(b)
    for path, outs in _both_paths(lambda: capi.decompress_images(blocks, MIXED, bc, df), capi.lib.dxb200_decompress_device, (df,), blocks, bc, df):
        for i, ((w, h), b, o) in enumerate(zip(MIXED, blocks, outs)):
            hr, want = oracle.decompress(b, w, h, bc, df)
            assert hr == 0
            S.assert_same(o, want, df, "%s batch decompress %d -> %d image %d (%dx%d)" % (path, bc, df, i, w, h))
            assert np.array_equal(o, capi.decompress(b, w, h, bc, df)), (path, i)


@pytest.mark.parametrize("fmt,flags", [(2, 0), (2, 2), (10, 0), (10, 2)])
def test_mixed_size_batch_premultiply_alpha(oracle, fmt, flags):
    srcs = _mixed_sources(fmt)
    host = lambda: capi.premultiply_alpha_images(srcs, MIXED, fmt, flags)
    for path, outs in _both_paths(host, capi.lib.dxb200_premultiply_alpha_device, (flags,), srcs, fmt, fmt):
        for i, ((w, h), s_, o) in enumerate(zip(MIXED, srcs, outs)):
            hr, want = oracle.premultiply_alpha(s_, w, h, fmt, flags)
            assert hr == 0
            S.assert_same(o, want, fmt, "%s batch pmalpha fmt %d flags %d image %d (%dx%d)" % (path, fmt, flags, i, w, h))
            assert np.array_equal(o, capi.premultiply_alpha(s_, w, h, fmt, flags)), (path, i)
