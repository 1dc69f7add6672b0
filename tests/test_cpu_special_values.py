"""CPU suite: the host lock-step emulator of our kernels against the oracle on the special-value corpus
(tests/special_values.py): +-0, denormals, the half overflow points, +-Inf, FLT_MAX, the rounding ties of every store, every
non-NaN half pattern and the packed-source patterns.  Convert over every supported pair and flag family, mip chains with
every filter, BC1-BC5; and the GPU suite's lists of vector-kernel routes against the kernels compiled into the library.
No GPU needed."""
import numpy as np
import pytest

from directxtex_b200 import formats as F
from tests import special_values as S, test_gpu_mip_routes as R, test_gpu_special_values as V
from tests.kernel_routes import kernel_entries

PIXEL_FORMATS = sorted(F.BYTES_PER_PIXEL)
CONVERT_FLAGS = (0, F.TEX_FILTER_FLOAT_X2BIAS, F.TEX_FILTER_RGB_COPY_RED, F.TEX_FILTER_RGB_COPY_GREEN, F.TEX_FILTER_RGB_COPY_BLUE,
                 F.TEX_FILTER_DITHER, F.TEX_FILTER_DITHER_DIFFUSION, F.TEX_FILTER_SRGB_IN, F.TEX_FILTER_SRGB_OUT, F.TEX_FILTER_SRGB)
CORPUS_SOURCES = S.F32_FORMATS + S.F16_FORMATS + S.PACKED16 + (26, 67)


def corpus_source(fmt):
    """(bytes, w, h): the fp32 corpus at 64 x 20, the half corpus, the packed-source patterns"""
    if fmt in S.F32_FORMATS:
        return S.f32_image(fmt, 64, 20).view(np.uint8).reshape(-1), 64, 20
    if fmt in S.F16_FORMATS:
        img, h = S.half_image(fmt, 256)
        return img.view(np.uint8).reshape(-1), 256, h
    return S.source_image(fmt, 256, 256), 256, 256


def test_gpu_vector_kernel_lists_name_every_compiled_instantiation():
    """the GPU suite's k_convert_vec pairs and k_pmalpha_vec formats, each format replaced by its UNORM twin (dxb_make_linear),
    are exactly the instantiations compiled into the library (k_pmalpha_vec: each format in both directions, sRGB or not)"""
    twin = lambda f: R.TWIN.get(f, f)
    k = kernel_entries()
    assert {(twin(a), twin(b)) for a, b in V.VEC_PAIRS} == k["k_convert_vec"]
    assert {(twin(f), rev, srgb) for f in V.PMALPHA_VEC_FORMATS for rev in (False, True) for srgb in (False, True)} == k["k_pmalpha_vec"]


@pytest.mark.parametrize("sf", CORPUS_SOURCES)
def test_convert_every_pair_special_values(oracle, emul, sf):
    src, w, h = corpus_source(sf)
    n = 0
    for df in PIXEL_FORMATS:
        if df == sf:
            continue
        for fl in CONVERT_FLAGS:
            if S.convert_refused(df, fl):
                continue
            hr, want = oracle.convert(src, w, h, sf, df, fl)
            he, got = emul.convert(src, w, h, sf, df, fl)
            assert hr == 0 and he == 0, (sf, df, hex(fl), hex(hr), hex(he))
            S.assert_same(got, want, df, "convert %d -> %d flags %#x" % (sf, df, fl))
            n += 1
    assert n >= 250


MIP_FILTERS = (F.TEX_FILTER_POINT, F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, 0,
               F.TEX_FILTER_LINEAR | F.TEX_FILTER_WRAP, F.TEX_FILTER_LINEAR | F.TEX_FILTER_MIRROR,
               F.TEX_FILTER_CUBIC | F.TEX_FILTER_WRAP, F.TEX_FILTER_CUBIC | F.TEX_FILTER_MIRROR,
               F.TEX_FILTER_TRIANGLE | F.TEX_FILTER_WRAP, F.TEX_FILTER_BOX | F.TEX_FILTER_WRAP)


def mip_sources(fmt):
    """(bytes, w, h) corpus images for mip chains: one power-of-two size (BOX) and one odd size per format"""
    out = []
    for (w, h) in ((32, 32), (37, 19)):
        if fmt in (2, 41):
            out.append((S.f32_image(fmt, w, h, seed=w).view(np.uint8).reshape(-1), w, h))
        elif fmt == 10:
            with np.errstate(over="ignore"):                    # values beyond 65504 become half Inf: part of the corpus
                out.append((S.edge_image(w, h, seed=w).astype(np.float16).view(np.uint8).reshape(-1), w, h))
        else:
            out.append((S.source_image(fmt, w, h, seed=w), w, h))
    if fmt == 10:
        img, h = S.half_image(10, 256)
        out.append((np.ascontiguousarray(img[:128]).view(np.uint8).reshape(-1), 256, 128))
    return out


@pytest.mark.parametrize("fmt", [2, 10, 41, 26, 67])
def test_mips_every_filter_special_values(oracle, emul, fmt):
    for src, w, h in mip_sources(fmt):
        for fl in MIP_FILTERS:
            if (fl & 0xF00000) == F.TEX_FILTER_BOX and (w & (w - 1) or h & (h - 1)):
                continue
            hr, want = oracle.generate_mipmaps(src, w, h, fmt, fl)
            he, got = emul.generate_mipmaps(src, w, h, fmt, fl)
            assert hr == 0 and he == 0, (fmt, w, h, hex(fl))
            S.assert_same(got, want, fmt, "mips fmt %d %dx%d filter %#x" % (fmt, w, h, fl))


@pytest.mark.parametrize("bc", [71, 74, 77, 80, 81, 83, 84])
def test_bc15_special_values(oracle, emul, bc):
    srcs = [(S.f32_image(sf, 64, 20, seed=bc).view(np.uint8).reshape(-1), 64, 20, sf) for sf in S.F32_FORMATS]
    img, h = S.half_image(10, 256)
    srcs.append((img.view(np.uint8).reshape(-1), 256, h, 10))
    for src, w, h, sf in srcs:
        for flags in (0, F.TEX_COMPRESS_UNIFORM, F.TEX_COMPRESS_DITHER):
            hr, want = oracle.compress(src, w, h, sf, bc, flags)
            he, got = emul.compress(src, w, h, sf, bc, flags)
            assert hr == 0 and he == 0
            S.assert_same(got, want, bc, "BC %d from %d flags %#x" % (bc, sf, flags))


def test_corpus_properties():
    """the corpus itself: no NaN anywhere, every edge value in every channel position, +Inf next to -Inf"""
    e = S.f32_edges()
    assert not np.isnan(e).any() and np.isinf(e).sum() == 2 and (e.view(np.uint32) == 0x80000000).any()
    img = S.edge_image(64, 20)
    for c in range(4):
        assert np.isin(e.view(np.uint32), img[..., c].reshape(-1).view(np.uint32)).all(), c
    blk = img[0:2, 0:2].reshape(-1, 4)
    assert (blk == np.inf).any(0).all() and (blk == -np.inf).any(0).all()
    hp = S.half_patterns()
    assert hp.size == 63490 and not np.isnan(hp.view(np.float16)).any()
    himg, _ = S.half_image(10, 256)
    for c in range(4):
        assert np.isin(hp, himg[..., c]).all(), c
    p26 = S.packed_patterns(26)
    for off, mb in ((0, 6), (11, 6), (22, 5)):
        m, ex = (p26 >> off) & ((1 << mb) - 1), (p26 >> (off + mb)) & 0x1F
        assert not ((ex == 31) & (m != 0)).any() and ((ex == 31) & (m == 0)).any()
