"""GPU suite for the per-axis address modes (TEX_FILTER_WRAP_U / _V, MIRROR_U / _V, and the W bits as no-ops) of every mip and
resize route; the case table and its content are tests/address_modes.py.

Every case and word runs through dxb200_generate_mipmaps / dxb200_resize on host images and through their _device variants at a
row pitch 16 bytes wider than tight, each with DXB200_OPT_MIP_KERNELS 0 (the families the case names must launch) and 1 (only
k_mip_level), by test_gpu_mip_routes.check_route_and_result: bit for bit against the oracle, and with sRGB the generic kernel
level by level within one code, the specialised kernels bit for bit against the generic one.  Host and device results agree
bit for bit.  dxb200_mipmaps_compress to BC1 / BC3 equals the oracle's GenerateMipMaps + Compress, and
dxb200_mipmaps_compress_from with different words for its Resize and its mips equals the oracle's Resize + GenerateMipMaps +
Compress.  tests/test_cpu_address_modes.py checks on the reference that each case's words give different results wherever the
reference's filters read them, so a route that swaps, ORs or drops an axis fails here."""
import numpy as np
import pytest

from directxtex_b200 import capi
from tests import address_modes as A, test_gpu_mip_routes as R
from tests.test_gpu_mipmaps_compress_from import reference, reference_exact

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _init():
    assert capi.lib.dxb200_init(0) == 0


def check_case(oracle, c):
    srcs = A.sources(c)
    for word in c.words:
        host = R.check_route_and_result(oracle, A.route_case(c, word), srcs)
        dev = R.check_route_and_result(oracle, A.route_case(c, word, "pad16"), srcs)
        for l in range(len(host)):
            assert np.array_equal(host[l], dev[l]), (A.case_id(c), hex(word), "host != device", l)


@pytest.mark.parametrize("c", A.CASES, ids=A.case_id)
def test_every_route_and_word(oracle, c):
    check_case(oracle, c)


def test_triangle_grid(oracle):
    for c in A.TRI_GRID:
        check_case(oracle, c)


# ---- the fused mip-and-compress calls ---------------------------------------------------------------------------------
COMPRESS_CASES = [c for c in A.CASES if not c.resize and not c.fl and c.items == 1 and c.w * c.h <= 1 << 15 and
                  reference_exact(c.fmt, c.fmt, 71) and A.R.mode_of(A.route_case(c, 0)) in (A.CUB, A.TRI)]


@pytest.mark.parametrize("df", [71, 77])
def test_mipmaps_compress(oracle, df):
    """dxb200_mipmaps_compress to BC1 / BC3 = the oracle's GenerateMipMaps then Compress of every level, bit for bit"""
    assert {c.fmt for c in COMPRESS_CASES} >= {28, 87, 2, 10, 61, 41}, sorted({c.fmt for c in COMPRESS_CASES})
    for c in COMPRESS_CASES:
        src = A.sources(c)[0]
        for word in A.SHORT:
            fl = c.mode | word
            got = capi.mipmaps_compress([src], c.w, c.h, c.fmt, df, fl)[0]
            want = reference(oracle, src, c.w, c.h, c.fmt, df, c.fmt, (c.w, c.h), 0, fl)
            assert np.array_equal(got, want), (A.case_id(c), hex(word), df)


# (base extent, fmt, resized extent, Resize filter, mip filter): the two words act on different axes, so a call that used one
# step's word for the other would give another result
FROM_CASES = [((40, 30), 28, (120, 90), A.LIN | A.WU, A.CUB | A.WV), ((40, 30), 28, (120, 90), A.LIN | A.WV, A.CUB | A.WU),
              ((7, 5), 87, (20, 13), A.CUB | A.MU | A.WV, A.TRI | A.WU), ((30, 40), 10, (90, 120), A.CUB | A.MV, A.CUB | A.WU | A.MV),
              ((200, 30), 28, (50, 90), A.CUB | A.MV, A.TRI | A.WU)]


@pytest.mark.parametrize("df", [71, 77])
@pytest.mark.parametrize("base, fmt, size, rf, mf", FROM_CASES)
def test_mipmaps_compress_from_keeps_the_two_words_apart(oracle, df, base, fmt, size, rf, mf):
    """dxb200_mipmaps_compress_from with source.resizeFilter and filter set to different asymmetric words = the oracle's Resize
    with the first, GenerateMipMaps with the second, Compress; and that result differs from the one with the words exchanged"""
    (w, h), mode = base, R.MODE_MASK
    src = A.encode(fmt, A.content_rgba(w, h))
    got = capi.mipmaps_compress_from([src], w, h, fmt, df, source=capi.chain_source(0, size[0], size[1], rf), filter=mf)[0]
    want = reference(oracle, src, w, h, fmt, df, fmt, size, rf, mf)
    assert np.array_equal(got, want), (base, fmt, size, hex(rf), hex(mf), df)
    swapped = reference(oracle, src, w, h, fmt, df, fmt, size, (rf & mode) | (mf & ~mode), (mf & mode) | (rf & ~mode))
    assert not np.array_equal(want, swapped)
