"""CPU suite: the coverage search of a whole batch replayed from recorded counts, and the argument checks of
dxb200_mipmaps_compress_ex.

The batched emulator (tests/emul/coverage_batch.cpp) plans its batch with the library's job table and advances every job's
search one step at a time from the counts recorded so far, with the rule the kernels replay (dxb_coverage.h); each item must come
out as the reference's ScaleMipMapsAlphaForCoverage makes it.  The HRESULT table needs no device: every check of the four steps
happens before anything is uploaded."""
import ctypes as C
import os

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import oracle_lib
from tests.bc7_ranking_build import host_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def batch_emul(tmp_path_factory):
    L = host_lib("coverage_batch.cpp", tmp_path_factory.mktemp("coverage_batch"), os.path.join(ROOT, "tests", "emul"))
    sz = C.c_size_t
    L.emul_scale_mips_alpha_batch.argtypes = [C.c_void_p, C.c_void_p, sz, sz] + [C.POINTER(sz)] * 4 + [sz, C.c_uint32, C.c_float]
    L.emul_scale_mips_alpha_batch.restype = C.c_int32
    return L


def scale_batch(L, chains, w, h, fmt, ref):
    """the emulator's batched search over equally sized chains (ScratchImage layout, one bytes array each); (hr, results)"""
    layout, total = F.mip_chain_layout(fmt, w, h, 0)
    src = np.concatenate([np.ascontiguousarray(c).view(np.uint8).reshape(-1) for c in chains])
    out = np.zeros_like(src)
    A = C.c_size_t * len(layout)
    cols = [A(*[l[k] for l in layout]) for k in range(4)]
    hr = L.emul_scale_mips_alpha_batch(src.ctypes.data, out.ctypes.data, total, len(chains), *cols, len(layout), fmt, ref)
    return F.hr_u32(hr), [out[i * total:(i + 1) * total] for i in range(len(chains))]


def alpha_codes(fmt, ref):
    """alpha values next to `ref` in the format's own precision: the code below, the code of ref, the code above"""
    if fmt in (28, 29, 87):
        c = int(round(ref * 255))
        return np.array([c - 1, c, c + 1]) / 255.0
    dt = np.float16 if fmt == 10 else np.float32
    r = dt(ref)
    return np.array([np.nextafter(r, dt(0)), r, np.nextafter(r, dt(1))], np.float64)


def batch_items(fmt, w, h, ref, rng):
    """4 items that stop at different steps: opaque (step 0), smooth random alpha, alphas at ref +-1 code, sparse alpha"""
    yy, xx = np.mgrid[0:h, 0:w]
    smooth = np.clip(0.5 + 0.4 * np.sin(xx * 0.4) * np.cos(yy * 0.3) + rng.normal(0, 0.12, (h, w)), 0, 1)
    near = alpha_codes(fmt, ref)[rng.integers(0, 3, (h, w))]
    sparse = np.where(rng.random((h, w)) < 0.15, 1.0, 0.0)
    alphas = [np.ones((h, w)), smooth, near, sparse]
    out = []
    for a in alphas:
        if fmt in (28, 29, 87):
            img = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
            img[..., 3] = np.round(a * 255).astype(np.uint8)
        elif fmt == 86:                                             # B5G5R5A1: alpha is bit 15
            img = rng.integers(0, 1 << 15, (h, w), dtype=np.uint16) | (np.where(a >= 0.5, 1, 0).astype(np.uint16) << 15)
        else:
            img = rng.random((h, w, 4), dtype=np.float32)
            img[..., 3] = a
            img = img.astype(np.float16) if fmt == 10 else img
        out.append(np.ascontiguousarray(img))
    return out


@pytest.mark.parametrize("fmt", [28, 87, 2, 10, 86])
def test_batched_search_equals_reference_per_item(oracle, batch_emul, fmt):
    """Four items per call whose searches stop at different steps (an opaque item stops at step 0), on 64 x 16 (its deep levels
    are one pixel high, so they have no 2x2 cell) and 40 x 24, at references 0.5 and 0.25: every item of the batch equals the
    reference's GenerateMipMaps + ScaleMipMapsAlphaForCoverage of that item alone, bit for bit."""
    rng = np.random.default_rng(fmt)
    for (w, h) in ((64, 16), (40, 24)):
        for ref in (0.5, 0.25):
            items = batch_items(fmt, w, h, ref, rng)
            plains, wants = [], []
            for img in items:
                hr, plain, want = oracle.mips_alpha_coverage(img, w, h, fmt, ref)
                assert hr == 0, (fmt, w, h, ref, hex(hr))
                plains.append(plain)
                wants.append(want)
            hr, gots = scale_batch(batch_emul, plains, w, h, fmt, ref)
            assert hr == 0
            for i, (got, want) in enumerate(zip(gots, wants)):
                assert np.array_equal(got, want), (fmt, w, h, ref, "item", i)
            (o1, _, _, _, s1) = F.mip_chain_layout(fmt, w, h, 0)[0][1]
            assert np.array_equal(wants[0][o1:o1 + s1], plains[0][o1:o1 + s1]), "the opaque item's level 1 stops at step 0, scale 1"


def _ex(base_imgs, items, levels, filter, steps, dst_fmt, dst):
    return F.hr_u32(capi.lib.dxb200_mipmaps_compress_ex(base_imgs, items, levels, filter, C.byref(steps) if steps is not None else None,
                                                        dst_fmt, 0, 0.5, 1.0, dst))


def _call(w, h, fmt, dst_fmt=77, filter=0, levels=0, steps=None):
    """dxb200_mipmaps_compress_ex of one w x h item; its HRESULT"""
    row, sl = F.compute_pitch(fmt, w, h)
    src = np.zeros(max(sl, 16), np.uint8)
    levels = levels or F.count_mips(w, h)
    layout, total = capi.texture_layout(dst_fmt, w, h, 1, min(levels, F.count_mips(w, h)))
    out = np.zeros(total + 16, np.uint8)
    d = capi.images([capi.Image(lw, lh, dst_fmt, r, sp, out.ctypes.data + off) for (off, lw, lh, r, sp) in layout] * 2)
    return _ex(capi.images([capi.Image(w, h, fmt, row, sl, src.ctypes.data)]), 1, levels, filter, steps, dst_fmt, d)


def test_mipmaps_compress_ex_hresults(oracle):
    """The HRESULT of the first step of GenerateMipMaps -> ScaleMipMapsAlphaForCoverage -> PremultiplyAlpha -> Compress that
    fails, decided before any upload; where the reference defines it, its own composed calls give the same code."""
    both = capi.chain_steps(0.5, True)
    pm = capi.chain_steps(premultiply=True)
    img = np.zeros(8, np.uint8)
    good = capi.images([capi.Image(8, 8, 28, 32, 256, np.zeros(256, np.uint8).ctypes.data)])
    dst = capi.images([capi.Image(8, 8, 77, 32, 64, img.ctypes.data)] * 4)
    # pointers and counts
    assert _ex(None, 1, 4, 0, both, 77, dst) == F.E_INVALIDARG
    assert _ex(good, 1, 4, 0, both, 77, None) == F.E_INVALIDARG
    assert _ex(good, 0, 4, 0, both, 77, dst) == F.E_INVALIDARG
    assert _ex(good, 1, 0, 0, both, 77, dst) == F.E_INVALIDARG
    assert _ex(capi.images([capi.Image(8, 8, 28, 32, 256, None)]), 1, 4, 0, both, 77, dst) == F.E_POINTER
    rng = np.random.default_rng(3)
    # more levels than the chain has (GenerateMipMaps)
    src = oracle_lib.random_image(28, 40, 24, rng)
    hr_ref, _ = oracle.generate_mipmaps(src, 40, 24, 28, 0, 7)
    assert _call(40, 24, 28, levels=7, steps=both) == hr_ref == F.E_INVALIDARG
    # BOX on a size that is not a power of two (GenerateMipMaps :1005-1006)
    hr_ref, _ = oracle.generate_mipmaps(src, 40, 24, 28, F.TEX_FILTER_BOX)
    assert _call(40, 24, 28, filter=F.TEX_FILTER_BOX, steps=both) == hr_ref == F.E_FAIL
    # premultiply on formats without alpha (PremultiplyAlpha :224-229), with and without the coverage step in front
    for fmt in (61, 41):
        src = oracle_lib.random_image(fmt, 16, 16, rng)
        hr_mips, chain = oracle.generate_mipmaps(src, 16, 16, fmt)
        hr_pm, _ = oracle.premultiply_alpha(chain, 16, 16, fmt)
        assert hr_mips == 0 and hr_pm == F.HRESULT_E_NOT_SUPPORTED
        for steps in (pm, both):
            assert _call(16, 16, fmt, steps=steps) == hr_pm, fmt
    # a BC base: GenerateMipMaps refuses it
    assert _call(16, 16, 71, steps=both) == F.HRESULT_E_NOT_SUPPORTED
    # valid arguments reach the device; without one the call fails, as every compute entry point does
    if capi.lib.dxb200_device_count() == 0:
        for steps in (None, pm, both, capi.chain_steps(0.25), capi.chain_steps(-1.0, True, 0x2)):
            assert _call(40, 24, 28, steps=steps) == F.E_FAIL
