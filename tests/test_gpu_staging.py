"""GPU suite for the host staging: every kernel on the batches split_bands / run_staged build (dxb_api.cu).

Almost every other GPU test hands a host-pointer call one small, tight image, which fits in one band and one chunk, so the kernel
gets exactly the job the test built.  Here the cases of tests/staging_cases.py (each named for the band cut, chunk packing or
kernel route it exists for; tests/test_cpu_staging.py checks that it hits them) run through the host-pointer calls

  - on numpy memory, on memory from dxb200_host_alloc, and with row pitches wider than tight (different per image, on both sides);
  - and each result must equal, bit for bit, the same operation as ONE _device launch on the whole batch (no bands, no chunks),
    and the reference: the oracle wherever the contract is bit-exact (BC1-BC5, decompress, non-sRGB convert and premultiply; the
    one-code rule where a decompress converts between sRGB and linear), the host emulator for BC6H / BC7 on the block rows next
    to every band cut.

Then: the status callbacks of compress_ex / convert_ex (values, count, abort at every callback and the next call on the same
lane), dxb200_mipmaps_compress against generate_mipmaps + compress for every BC target, source, filter and level count, BC6H /
BC7 on a second device, and four multi-chunk calls of different entry points at once (more than NLANE lanes)."""
import contextlib
import ctypes as C
import threading
import zlib

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import oracle_lib, special_values as S, staging_cases as SC
from tests.test_gpu_bc_formats import decompress_matches
from tests.test_gpu_special_values import device_call

pytestmark = pytest.mark.gpu

L = capi.lib
HOST = {SC.COMPRESS: L.dxb200_compress, SC.DECOMPRESS: L.dxb200_decompress, SC.CONVERT: L.dxb200_convert,
        SC.PMALPHA: L.dxb200_premultiply_alpha}
HOST_EX = {SC.COMPRESS: L.dxb200_compress_ex, SC.CONVERT: L.dxb200_convert_ex}
DEVICE = {SC.COMPRESS: L.dxb200_compress_device, SC.DECOMPRESS: L.dxb200_decompress_device, SC.CONVERT: L.dxb200_convert_device,
          SC.PMALPHA: L.dxb200_premultiply_alpha_device}
BC67 = (95, 96, 98, 99)
BC7_KERNELS = ("k_compress_bc7_tma", "k_compress_bc7")
CASES = {c.name: c for c in SC.CASES}


def only_device_0():
    """make device 0 the only initialised device: the expectations of this module (band cuts, chunks, callback values, kernel
    counts) are those of one device, and an earlier test may have initialised every GPU (run_sharded would then split the work)"""
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0
    devs = (C.c_int * 8)()
    assert L.dxb200_initialized_devices(devs, 8) == 1 and devs[0] == 0


@pytest.fixture(scope="module", autouse=True)
def _init():
    only_device_0()


def middle(case):
    """the arguments between (src, n) and dst of the case's entry point"""
    return {SC.COMPRESS: (case.df, case.flags, 0.5, 1.0), SC.DECOMPRESS: (case.df,), SC.CONVERT: (case.df, case.flags, 0.5),
            SC.PMALPHA: (case.flags,)}[case.op]


def _rows(fmt, w, h):
    row, sl = F.compute_pitch(fmt, w, h)
    return row, sl // row


def sources(case):
    rng = np.random.default_rng(zlib.crc32(case.name.encode()))
    out = []
    for (w, h) in case.sizes:
        if case.op == SC.DECOMPRESS:
            out.append(rng.integers(0, 256, F.compute_pitch(case.sf, w, h)[1], dtype=np.uint8))
        else:
            out.append(np.ascontiguousarray(oracle_lib.random_image(case.sf, w, h, rng)).view(np.uint8).reshape(-1))
    return out


def host_call(entry, mid, srcs, sizes, sf, df, spitches=None, dpitches=None, pinned=False, status=None):
    """entry(src images, n, *mid, dst images[, status, None]) on host copies of the tightly packed `srcs` with the given row
    pitches (default tight), in numpy or dxb200_host_alloc memory; returns (HRESULT, tightly packed results)"""
    spitches = spitches or [_rows(sf, w, h)[0] for (w, h) in sizes]
    dpitches = dpitches or [_rows(df, w, h)[0] for (w, h) in sizes]
    pins = []

    def buf(n):
        if not pinned:
            return np.empty(n, np.uint8)
        p = L.dxb200_host_alloc(n)
        assert p, "dxb200_host_alloc(%d)" % n
        pins.append(p)
        return np.ctypeslib.as_array((C.c_uint8 * n).from_address(p))
    try:
        simgs, dimgs, outs = [], [], []
        for src, (w, h), sp, dp in zip(srcs, sizes, spitches, dpitches):
            (srow, sn), (drow, dn) = _rows(sf, w, h), _rows(df, w, h)
            a, o = buf(sn * sp), buf(dn * dp)
            a.fill(0xA5)
            a.reshape(sn, sp)[:, :srow] = src.reshape(sn, srow)
            o.fill(0x5A)
            simgs.append(capi.Image(w, h, sf, sp, sn * sp, a.ctypes.data))
            dimgs.append(capi.Image(w, h, df, dp, dn * dp, o.ctypes.data))
            outs.append((a, o, dn, dp, drow))
        args = (capi.images(simgs), len(srcs)) + tuple(mid) + (capi.images(dimgs),)
        hr = entry(*args) if status is None else entry(*args, status, None)
        return F.hr_u32(hr), [o.reshape(dn, dp)[:, :drow].copy().reshape(-1) for (_, o, dn, dp, drow) in outs]
    finally:
        for p in pins:
            L.dxb200_host_free(p)


@contextlib.contextmanager
def bc7_feed(feed):
    old = L.dxb200_get_option(capi.OPT_BC7_FEED)
    if feed is not None:
        assert L.dxb200_set_option(capi.OPT_BC7_FEED, feed) == 0
    try:
        yield
    finally:
        L.dxb200_set_option(capi.OPT_BC7_FEED, old)


def counts():
    return {k: capi.kernel_launch_count(k) for k in BC7_KERNELS}


def strips(case, m, h):
    """pixel row ranges, on block rows, around every band cut of image m (and its last block row); the whole of a small image"""
    if h <= 16:
        return [(0, h)]
    bands = SC.plan(case)[0]
    cuts = [b.row0 for b in bands if b.image == m and b.row0 > 0]
    return [(max(0, c - 8), min(h, c + 8)) for c in cuts] + [(max(0, (h - 1) // 4 * 4 - 4), h)]


def check_reference(oracle, emul, case, srcs, outs):
    sf, df, fl = case.sf, case.df, case.flags
    for m, ((w, h), src, got) in enumerate(zip(case.sizes, srcs, outs)):
        ctx = "%s image %d (%dx%d)" % (case.name, m, w, h)
        if case.op == SC.COMPRESS and df in BC67:
            row = _rows(sf, w, h)[0]
            blocks = got.reshape(-1, ((w + 3) // 4) * 16)
            for r0, r1 in strips(case, m, h):
                he, em = emul.compress(src.reshape(h, row)[r0:r1], w, r1 - r0, sf, df, fl)
                assert he == 0
                assert np.array_equal(blocks[r0 // 4:(r1 + 3) // 4].reshape(-1), em), (ctx, r0, r1)
        elif case.op == SC.COMPRESS:
            hr, want = oracle.compress(src, w, h, sf, df, fl)
            assert hr == 0 and np.array_equal(got, want), ctx
        elif case.op == SC.DECOMPRESS:
            hr, want = oracle.decompress(src, w, h, sf, df)
            assert hr == 0 and decompress_matches(oracle, got, want, w, h, sf, df), ctx
        elif case.op == SC.CONVERT:
            hr, want = oracle.convert(src, w, h, sf, df, fl)
            assert hr == 0 and not S.mismatches(got, want, df).any(), ctx
        else:
            hr, want = oracle.premultiply_alpha(src, w, h, sf, fl)
            assert hr == 0 and not S.mismatches(got, want, sf).any(), ctx


# ---- 1. every band call: host memory, pinned memory, wide pitches == one device launch == the reference ---------------------
@pytest.mark.parametrize("case", SC.CASES, ids=lambda c: c.name)
def test_band_call_equals_one_device_launch_and_reference(oracle, emul, case):
    """Three host-pointer runs of the case (numpy, dxb200_host_alloc, wide pitches) equal one _device launch on the whole batch
    bit for bit, and that launch equals the reference.  BC7 runs under DXB200_OPT_BC7_FEED 0, 1 and 4, and each chunk must run
    the kernel staging_cases.bc7_kernel predicts for its jobs (the TMA feed for equal jobs at a constant stride)."""
    srcs = sources(case)
    bc7 = case.op == SC.COMPRESS and case.df in (98, 99)
    with bc7_feed(0 if bc7 else None):
        one = device_call(DEVICE[case.op], middle(case), srcs, list(case.sizes), case.sf, case.df)
    check_reference(oracle, emul, case, srcs, one)
    for feed in ((0, 1, 4) if bc7 else (None,)):
        for layout, pinned in (("tight", False), ("tight", True), ("wide", False)):
            sp, dp = SC.case_pitches(case, layout)
            before = counts()
            with bc7_feed(feed):
                hr, got = host_call(HOST[case.op], middle(case), srcs, case.sizes, case.sf, case.df, sp, dp, pinned)
            ctx = (case.name, layout, "pinned" if pinned else "numpy", feed)
            assert hr == 0, (ctx, hex(hr), capi.last_error())
            for m, (g, o) in enumerate(zip(got, one)):
                assert np.array_equal(g, o), (ctx, "image %d differs from the device launch" % m)
            if bc7:
                want = [SC.bc7_kernel(js, feed) for js in SC.plan(case, layout)[2]]
                moved = {k: v - before[k] for k, v in counts().items()}
                assert moved == {k: want.count(k) for k in BC7_KERNELS}, (ctx, moved, want)


# ---- 2. progress and abort through the C ABI ----------------------------------------------------------------------------------
def expected_progress(case):
    """the callback values of a band call: before every chunk the units done so far, then (total, total) (DirectXTexCompress.cpp
    reports pixel rows of one image, images of an array)"""
    bands, chunks, _ = SC.plan(case)
    total, done, seq = sum(b.units for b in bands), 0, []
    for c in chunks:
        seq.append((done, total))
        done += sum(bands[i].units for i in c)
    return seq + [(total, total)]


def status_call(case, srcs, stop_at=None):
    calls = []

    def cb(done, total, user):
        calls.append((done, total))
        return 0 if stop_at is not None and len(calls) == stop_at + 1 else 1
    fn = capi.STATUS_FN(cb)
    hr, outs = host_call(HOST_EX[case.op], middle(case), srcs, case.sizes, case.sf, case.df, status=fn)
    return hr, outs, calls


@pytest.mark.parametrize("name", [c.name for c in SC.CASES if c.op in HOST_EX])
def test_progress_values_and_abort_at_every_callback(name):
    """compress_ex / convert_ex on every compress and convert case: the callback starts at 0, rises in pixel rows of a single
    image (images of an array) once per chunk -- run_staged reports before each chunk, which holds whole bands -- and ends with
    (total, total): the values the Python copy of the staging predicts, and total = height or the image count.  Returning false at callback k, for every k, gives E_ABORT with no later callback, and the same call right after it
    without a callback returns the full result: an abort between chunks leaves no busy lane or unsynchronised slot behind."""
    case = CASES[name]
    srcs = sources(case)
    hr, ref = host_call(HOST[case.op], middle(case), srcs, case.sizes, case.sf, case.df)
    assert hr == 0
    want = expected_progress(case)
    total = case.sizes[0][1] if len(case.sizes) == 1 else len(case.sizes)
    hr, outs, calls = status_call(case, srcs)
    assert hr == 0 and calls == want and want[-1] == (total, total), (name, calls, want)
    assert all(a[0] <= b[0] for a, b in zip(calls, calls[1:]))
    for o, r in zip(outs, ref):
        assert np.array_equal(o, r), name
    for k in range(len(want)):
        hr, _, calls = status_call(case, srcs, stop_at=k)
        assert hr == F.E_ABORT and calls == want[:k + 1], (name, k, hex(hr), calls)
        hr, outs = host_call(HOST[case.op], middle(case), srcs, case.sizes, case.sf, case.df)
        assert hr == 0, (name, k, capi.last_error())
        for o, r in zip(outs, ref):
            assert np.array_equal(o, r), (name, "after abort at", k)


# ---- 3. dxb200_mipmaps_compress across targets, sources, filters and layouts ------------------------------------------------
MIP_FILTERS = (F.TEX_FILTER_POINT, F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, 0)
MIP_SOURCES = (28, 2, 10, 61, 49)


def mipmaps_compress(srcs, w, h, sf, df, filter, levels, extras=None):
    """dxb200_mipmaps_compress of equally sized host images whose level 0 rows are `extras[i]` bytes wider than tight; returns
    (HRESULT, one packed BC chain per image)"""
    extras = extras or [0] * len(srcs)
    row, _ = F.compute_pitch(sf, w, h)
    layout, total = capi.texture_layout(df, w, h, 1, levels)
    bases, outs = [], [np.zeros(total, np.uint8) for _ in srcs]
    for src, e in zip(srcs, extras):
        a = np.full((h, row + e), 0xA5, np.uint8)
        a[:, :row] = src.reshape(h, row)
        bases.append(a)
    s = capi.images([capi.Image(w, h, sf, row + e, (row + e) * h, a.ctypes.data) for a, e in zip(bases, extras)])
    d = capi.images([capi.Image(lw, lh, df, r, sp, o.ctypes.data + off) for o in outs for (off, lw, lh, r, sp) in layout])
    hr = L.dxb200_mipmaps_compress(s, len(srcs), levels, filter, df, 0, 0.5, 1.0, d)
    return F.hr_u32(hr), outs


def two_calls(src, w, h, sf, df, filter, levels):
    chain, layout = capi.generate_mipmaps(src, w, h, sf, filter, levels)
    return chain, layout, np.concatenate([capi.compress(chain[off:off + sl], lw, lh, sf, df) for (off, lw, lh, row, sl) in layout])


@pytest.mark.parametrize("df", sorted(F.BLOCK_BYTES))
def test_mipmaps_compress_every_target_source_filter(oracle, df):
    """Every source (28, 2, 10, 61, 49) x filter (POINT, BOX, LINEAR, CUBIC, TRIANGLE, 0) x a full chain and levels = 2 on 64 x 16
    (a non-square power-of-two chain down to height 1: BOX's stale row) and 40 x 24 (deep levels smaller than a block; BOX is
    refused there): bit for bit generate_mipmaps + compress on the GPU, and for BC1-BC5 without a powf step the reference's
    compression of the reference's chain."""
    bad, total = [], 0
    for sf in MIP_SOURCES:
        rng = np.random.default_rng(df * 101 + sf)
        for (w, h) in ((64, 16), (40, 24)):
            srcs = [np.ascontiguousarray(oracle_lib.random_image(sf, w, h, rng)).view(np.uint8).reshape(-1) for _ in range(2)]
            for fl in MIP_FILTERS:
                for levels in (F.count_mips(w, h), 2):
                    hr, outs = mipmaps_compress(srcs, w, h, sf, df, fl, levels)
                    ctx = "%d -> %d %dx%d filter %#x levels %d" % (sf, df, w, h, fl, levels)
                    if fl == F.TEX_FILTER_BOX and (w, h) == (40, 24):
                        assert hr == F.E_FAIL, (ctx, hex(hr))          # BOX needs power-of-two sizes (GenerateMipMaps)
                        continue
                    assert hr == 0, (ctx, hex(hr), capi.last_error())
                    for i, (src, got) in enumerate(zip(srcs, outs)):
                        total += 1
                        chain, layout, want = two_calls(src, w, h, sf, df, fl, levels)
                        if not np.array_equal(got, want):
                            bad.append("%s image %d != two calls" % (ctx, i))
                            continue
                        if df in BC67 or S.powf_direction(0, sf, df):
                            continue
                        hr, rchain = oracle.generate_mipmaps(src, w, h, sf, fl, levels)
                        assert hr == 0
                        ref = np.concatenate([oracle.compress(rchain[off:off + sl], lw, lh, sf, df)[1] for (off, lw, lh, row, sl) in layout])
                        if not np.array_equal(got, ref):
                            bad.append("%s image %d != reference" % (ctx, i))
    assert not bad, "%d of %d differ; first: %s" % (len(bad), total, "; ".join(bad[:6]))


@pytest.mark.parametrize("sf,df,w,h,items,fl,extras,nchunks", [
    (28, 77, 1024, 1024, 12, 0, (0, 64, 4), 2),                     # eleven chains per chunk, then one
    (2, 98, 2048, 2048, 2, F.TEX_FILTER_CUBIC, (64, 16), 2),        # each chain larger than a chunk
    (10, 95, 512, 128, 3, F.TEX_FILTER_BOX, (8, 0, 136), 1),        # a non-square chain down to height 1
    (61, 80, 1000, 600, 2, F.TEX_FILTER_TRIANGLE, (4, 68), 1)])
def test_mipmaps_compress_over_chunks_with_wide_level0(sf, df, w, h, items, fl, extras, nchunks):
    """Arrays of chains over several 80 MiB chunks, single chains larger than a chunk and single-chunk arrays, level 0 at row pitches wider than
    tight (different per item; the other levels are tight in device memory): each chain equals generate_mipmaps + compress."""
    levels = F.count_mips(w, h)
    ex = [extras[i % len(extras)] for i in range(items)]
    chunks, item_bytes = SC.chain_chunks(sf, df, w, h, items, levels, max(ex))
    assert len(chunks) == nchunks, chunks
    rng = np.random.default_rng(w + items)
    srcs = [np.ascontiguousarray(oracle_lib.random_image(sf, w, h, rng)).view(np.uint8).reshape(-1) for _ in range(items)]
    hr, outs = mipmaps_compress(srcs, w, h, sf, df, fl, levels, ex)
    assert hr == 0, (hex(hr), capi.last_error())
    for i, (src, got) in enumerate(zip(srcs, outs)):
        assert np.array_equal(got, two_calls(src, w, h, sf, df, fl, levels)[2]), (sf, df, w, h, i)


# ---- 4. more than one device --------------------------------------------------------------------------------------------------
def test_bc7_bc6h_on_every_device():
    """With every GPU initialised, BC7 (a single image under feed 0, a TMA-fed array) and BC6H through the host API are sharded
    over the devices and equal one device's launch; the _device calls work on pointers that live on device 1.  The BC7 kernels
    need their shared-memory limit raised in every device's context."""
    torch = pytest.importorskip("torch")
    n = L.dxb200_device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    capi.init_devices(list(range(n)))
    try:
        compare_on_every_device(torch, n)
    finally:
        only_device_0()


def compare_on_every_device(torch, n):
    single, array, bc6h = CASES["bc7-2bands"], CASES["bc7-array"], CASES["bc6h-2bands"]
    rng = np.random.default_rng(5)
    arr_sizes = [(256, 256)] * (4 * n)
    arr = [np.ascontiguousarray(oracle_lib.random_image(2, 256, 256, rng)).view(np.uint8).reshape(-1) for _ in arr_sizes]
    for name, srcs, sizes, df, feed in (("single", sources(single), single.sizes, 98, 0), ("array", arr, arr_sizes, 98, 4),
                                        ("bc6h", sources(bc6h), bc6h.sizes, 96, None), ("bc6h array", arr, arr_sizes, 96, None)):
        with bc7_feed(feed):
            one = device_call(L.dxb200_compress_device, (df, 0, 0.5, 1.0), srcs, list(sizes), 2, df)
            hr, got = host_call(L.dxb200_compress, (df, 0, 0.5, 1.0), srcs, sizes, 2, df)
            assert hr == 0, (name, hex(hr), capi.last_error())
            for g, o in zip(got, one):
                assert np.array_equal(g, o), name
            with torch.cuda.device(1):
                on1 = device_call(L.dxb200_compress_device, (df, 0, 0.5, 1.0), srcs, list(sizes), 2, df)
            for a, o in zip(on1, one):
                assert np.array_equal(a, o), (name, "device 1")


# ---- 5. four threads, more calls than lanes -----------------------------------------------------------------------------------
def test_four_multi_chunk_calls_at_once():
    """A TMA-fed BC7 array, a generic convert, a mip array and a decompress, each over several chunks, from four threads at once
    (more calls than a device has lanes): every result equals the same call made alone."""
    bc7, cvt, dec = CASES["bc7-array"], CASES["cvt2-87"], CASES["dec71-28"]
    mip_items, mw = 20, 1024
    rng = np.random.default_rng(11)
    mips = [oracle_lib.random_image(28, mw, mw, rng) for _ in range(mip_items)]
    chain_bytes = sum(SC.pad256(sl) for (_, _, _, _, sl) in F.mip_chain_layout(28, mw, mw)[0])
    assert len(SC.group_chunks([chain_bytes] * mip_items, SC.ITEM_CHUNK)) >= 2
    jobs = {
        "bc7": lambda s=sources(bc7): host_call(HOST[bc7.op], middle(bc7), s, bc7.sizes, bc7.sf, bc7.df),
        "convert": lambda s=sources(cvt): host_call(HOST[cvt.op], middle(cvt), s, cvt.sizes, cvt.sf, cvt.df),
        "decompress": lambda s=sources(dec): host_call(HOST[dec.op], middle(dec), s, dec.sizes, dec.sf, dec.df),
        "mips": lambda: (0, capi.generate_mipmaps_images(mips, mw, mw, 28, 0)),
    }
    before = capi.tma_launch_count()
    alone = {k: f() for k, f in jobs.items()}
    assert capi.tma_launch_count() >= before + 2
    res, errs = {}, []

    def work(k):
        try:
            res[k] = jobs[k]()
        except Exception as e:          # reported below: an exception in a thread would otherwise vanish
            errs.append((k, e))
    th = [threading.Thread(target=work, args=(k,)) for k in jobs]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for k, (hr, outs) in alone.items():
        assert hr == 0 and res[k][0] == 0, k
        for a, b in zip(outs, res[k][1]):
            assert np.array_equal(a, b), k


# ---- 6. host images at any address --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bc", [71, 77, 98])
def test_host_bc_images_at_unaligned_addresses(oracle, bc):
    """A host-pointer call stages its images into aligned device buffers, so a BC image may sit at any host address (block data
    at offset 148 of a DX10 DDS file, a destination 4 bytes into a buffer): compress and decompress there equal the same calls
    on aligned buffers, and the reference."""
    w, h = 40, 28
    row, sl = F.compute_pitch(bc, w, h)
    rng = np.random.default_rng(bc)
    src = np.ascontiguousarray(oracle_lib.random_image(28, w, h, rng)).view(np.uint8).reshape(-1)
    want = capi.compress(src, w, h, 28, bc)
    out = np.zeros(sl + 4, np.uint8)
    s = capi.images([capi.Image(w, h, 28, w * 4, w * h * 4, src.ctypes.data)])
    d = capi.images([capi.Image(w, h, bc, row, sl, out.ctypes.data + 4)])
    assert L.dxb200_compress(s, 1, bc, 0, 0.5, 1.0, d) == 0, capi.last_error()
    assert np.array_equal(out[4:], want)
    blob = np.zeros(148 + sl, np.uint8)
    blob[148:] = want
    pix = np.zeros(w * h * 4, np.uint8)
    s = capi.images([capi.Image(w, h, bc, row, sl, blob.ctypes.data + 148)])
    d = capi.images([capi.Image(w, h, 28, w * 4, w * h * 4, pix.ctypes.data)])
    assert L.dxb200_decompress(s, 1, 28, d) == 0, capi.last_error()
    hr, ref = oracle.decompress(want, w, h, bc, 28)
    assert hr == 0 and np.array_equal(pix, capi.decompress(want, w, h, bc, 28)) and np.array_equal(pix, ref)
