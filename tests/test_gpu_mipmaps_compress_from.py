"""GPU suite: dxb200_mipmaps_compress_from, texconv's Decompress -> Resize -> GenerateMipMaps -> [coverage] -> [premultiply] -> Compress
with every intermediate kept in device memory.

Every result equals the separate library calls (decompress, resize, mipmaps_compress_ex) bit for bit, and where the reference's
own composed calls are bit-exact, those too."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import special_values as S, staging_cases as SC
from tests.test_gpu_chain_steps import alpha_image, compress_chain, family, launches, separate_chains

pytestmark = pytest.mark.gpu
L = capi.lib
BC = sorted(F.BLOCK_BYTES)
HDR = (95, 96)
FILTERS = (0, F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, F.TEX_FILTER_POINT)
POINT, LINEAR, CUBIC, TRIANGLE, BOX = F.TEX_FILTER_POINT, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, F.TEX_FILTER_BOX
DEFAULT = {71: 28, 74: 28, 77: 28, 98: 28, 72: 29, 75: 29, 78: 29, 99: 29, 80: 61, 81: 63, 83: 49, 84: 51, 95: 2, 96: 2}
# one explicit decompress format per BC source: R8G8B8A8_SNORM for the SNORM formats (texconv's pick), RGBA16F for BC6H, BGRA8 for
# the UNORM colour formats, RGBA8 for BC4 / BC5 UNORM
EXPLICIT = {71: 87, 74: 87, 77: 87, 98: 87, 72: 91, 75: 91, 78: 91, 99: 91, 80: 28, 81: 31, 83: 28, 84: 31, 95: 10, 96: 10}


@pytest.fixture(autouse=True)
def one_device():
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0


def bc_base(fmt, w, h, rng):
    """a w x h image of `fmt` made by the library's encoder from random content (LDR alpha edges; HDR floats for BC6H)"""
    if fmt in HDR:
        img = (rng.random((h, w, 4), dtype=np.float32) * 4.0).astype(np.float32)
        return capi.compress(np.ascontiguousarray(img), w, h, 2, fmt)
    return capi.compress(alpha_image(28, w, h, rng), w, h, 28, fmt)


def hr_of(fn, *args, **kw):
    try:
        return 0, fn(*args, **kw)
    except capi.DxTexError as e:
        return e.hr, None


def from_call(bases, w, h, fmt, df, source, filter=0, steps=None, extras=None):
    """dxb200_mipmaps_compress_from of equally sized host images, rows of item i `extras[i]` bytes wider than tight; (hr, chains)"""
    extras = extras or [0] * len(bases)
    row, sl = F.compute_pitch(fmt, w, h)
    rows = sl // row
    cw, ch = (source.width, source.height) if source is not None and source.width else (w, h)
    levels = F.count_mips(cw, ch)
    layout, total = capi.texture_layout(df, cw, ch, 1, levels)
    held, outs = [], [np.zeros(total, np.uint8) for _ in bases]
    for b, e in zip(bases, extras):
        a = np.full((rows, row + e), 0xA5, np.uint8)
        a[:, :row] = np.ascontiguousarray(b).view(np.uint8).reshape(rows, row)
        held.append(a)
    s = capi.images([capi.Image(w, h, fmt, row + e, (row + e) * rows, a.ctypes.data) for a, e in zip(held, extras)])
    d = capi.images([capi.Image(lw, lh, df, r, sp, o.ctypes.data + off) for o in outs for (off, lw, lh, r, sp) in layout])
    hr = L.dxb200_mipmaps_compress_from(s, len(bases), C.byref(source) if source is not None else None, levels, filter,
                                        C.byref(steps) if steps is not None else None, df, 0, 0.5, 1.0, d)
    return F.hr_u32(hr), outs


def separate(bases, w, h, fmt, df, dfmt, size, rfilter, filter, steps=None):
    """decompress (a BC base) -> resize (another size) -> mipmaps_compress_ex as separate library calls; (hr, chains)"""
    imgs, lw, lh = bases, w, h
    if fmt in F.BLOCK_BYTES:
        imgs = capi.decompress_images(bases, [(w, h)] * len(bases), fmt, dfmt)
        fmt = dfmt
    if size != (w, h):
        imgs = capi.resize_images(imgs, w, h, fmt, size[0], size[1], rfilter)
        lw, lh = size
    return hr_of(capi.mipmaps_compress, imgs, lw, lh, fmt, df, filter, steps=steps)


def reference(oracle, base, w, h, fmt, df, dfmt, size, rfilter, filter):
    """the reference's Decompress -> Resize -> GenerateMipMaps -> Compress of one item"""
    img = base
    if fmt in F.BLOCK_BYTES:
        hr, img = oracle.decompress(base, w, h, fmt, dfmt)
        assert hr == 0
        fmt = dfmt
    if size != (w, h):
        hr, img = oracle.resize(img, w, h, fmt, size[0], size[1], rfilter)
        assert hr == 0
        w, h = size
    hr, chain = oracle.generate_mipmaps(img, w, h, fmt, filter)
    assert hr == 0
    return np.concatenate([oracle.compress(chain[off:off + sl], lw, lh, fmt, df)[1] for (off, lw, lh, _, sl) in F.mip_chain_layout(fmt, w, h, 0)[0]])


def reference_exact(fmt, dfmt, df):
    """the composed reference calls are bit-exact here: a BC1-BC5 target, and no sRGB (powf) step in the decompress, the mips or
    the compression"""
    return (df not in (94, 95, 96, 97, 98, 99) and dfmt not in (29, 91) and not S.powf_direction(0, fmt, dfmt)
            and not S.powf_direction(0, dfmt, df))


def test_every_bc_source_every_filter(oracle):
    """All 14 BC formats with decompressFormat 0 and one explicit format, into BC1 / BC3 / BC4 / BC7 (and BC6H from BC6H), with
    filters 0 / BOX / LINEAR / CUBIC / TRIANGLE / POINT, two items at 64 x 16 and at 37 x 22: bit for bit decompress ->
    mipmaps_compress_ex, and for BC1-BC5 targets without a powf step the reference's Decompress -> GenerateMipMaps -> Compress."""
    bad, total, refs = [], 0, 0
    for fmt in BC:
        rng = np.random.default_rng(fmt)
        targets = (71, 77, 80, 98) + ((95,) if fmt in HDR else ())
        for (w, h) in ((64, 16), (37, 22)):
            bases = [bc_base(fmt, w, h, rng) for _ in range(2)]
            for asked in (0, EXPLICIT[fmt]):
                dfmt = asked or DEFAULT[fmt]
                for fl in FILTERS:
                    for df in targets:
                        ctx = "%d -> %d (asked %d) %dx%d filter %#x -> %d" % (fmt, dfmt, asked, w, h, fl, df)
                        hr, outs = from_call(bases, w, h, fmt, df, capi.chain_source(asked), fl)
                        hr_sep, want = separate(bases, w, h, fmt, df, dfmt, (w, h), 0, fl)
                        if hr != hr_sep:
                            bad.append("%s: hr %#x != separate %#x" % (ctx, hr, hr_sep))
                            continue
                        if hr:
                            assert fl == BOX and (w, h) == (37, 22) and hr == F.E_FAIL, (ctx, hex(hr))
                            continue
                        for i in range(2):
                            total += 1
                            if not np.array_equal(outs[i], want[i]):
                                bad.append("%s item %d != separate calls" % (ctx, i))
                            elif reference_exact(fmt, dfmt, df):
                                refs += 1
                                if not np.array_equal(outs[i], reference(oracle, bases[i], w, h, fmt, df, dfmt, (w, h), 0, fl)):
                                    bad.append("%s item %d != reference" % (ctx, i))
    assert not bad, "%d of %d differ; first: %s" % (len(bad), total, "; ".join(bad[:6]))
    assert refs > 0


# (base format, base size, target size, resize filter, mip filter)
RESIZES = [
    (28, (64, 32), (32, 16), 0, 0),                  # 2:1, filter 0 (BOX)
    (77, (64, 32), (32, 16), 0, 0),
    (28, (96, 48), (32, 16), LINEAR, 0),             # 3:1
    (77, (96, 48), (32, 16), LINEAR, LINEAR),
    (28, (16, 16), (48, 48), CUBIC, 0),              # 1:3
    (71, (16, 16), (48, 48), CUBIC, CUBIC),
    (28, (100, 60), (37, 91), TRIANGLE, 0),          # non-square, both ways
    (98, (100, 60), (37, 91), TRIANGLE, TRIANGLE),
    (28, (64, 40), (20, 30), POINT, POINT),
    (80, (64, 40), (20, 30), POINT, 0),
    (28, (256, 256), (16, 8), LINEAR, BOX),          # a chain shorter than the base's
    (77, (256, 256), (16, 8), CUBIC, 0),
]


@pytest.mark.parametrize("fmt,size,to,rf,fl", RESIZES)
def test_resize_cases(oracle, fmt, size, to, rf, fl):
    """Each equals resize -> mipmaps_compress_ex (decompress first for a BC base), and for an RGBA8 base into BC1 / BC3 the
    reference's Resize -> GenerateMipMaps -> Compress."""
    rng = np.random.default_rng(size[0] + to[0])
    w, h = size
    bases = [bc_base(fmt, w, h, rng) if fmt in F.BLOCK_BYTES else alpha_image(28, w, h, rng) for _ in range(2)]
    dfmt = DEFAULT.get(fmt, fmt)
    for df in (71, 77, 98):
        hr, outs = from_call(bases, w, h, fmt, df, capi.chain_source(0, to[0], to[1], rf), fl)
        assert hr == 0, (hex(hr), capi.last_error())
        hr, want = separate(bases, w, h, fmt, df, dfmt, to, rf, fl)
        assert hr == 0
        for i in range(2):
            assert np.array_equal(outs[i], want[i]), (fmt, size, to, rf, fl, df, i)
            if fmt == 28 and df != 98:
                assert np.array_equal(outs[i], reference(oracle, bases[i], w, h, fmt, df, dfmt, to, rf, fl)), (fmt, size, to, df, i)


def test_texconv_full_sequence():
    """A BC3 base -> Resize -> GenerateMipMaps -> coverage 0.5 -> premultiply -> BC7 equals the six separate calls."""
    rng = np.random.default_rng(5)
    w, h, to = 96, 64, (40, 24)
    bases = [bc_base(77, w, h, rng) for _ in range(3)]
    hr, outs = from_call(bases, w, h, 77, 98, capi.chain_source(0, to[0], to[1], LINEAR), 0, capi.chain_steps(0.5, True, 0))
    assert hr == 0, (hex(hr), capi.last_error())
    dec = capi.decompress_images(bases, [(w, h)] * 3, 77, 28)
    res = capi.resize_images(dec, w, h, 28, to[0], to[1], LINEAR)
    chains, layout = separate_chains(res, to[0], to[1], 28, 0, 0.5, 0)
    for i in range(3):
        assert np.array_equal(outs[i], compress_chain(chains[i], layout, 28, 98)), i


def from_chunks(fmt, w, h, dfmt, to, df, items, extra=0):
    """run_staged's chunks of a mipmaps_compress_from call: per item the base (at its row pitch), the decompressed image when a
    resize follows, the chain (level 0 at compute_pitch) and the blocks, each on a 256-byte boundary"""
    row, sl = F.compute_pitch(fmt, w, h)
    b = SC.pad256((row + extra) * (sl // row))
    if fmt in F.BLOCK_BYTES and to != (w, h):
        b += SC.pad256(F.compute_pitch(dfmt, w, h)[1])
    for (_, lw, lh, _, lsl) in F.mip_chain_layout(dfmt, to[0], to[1], 0)[0]:
        b += SC.pad256(lsl) + SC.pad256(F.compute_pitch(df, lw, lh)[1])
    return SC.group_chunks([b] * items, SC.ITEM_CHUNK)


@pytest.mark.parametrize("fmt,size,to,rf,df,items,extras,nchunks", [
    (77, (1024, 1024), (1024, 1024), 0, 71, 12, (0, 16, 48), 2),           # eleven items per chunk, then one
    (98, (4096, 4096), (4096, 4096), 0, 71, 2, (0, 32), 2),                # each base fills a chunk alone
    (71, (1024, 1024), (768, 512), CUBIC, 77, 16, (8, 0, 24), 2),          # with the decompressed image in the buffer
    (28, (1024, 1024), (512, 512), 0, 77, 24, (4, 0, 132), 2)])            # an uncompressed base resized
def test_arrays_over_chunks(fmt, size, to, rf, df, items, extras, nchunks):
    """Arrays over several 80 MiB chunks, bases that fill a chunk alone and base row pitches wider than tight: every item equals
    the separate calls."""
    w, h = size
    ex = [extras[i % len(extras)] for i in range(items)]
    dfmt = DEFAULT.get(fmt, fmt)
    chunks = from_chunks(fmt, w, h, dfmt, to, df, items, max(ex))
    assert len(chunks) == nchunks, [len(c) for c in chunks]
    rng = np.random.default_rng(items)
    uniq = [bc_base(fmt, w, h, rng) if fmt in F.BLOCK_BYTES else alpha_image(28, w, h, rng) for _ in range(min(items, 3))]
    bases = [uniq[i % len(uniq)] for i in range(items)]
    hr, outs = from_call(bases, w, h, fmt, df, capi.chain_source(0, to[0], to[1], rf), 0, None, ex)
    assert hr == 0, (hex(hr), capi.last_error())
    hr, want = separate(uniq, w, h, fmt, df, dfmt, to, rf, 0)
    assert hr == 0
    for i in range(items):
        assert np.array_equal(outs[i], want[i % len(uniq)]), (fmt, size, to, i)


@pytest.mark.parametrize("to,rf", [((1024, 1024), 0), ((512, 256), LINEAR)])
def test_routes(to, rf):
    """The kernel families of one call are exactly the separate calls' families, with one decompress launch per chunk."""
    w = h = 1024
    items = 12
    rng = np.random.default_rng(3)
    bases = [bc_base(77, w, h, rng) for _ in range(items)]
    chunks = from_chunks(77, w, h, 28, to, 71, items)
    (hr, outs), ran = launches(from_call, bases, w, h, 77, 71, capi.chain_source(0, to[0], to[1], rf), 0)
    assert hr == 0
    dec = sum(n for k, n in ran.items() if family(k) == "k_decompress")
    assert dec == len(chunks), (ran, len(chunks))
    sep = set()
    imgs, ran_d = launches(capi.decompress_images, bases, [(w, h)] * items, 77, 28)
    sep |= set(ran_d)
    if to != (w, h):
        imgs, ran_r = launches(capi.resize_images, imgs, w, h, 28, to[0], to[1], rf)
        sep |= set(ran_r)
    _, ran_m = launches(capi.mipmaps_compress, imgs, to[0], to[1], 28, 71, 0)
    sep |= set(ran_m)
    assert {family(k) for k in ran} == {family(k) for k in sep}, (sorted(ran), sorted(sep))


def test_sharded_equals_one_device():
    """With every GPU initialised, the call shards items over the devices and equals one device's result."""
    n = L.dxb200_device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    rng = np.random.default_rng(9)
    bases = [bc_base(77, 256, 256, rng) for _ in range(4 * n)]
    src = capi.chain_source(0, 128, 96, LINEAR)
    hr, one = from_call(bases, 256, 256, 77, 98, src, 0, capi.chain_steps(0.5, True))
    assert hr == 0
    capi.init_devices(list(range(n)))
    try:
        hr, many = from_call(bases, 256, 256, 77, 98, src, 0, capi.chain_steps(0.5, True))
    finally:
        L.dxb200_shutdown()
        assert L.dxb200_init(0) == 0
    assert hr == 0
    for a, b in zip(one, many):
        assert np.array_equal(a, b)


def test_no_op_source_is_ex():
    """source == NULL, a source of the base's own size (any filter) and a decompress format on an uncompressed base are
    byte-identical to mipmaps_compress_ex, also at row pitches wider than tight."""
    rng = np.random.default_rng(17)
    w, h = 80, 48
    bases = [alpha_image(28, w, h, rng) for _ in range(3)]
    steps = capi.chain_steps(0.5, True)
    want = capi.mipmaps_compress(bases, w, h, 28, 77, 0, steps=steps)
    for source in (None, capi.chain_source(), capi.chain_source(0, w, h, CUBIC), capi.chain_source(31, 0, 0, BOX)):
        for extras in (None, [4, 0, 64]):
            hr, got = from_call(bases, w, h, 28, 77, source, 0, steps, extras)
            assert hr == 0
            for a, b in zip(got, want):
                assert np.array_equal(a, b), (source, extras)
