"""GPU suite: dxb200_mipmaps_convert_from, texconv's path to an uncompressed target (Decompress -> Resize -> swizzle -> Convert ->
colour key / invert Y / reconstruct Z -> GenerateMipMaps -> [coverage] -> [premultiply] -> IsAlphaAllOpaque) with every intermediate
kept in device memory.

Every chain equals the separate library calls byte for byte, every level of every item, and so does the alpha-opaque answer.  Item
0 also equals the reference's composed calls (tests/cpp/channel_steps_probe.cpp for the channel steps), bit for bit, or within one
code where an sRGB (powf) step runs.  Each chunk runs one Convert launch on the kernel dxb200_convert takes, none when the formats
match, the channel-step launches that are enabled and no compress kernel."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import alpha_opaque_lib as AO, channel_steps_lib as CS
from tests import staging_cases as SC
from tests.test_cpu_channel_steps import _texconv_pick
from tests.test_gpu_chain_steps import alpha_image, launches
from tests.test_gpu_channel_steps import _bases as channel_bases
from tests.test_gpu_mipmaps_compress_from import DEFAULT, bc_base

pytestmark = pytest.mark.gpu
L = capi.lib
LINEAR, CUBIC = F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC
CONVERT = ("k_convert", "k_convert_vec", "k_convert_diffuse")


@pytest.fixture(autouse=True)
def one_device():
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0


@pytest.fixture(scope="module")
def probe(tmp_path_factory, oracle):
    return CS.Probe(tmp_path_factory.mktemp("convert_from_ref"))


def split(ch):
    """(the swizzle and masks, the later steps) of channel-steps kwargs, each None when nothing in it is enabled"""
    ch = ch or {}
    pre = {k: ch[k] for k in ("swizzle", "zero_mask", "one_mask") if k in ch}
    later = {k: ch[k] for k in ("color_key", "invert_y", "reconstruct_z") if k in ch}
    on_pre = tuple(pre.get("swizzle", (0, 1, 2, 3))) != (0, 1, 2, 3) or pre.get("zero_mask") or pre.get("one_mask")
    on_later = later.get("color_key") is not None or later.get("invert_y") or later.get("reconstruct_z")
    return (pre if on_pre else None), (later if on_later else None)


def front_format(bf, source, ch):
    """level 0's format before the Convert: the decompress format texconv picks for a BC base (source given), else the base's"""
    if bf not in F.BLOCK_BYTES or source is None:
        return bf
    return source.get("decompress_format") or _texconv_pick(bf, CS.steps(**(ch or {}))) or DEFAULT[bf]


def levels_of(fmt, w, h):
    return F.mip_chain_layout(fmt, w, h, 0)[0]


def separate(bases, w, h, bf, source, ch, df, cf, thr, filt, steps):
    """the separate library calls of the sequence; (chains, alpha-opaque answer, the Convert's kernels)"""
    fmt, n = front_format(bf, source, ch), len(bases)
    imgs, lw, lh = bases, w, h
    if bf in F.BLOCK_BYTES:
        imgs = capi.decompress_images(bases, [(w, h)] * n, bf, fmt)
    if source and source.get("width"):
        lw, lh = source["width"], source["height"]
        imgs = capi.resize_images(imgs, w, h, fmt, lw, lh, source.get("resize_filter", 0))
    pre, later = split(ch)
    if pre:
        imgs = capi.apply_channel_steps(imgs, lw, lh, fmt, CS.steps(**pre))
    ran = {}
    if fmt != df:
        imgs, ran = launches(capi.convert_images, imgs, [(lw, lh)] * n, fmt, df, cf, thr)
    if later:
        imgs = capi.apply_channel_steps(imgs, lw, lh, df, CS.steps(**later))
    chains = capi.generate_mipmaps_images(imgs, lw, lh, df, filt, 0)
    layout = levels_of(df, lw, lh)
    if steps is not None and steps.alphaReference > 0:
        chains = [capi.scale_mipmaps_alpha_for_coverage(c, lw, lh, df, steps.alphaReference) for c in chains]
    if steps is not None and steps.premultiply:
        sizes = [(a, b) for (_, a, b, _, _) in layout]
        chains = [np.concatenate(capi.premultiply_alpha_images([c[o:o + s] for (o, _, _, _, s) in layout], sizes, df, steps.pmalphaFlags))
                  for c in chains]
    opaque = all(capi.is_alpha_all_opaque([c[o:o + s] for c in chains], a, b, df) for (o, a, b, _, s) in layout)
    return chains, opaque, {k: v for k, v in ran.items() if k in CONVERT}


def reference(oracle, probe, base, w, h, bf, source, ch, df, cf, thr, filt, steps):
    """the reference's composed calls on item 0: its chain"""
    fmt = front_format(bf, source, ch)
    img, lw, lh = base, w, h
    if bf in F.BLOCK_BYTES:
        hr, img = oracle.decompress(base, w, h, bf, fmt)
        assert hr == 0
    if source and source.get("width"):
        lw, lh = source["width"], source["height"]
        hr, img = oracle.resize(img, w, h, fmt, lw, lh, source.get("resize_filter", 0))
        assert hr == 0
    pre, later = split(ch)
    if pre:
        img = probe.apply(fmt, lw, lh, [img], CS.steps(**pre))[0]
    if fmt != df:
        hr, img = oracle.convert(img, lw, lh, fmt, df, cf, thr)
        assert hr == 0
    if later:
        img = probe.apply(df, lw, lh, [img], CS.steps(**later))[0]
    if steps is not None and steps.alphaReference > 0:
        hr, _, chain = oracle.mips_alpha_coverage(img, lw, lh, df, steps.alphaReference, filt)
    else:
        hr, chain = oracle.generate_mipmaps(img, lw, lh, df, filt)
    assert hr == 0
    if steps is not None and steps.premultiply:
        parts = []
        for (o, a, b, _, s) in levels_of(df, lw, lh):
            hr, p = oracle.premultiply_alpha(chain[o:o + s], a, b, df, steps.pmalphaFlags)
            assert hr == 0
            parts.append(p)
        chain = np.concatenate(parts)
    return chain


def make_bases(kind, bf, w, h, items, seed):
    rng = np.random.default_rng(seed)
    if kind in ("bc5", "bc5s"):
        return channel_bases(kind, w, h, items)
    if bf in F.BLOCK_BYTES:
        return [bc_base(bf, w, h, rng) for _ in range(items)]
    return [alpha_image(bf, w, h, rng) for _ in range(items)]


# (name, base kind, base fmt, items, w, h, source kwargs (None: NULL), channel-steps kwargs, dst fmt, convert filter, threshold,
#  mip filter, chain steps, codes the reference may differ by)
SEQUENCES = [
    ("RGBA32F -> RGBA16F, CUBIC chains", "alpha", 2, 3, 64, 48, None, None, 10, 0, 0.5, CUBIC, None, 0),
    ("RGBA32F -> R11G11B10_FLOAT", "alpha", 2, 2, 40, 24, None, None, 26, 0, 0.5, 0, None, 0),
    ("BC3 -> BGRA8, coverage 0.5 + premultiply", "bc", 77, 3, 64, 64, dict(), None, 87, 0, 0.5, 0, capi.chain_steps(0.5, True), 0),
    ("BC7 -> RGBA8_SRGB with TEX_FILTER_SRGB", "bc", 98, 2, 64, 32, dict(), None, 29, F.TEX_FILTER_SRGB, 0.5, 0, None, 1),
    ("BC5_UNORM swizzle + reconstruct Z -> RGBA8 (no Convert)", "bc5", 83, 3, 64, 64, dict(), dict(swizzle=(1, 0, 2, 3), reconstruct_z=True),
     28, 0, 0.5, 0, None, 0),
    ("BC5_SNORM invert Y -> R16G16_SNORM", "bc5s", 84, 2, 64, 64, dict(), dict(invert_y=True), 37, 0, 0.5, 0, None, 0),
    ("RGBA8 swizzle -> B4G4R4A4 + colour key", "alpha", 28, 3, 48, 32, None, dict(swizzle=(2, 1, 0, 3), color_key=0x000000), 115, 0, 0.5, 0,
     None, 0),
    ("RGBA8 -> B5G5R5A1 at threshold 0.3", "alpha", 28, 2, 64, 64, None, None, 86, 0, 0.3, 0, None, 0),
    ("RGBA32F -> RGBA8 ordered dither", "alpha", 2, 2, 61, 37, None, None, 28, F.TEX_FILTER_DITHER, 0.5, 0, None, 0),
    ("RGBA32F -> RGBA8 error diffusion", "alpha", 2, 2, 61, 37, None, None, 28, F.TEX_FILTER_DITHER_DIFFUSION, 0.5, 0, None, 0),
    ("RGBA8 1000x600 -> 512x512 LINEAR -> RGBA16F", "alpha", 28, 2, 1000, 600, dict(width=512, height=512, resize_filter=LINEAR), None, 10,
     0, 0.5, 0, None, 0),
]


@pytest.mark.parametrize("seq", SEQUENCES, ids=[s[0] for s in SEQUENCES])
def test_equals_separate_calls_and_reference(oracle, probe, seq):
    name, kind, bf, items, w, h, source, ch, df, cf, thr, filt, steps, codes = seq
    bases = make_bases(kind, bf, w, h, items, len(name))
    src = capi.chain_source(**source) if source is not None else None
    chs = CS.steps(**ch) if ch is not None else None
    (outs, opaque), ran = launches(capi.mipmaps_convert_from, bases, w, h, bf, df, src, chs, cf, thr, filt, 0, steps)
    want, want_opaque, conv = separate(bases, w, h, bf, source, ch, df, cf, thr, filt, steps)
    for i, (a, b) in enumerate(zip(outs, want)):
        assert np.array_equal(a, b), (name, i)
    assert opaque == want_opaque, name
    assert not any(k.startswith("k_compress") for k in ran), (name, ran)
    # one chunk: the Convert's kernel is the one dxb200_convert took, once
    pre, later = split(ch)
    scan = 1 if df in AO.PIXEL_FORMATS else 0
    if conv:
        assert set(conv) <= set(ran) and all(ran[k] >= 1 for k in conv), (name, ran, conv)
    steps_launches = (1 if pre else 0) + (1 if later else 0) if conv else (1 if pre or later else 0)
    assert sum(ran.get(k, 0) for k in CONVERT) == (1 if conv else 0) + steps_launches + scan, (name, ran)
    lw, lh = (source["width"], source["height"]) if source and source.get("width") else (w, h)
    chain = reference(oracle, probe, bases[0], w, h, bf, source, ch, df, cf, thr, filt, steps)
    if codes:
        d = np.abs(outs[0].astype(np.int16) - chain.astype(np.int16))
        assert d.max() <= codes, (name, int(d.max()))
    else:
        assert np.array_equal(outs[0], chain), (name, int(np.count_nonzero(outs[0] != chain)))


def chunks_of(bf, w, h, df, items, scan):
    """run_staged's chunks of a call without front steps: per item the base, the chain at tight pitches and the alpha word"""
    b = SC.pad256(F.compute_pitch(bf, w, h)[1]) + sum(SC.pad256(s) for (_, _, _, _, s) in levels_of(df, w, h)) + (256 if scan else 0)
    return SC.group_chunks([b] * items, SC.ITEM_CHUNK)


@pytest.mark.parametrize("bf,df,cf,ch", [
    (2, 10, 0, None),                                              # k_convert_vec, the scan on k_convert
    (2, 28, F.TEX_FILTER_DITHER, dict(swizzle=(2, 1, 0, 3))),      # k_convert, the swizzle before it
    (28, 85, 0, dict(invert_y=True)),                               # no alpha, no scan; invert Y after the Convert
    (10, 10, 0, dict(swizzle=(1, 0, 2, 3), invert_y=True)),         # no Convert: one launch of both steps
    (10, 10, 0, None)])                                             # no Convert, no step
def test_arrays_over_chunks_and_launches(bf, df, cf, ch):
    """Arrays of 1024^2 images over several 80 MiB chunks: every item equals the separate calls, and each chunk runs exactly one
    Convert launch on the kernel dxb200_convert takes (none when the formats match), the enabled channel-step launches, one scan
    and no compress kernel."""
    w = h = 1024
    items, scan = 7, df in AO.PIXEL_FORMATS
    while len(chunks_of(bf, w, h, df, items, scan)) < 2:
        items += 6
    chunks = chunks_of(bf, w, h, df, items, scan)
    rng = np.random.default_rng(bf + df)
    uniq = [alpha_image(bf, w, h, rng) for _ in range(2)]
    bases = [uniq[i % 2] for i in range(items)]
    chs = CS.steps(**ch) if ch is not None else None
    (outs, opaque), ran = launches(capi.mipmaps_convert_from, bases, w, h, bf, df, None, chs, cf, 0.5, 0, 0, None)
    want, want_opaque, conv = separate(uniq, w, h, bf, None, ch, df, cf, 0.5, 0, None)
    for i in range(items):
        assert np.array_equal(outs[i], want[i % 2]), i
    assert opaque == want_opaque
    assert not any(k.startswith("k_compress") for k in ran), ran
    n = len(chunks)
    pre, later = split(ch)
    per_chunk = (1 if bf != df else 0) + ((1 if pre else 0) + (1 if later else 0) if bf != df else (1 if pre or later else 0)) + (1 if scan else 0)
    assert sum(ran.get(k, 0) for k in CONVERT) == n * per_chunk, (ran, n)
    if bf != df:
        (k,) = conv.keys()
        assert ran[k] >= n, (ran, conv)
        if k == "k_convert_vec":
            assert ran.get("k_convert", 0) == n * (per_chunk - 1), ran
    else:
        assert "k_convert_vec" not in ran and "k_convert_diffuse" not in ran


def test_sharded_equals_one_device():
    """With every GPU initialised, the call shards items over the devices and equals one device's result."""
    n = L.dxb200_device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    rng = np.random.default_rng(5)
    bases = [bc_base(77, 256, 256, rng) for _ in range(4 * n)]
    src = capi.chain_source(0, 128, 96, LINEAR)
    chs = CS.steps(swizzle=(2, 1, 0, 3), invert_y=True)
    one, o1 = capi.mipmaps_convert_from(bases, 256, 256, 77, 10, src, chs, 0, 0.5, 0, 0, capi.chain_steps(0.5, True))
    capi.init_devices(list(range(n)))
    try:
        many, o2 = capi.mipmaps_convert_from(bases, 256, 256, 77, 10, src, chs, 0, 0.5, 0, 0, capi.chain_steps(0.5, True))
    finally:
        L.dxb200_shutdown()
        assert L.dxb200_init(0) == 0
    assert o1 == o2
    for a, b in zip(one, many):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("bf,ch", [(2, dict(invert_y=True)), (10, None), (10, dict(color_key=0x4080C0)), (10, dict(swizzle=(2, 1, 0, 3)))],
                         ids=["convert", "copy", "copy_color_key", "copy_swizzle"])
def test_caller_pitches_and_no_opaque_word(bf, ch):
    """dst levels at row pitches wider than tight and alphaAllOpaque == NULL give the same pixels as the separate calls; a base at a
    wider row pitch is read at that pitch, also when no step writes level 0 and the base is copied there in device memory"""
    w, h, df = 40, 24, 10
    bpp = F.BYTES_PER_PIXEL[bf]
    rng = np.random.default_rng(11)
    bases = [alpha_image(bf, w, h, rng) for _ in range(2)]
    chs = CS.steps(**ch) if ch is not None else None
    want, _ = capi.mipmaps_convert_from(bases, w, h, bf, df, None, chs, 0, 0.5, CUBIC, 0, None)
    sep, _, _ = separate(bases, w, h, bf, None, ch, df, 0, 0.5, CUBIC, None)
    for a, b in zip(want, sep):
        assert np.array_equal(a, b)
    layout = levels_of(df, w, h)
    brow = w * bpp + 32
    held = []
    for b in bases:
        a = np.full((h, brow), 0x5A, np.uint8)
        a[:, :w * bpp] = np.ascontiguousarray(b).view(np.uint8).reshape(h, w * bpp)
        held.append(a)
    outs = []
    for _ in bases:
        outs.append([np.full((lh, lw * 8 + 24), 0xA5, np.uint8) for (_, lw, lh, _, _) in layout])
    s = capi.images([capi.Image(w, h, bf, brow, brow * h, a.ctypes.data) for a in held])
    d = capi.images([capi.Image(lw, lh, df, o.shape[1], o.nbytes, o.ctypes.data) for item in outs for o, (_, lw, lh, _, _) in zip(item, layout)])
    hr = L.dxb200_mipmaps_convert_from(s, 2, None, C.byref(chs) if chs is not None else None, df, 0, 0.5, len(layout), CUBIC, None, d, None)
    assert F.hr_u32(hr) == 0, capi.last_error()
    for i, item in enumerate(outs):
        for o, (off, lw, lh, _, sl) in zip(item, layout):
            assert np.array_equal(o[:, :lw * 8].reshape(-1), want[i][off:off + sl]), (i, lw)
