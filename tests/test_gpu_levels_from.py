"""GPU suite: dxb200_levels_from, texconv on textures that keep their own levels (Decompress -> [Resize] -> swizzle -> Convert ->
colour key / invert Y / reconstruct Z -> [premultiply] -> [Compress] -> IsAlphaAllOpaque over every level), with every intermediate
kept in device memory.

Every level of every item equals the separate library calls over all the levels as one array, byte for byte, and so does the
alpha-opaque answer.  Item 0 also equals the reference's composed calls level by level (tests/cpp/channel_steps_probe.cpp for the
channel steps) for BC1-BC5 and uncompressed targets, bit for bit, or within one code where an sRGB (powf) step runs; the alpha
answer equals the reference's IsAlphaAllOpaque.  Each chunk runs each enabled step as one launch over all its levels, no mip or
coverage kernel, and a BC chain that passes through runs no decompress or compress kernel."""
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
from tests.test_gpu_mipmaps_convert_from import split

pytestmark = pytest.mark.gpu
L = capi.lib
LINEAR, CUBIC = F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC
NOT_IN_LEVELS = ("k_mip", "k_alpha_coverage", "k_scale_alpha")


@pytest.fixture(autouse=True)
def one_device():
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0


@pytest.fixture(scope="module")
def probe(tmp_path_factory, oracle):
    return CS.Probe(tmp_path_factory.mktemp("levels_from_ref"))


@pytest.fixture(scope="module")
def ref_opaque(tmp_path_factory, oracle):
    return AO.Probe(tmp_path_factory.mktemp("levels_from_opaque"), True)


def chain_sizes(w, h, levels=0):
    return [(lw, lh) for (_, lw, lh, _, _) in F.mip_chain_layout(28, w, h, levels)[0]]


def working_format(bf, source, ch):
    """the format the front steps leave: the decompress format texconv picks for a BC base, else the base's"""
    if bf not in F.BLOCK_BYTES:
        return bf
    return (source or {}).get("decompress_format") or _texconv_pick(bf, CS.steps(**(ch or {}))) or DEFAULT[bf]


def passes_through(bf, df, source, ch, steps):
    resize = bool(source and source.get("width"))
    return bf in F.BLOCK_BYTES and bf == df and not any(split(ch)) and not (steps is not None and steps.premultiply) and not resize


def _tight(arrays, sizes, fmt):
    return capi.images([capi.Image(w, h, fmt, *F.compute_pitch(fmt, w, h), np.ascontiguousarray(a).ctypes.data)
                        for a, (w, h) in zip(arrays, sizes)])


def steps_images(arrays, sizes, fmt, s):
    """dxb200_apply_channel_steps of host images of different sizes in one call"""
    arrays = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in arrays]
    outs = [np.zeros_like(a) for a in arrays]
    hr = L.dxb200_apply_channel_steps(_tight(arrays, sizes, fmt), len(arrays), C.byref(s), _tight(outs, sizes, fmt))
    assert hr == 0, capi.last_error()
    return outs


def opaque_images(arrays, sizes, fmt):
    """dxb200_is_alpha_all_opaque of host images of different sizes in one call"""
    arrays = [np.ascontiguousarray(a) for a in arrays]
    opaque = C.c_int32(-1)
    assert L.dxb200_is_alpha_all_opaque(_tight(arrays, sizes, fmt), len(arrays), C.byref(opaque)) == 0, capi.last_error()
    return opaque.value == 1


def separate(bases, sizes, bf, source, ch, df, cf, flags, thr, steps):
    """the separate library calls of the sequence, each over all items * levels images as one array: (outs[i][l], alpha answer)"""
    n, levels = len(bases), len(sizes)
    imgs, szs = [a for item in bases for a in item], sizes * n
    if passes_through(bf, df, source, ch, steps):
        out = imgs
    else:
        fmt = working_format(bf, source, ch)
        if bf in F.BLOCK_BYTES:
            imgs = capi.decompress_images(imgs, szs, bf, fmt)
        if source and source.get("width"):
            (w, h), = sizes
            szs = [(source["width"], source["height"])] * n
            imgs = capi.resize_images(imgs, w, h, fmt, source["width"], source["height"], source.get("resize_filter", 0))
        pre, later = split(ch)
        if pre:
            imgs = steps_images(imgs, szs, fmt, CS.steps(**pre))
        if df not in F.BLOCK_BYTES and fmt != df:
            imgs, fmt = capi.convert_images(imgs, szs, fmt, df, cf, thr), df
        if later:
            imgs = steps_images(imgs, szs, fmt, CS.steps(**later))
        if steps is not None and steps.premultiply:
            imgs = capi.premultiply_alpha_images(imgs, szs, fmt, steps.pmalphaFlags)
        out = capi.compress_images(imgs, szs, fmt, df, flags, thr) if df in F.BLOCK_BYTES else imgs
    out = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in out]
    return [out[i * levels:(i + 1) * levels] for i in range(n)], opaque_images(out, szs, df)


def reference(oracle, probe, item, sizes, bf, source, ch, df, cf, flags, thr, steps):
    """the reference's composed calls on one item, level by level: its levels"""
    if passes_through(bf, df, source, ch, steps):
        return item
    fmt0, out = working_format(bf, source, ch), []
    for img, (w, h) in zip(item, sizes):
        fmt = fmt0
        if bf in F.BLOCK_BYTES:
            hr, img = oracle.decompress(img, w, h, bf, fmt)
            assert hr == 0
        if source and source.get("width"):
            hr, img = oracle.resize(img, w, h, fmt, source["width"], source["height"], source.get("resize_filter", 0))
            assert hr == 0
            w, h = source["width"], source["height"]
        pre, later = split(ch)
        if pre:
            img = probe.apply(fmt, w, h, [img], CS.steps(**pre))[0]
        if df not in F.BLOCK_BYTES and fmt != df:
            hr, img = oracle.convert(img, w, h, fmt, df, cf, thr)
            assert hr == 0
            fmt = df
        if later:
            img = probe.apply(fmt, w, h, [img], CS.steps(**later))[0]
        if steps is not None and steps.premultiply:
            hr, img = oracle.premultiply_alpha(img, w, h, fmt, steps.pmalphaFlags)
            assert hr == 0
        if df in F.BLOCK_BYTES:
            hr, img = oracle.compress(img, w, h, fmt, df, flags, thr)
            assert hr == 0
        out.append(np.ascontiguousarray(img).view(np.uint8).reshape(-1))
    return out


def make_chains(kind, bf, sizes, items, seed):
    """items chains of bf, one image per size"""
    rng = np.random.default_rng(seed)
    if kind in ("bc5", "bc5s"):
        per = [channel_bases(kind, w, h, items) for (w, h) in sizes]
        return [[per[l][i] for l in range(len(sizes))] for i in range(items)]
    if bf in F.BLOCK_BYTES:
        return [[bc_base(bf, w, h, rng) for (w, h) in sizes] for _ in range(items)]
    return [[alpha_image(bf, w, h, rng) for (w, h) in sizes] for _ in range(items)]


PM = capi.chain_steps(0.0, True)
C32 = chain_sizes(32, 32)                   # 32x32 .. 2x2, 1x1
C40 = chain_sizes(40, 24)                   # partial blocks at every level below 4x4
# (name, base kind, base fmt, items, sizes, channel-steps kwargs, dst fmt, convert filter, compress flags, chain steps,
#  codes the reference may differ by (None: not compared; the BC6H and BC7 encoders are compared with the separate calls only))
SEQUENCES = [
    ("BC3 -> BC7 + premultiply", "bc", 77, 2, C32, None, 98, 0, 0, PM, None),
    ("BC1 -> BC1_SRGB re-encodes", "bc", 71, 2, C40, None, 72, 0, 0, None, 0),
    ("BC5 invert Y -> BC5", "bc5", 83, 2, C32, dict(invert_y=True), 83, 0, 0, None, 0),
    ("BC5_SNORM reconstruct Z -> R8G8B8A8_SNORM", "bc5s", 84, 2, C32, dict(reconstruct_z=True), 31, 0, 0, None, 0),
    ("BC4 invert Y -> BC4 through RGBA8", "bc", 80, 2, C40, dict(invert_y=True), 80, 0, 0, None, 0),
    ("BC7 -> RGBA8_SRGB", "bc", 98, 2, C40, None, 29, 0, 0, None, 1),
    ("BC3 swizzle + reconstruct Z -> RGBA8 (no Convert)", "bc", 77, 2, C32, dict(swizzle=(1, 0, 2, 3), reconstruct_z=True), 28, 0, 0, None, 0),
    ("RGBA8 swizzle + colour key -> BC3", "alpha", 28, 3, C40, dict(swizzle=(2, 1, 0, 3), color_key=0x000000), 77, 0, 0, None, 0),
    ("RGBA8 premultiply -> BC2", "alpha", 28, 2, C32, None, 74, 0, 0, PM, 0),
    ("RGBA8_SRGB invert Y -> RGBA8", "alpha", 29, 2, C40, dict(invert_y=True), 28, 0, 0, None, 1),
    ("RGBA16F swizzle -> BC5", "alpha", 10, 2, C32, dict(swizzle=(3, 1, 2, 0)), 83, 0, 0, None, 0),
    ("RGBA16F reconstruct Z -> BC6H_UF16", "alpha", 10, 2, C40, dict(reconstruct_z=True), 95, 0, 0, None, None),
    ("RGBA32F -> RGBA8 error diffusion + premultiply", "alpha", 2, 2, C40, None, 28, F.TEX_FILTER_DITHER_DIFFUSION, 0, PM, 0),
    ("RGBA8 swizzle -> B4G4R4A4 + colour key", "alpha", 28, 2, C32, dict(swizzle=(2, 1, 0, 3), color_key=0x000000), 115, 0, 0, None, 0),
    ("RGBA16F -> RGBA16F copied", "alpha", 10, 2, C40, None, 10, 0, 0, None, 0),
    ("BC7 passes through", "bc", 98, 2, C40, None, 98, 0, 0, None, 0),
    ("levels that do not halve: RGBA8 -> RGBA32F", "alpha", 28, 2, [(40, 40), (33, 7), (2, 2), (1, 3)], dict(invert_y=True), 2, 0, 0, None,
     0),
]


@pytest.mark.parametrize("seq", SEQUENCES, ids=[s[0] for s in SEQUENCES])
def test_equals_separate_calls_and_reference(oracle, probe, ref_opaque, seq):
    name, kind, bf, items, sizes, ch, df, cf, flags, steps, codes = seq
    bases = make_chains(kind, bf, sizes, items, len(name))
    chs = CS.steps(**ch) if ch is not None else None
    (outs, opaque), ran = launches(capi.levels_from, bases, sizes, bf, df, None, chs, cf, flags, 0.5, steps)
    want, want_opaque = separate(bases, sizes, bf, None, ch, df, cf, flags, 0.5, steps)
    for i in range(items):
        for l in range(len(sizes)):
            assert np.array_equal(outs[i][l], want[i][l]), (name, i, l)
    assert opaque == want_opaque, name
    assert not any(k.startswith(NOT_IN_LEVELS) for k in ran), (name, ran)
    # one chunk: every step that runs is one launch over all the levels
    if passes_through(bf, df, None, ch, steps):
        assert not any(k.startswith("k_compress") or k == "k_decompress_t" for k in ran), ran
        assert ran.get("k_decompress", 0) == (1 if df in AO.BLOCK_FORMATS else 0), ran      # the alpha scan only
    else:
        assert sum(v for k, v in ran.items() if k.startswith("k_compress")) == (1 if df in F.BLOCK_BYTES else 0), (name, ran)
    if steps is not None and steps.premultiply:
        assert ran.get("k_pmalpha", 0) + ran.get("k_pmalpha_vec", 0) == 1, (name, ran)
    if codes is None:
        return
    chain = reference(oracle, probe, bases[0], sizes, bf, None, ch, df, cf, flags, 0.5, steps)
    for l, (a, b) in enumerate(zip(outs[0], chain)):
        if codes:
            d = np.abs(a.astype(np.int16) - b.astype(np.int16))
            assert d.max() <= codes, (name, l, int(d.max()))
        else:
            assert np.array_equal(a, b), (name, l, int(np.count_nonzero(a != b)))
    if sizes[1:] == [(max(1, sizes[0][0] >> l), max(1, sizes[0][1] >> l)) for l in range(1, len(sizes))]:
        packed = np.concatenate([a for item in outs for a in item])
        assert opaque == ref_opaque.opaque(df, sizes[0][0], sizes[0][1], packed, items, len(sizes)), name


def test_pass_through_is_the_base_and_srgb_twin_reencodes():
    """BC1 -> BC1 keeps the base's bytes with no decompress or compress kernel (and no scan without alphaAllOpaque); BC1 ->
    BC1_UNORM_SRGB decompresses and compresses once per chunk"""
    sizes = C40
    bases = make_chains("bc", 71, sizes, 3, 1)
    flat = [a for item in bases for a in item]
    s = _tight(flat, sizes * 3, 71)
    outs = [np.zeros_like(a) for a in flat]
    d = _tight(outs, sizes * 3, 71)
    before = {k: capi.kernel_launch_count(k) for k in ("k_decompress", "k_decompress_t", "k_compress_bc15", "k_compress_bc15_t")}
    assert L.dxb200_levels_from(s, 3, len(sizes), None, None, 71, 0, 0, 0.5, None, d, None) == 0, capi.last_error()
    assert all(capi.kernel_launch_count(k) == v for k, v in before.items())
    for a, b in zip(outs, flat):
        assert np.array_equal(a, b)
    (twin, _), ran = launches(capi.levels_from, bases, sizes, 71, 72)
    want, _ = separate(bases, sizes, 71, None, None, 72, 0, 0, 0.5, None)
    assert ran.get("k_decompress_t", 0) + ran.get("k_decompress", 0) == 2 and ran.get("k_compress_bc15", 0) + ran.get("k_compress_bc15_t", 0) == 1, ran
    for i in range(3):
        for a, b in zip(twin[i], want[i]):
            assert np.array_equal(a, b)


# (name, base fmt, w, h, source kwargs, channel-steps kwargs, dst fmt, chain steps)
ONE_LEVEL = [
    ("BC3 1000x600 -> 512x256 CUBIC -> BC7 + premultiply", 77, 1000, 600, dict(width=512, height=256, resize_filter=CUBIC), None, 98, PM),
    ("RGBA8 100x60 -> 64x32 swizzle -> BC1", 28, 100, 60, dict(width=64, height=32, resize_filter=LINEAR), dict(swizzle=(2, 1, 0, 3)), 71, None),
    ("BC5 64x64 -> 32x32 invert Y -> R8G8_SNORM", 83, 64, 64, dict(width=32, height=32), dict(invert_y=True), 51, None),
    ("RGBA32F 90x70 -> 45x35 -> RGBA16F + premultiply", 2, 90, 70, dict(width=45, height=35, resize_filter=LINEAR), None, 10, PM),
]


@pytest.mark.parametrize("case", ONE_LEVEL, ids=[c[0] for c in ONE_LEVEL])
def test_one_level_with_resize(case):
    """levels == 1 with a Resize equals the separate calls and level 0 of the generating call with two levels"""
    name, bf, w, h, source, ch, df, steps = case
    kind = "bc5" if bf == 83 else "bc" if bf in F.BLOCK_BYTES else "alpha"
    bases = make_chains(kind, bf, [(w, h)], 3, len(name))
    src, chs = capi.chain_source(**source), CS.steps(**ch) if ch is not None else None
    (outs, opaque), ran = launches(capi.levels_from, bases, [(w, h)], bf, df, src, chs, 0, 0, 0.5, steps)
    want, want_opaque = separate(bases, [(w, h)], bf, source, ch, df, 0, 0, 0.5, steps)
    assert opaque == want_opaque, name
    # the Resize is the one mip-kernel launch (a chain would add one per level), and no coverage kernel runs
    assert sum(v for k, v in ran.items() if k.startswith("k_mip")) == 1, ran
    assert not any(k.startswith(NOT_IN_LEVELS[1:]) for k in ran), ran
    flat = [item[0] for item in bases]
    if df in F.BLOCK_BYTES:
        gen, gen_opaque = capi.mipmaps_compress_from_channels(flat, w, h, bf, df, src, chs, 0, 2, 0, steps)
    else:
        gen, gen_opaque = capi.mipmaps_convert_from(flat, w, h, bf, df, src, chs, 0, 0.5, 0, 2, steps)
    size0 = F.compute_pitch(df, source["width"], source["height"])[1]
    for i in range(3):
        assert np.array_equal(outs[i][0], want[i][0]), (name, i)
        assert np.array_equal(outs[i][0], gen[i][:size0]), (name, i)


def chunks_of(bf, df, sizes, items, front, scan):
    """run_staged's chunks of a call: per item every level of the base, of the working images when a front step writes them and
    the output is compressed, of dst, and the alpha word"""
    b = sum(SC.pad256(F.compute_pitch(bf, w, h)[1]) for (w, h) in sizes) + sum(SC.pad256(F.compute_pitch(df, w, h)[1]) for (w, h) in sizes)
    if front and df in F.BLOCK_BYTES:
        b += sum(SC.pad256(F.compute_pitch(28, w, h)[1]) for (w, h) in sizes)
    return SC.group_chunks([b + (256 if scan else 0)] * items, SC.ITEM_CHUNK)


# (base fmt, dst fmt, channel-steps kwargs, chain steps, {kernel family: launches per chunk})
ARRAYS = [
    (71, 77, dict(invert_y=True), PM, {"k_decompress": 2, "k_convert": 1, "k_pmalpha": 1, "k_compress_bc15": 1}),
    (28, 10, dict(swizzle=(2, 1, 0, 3), color_key=0x102030), None, {"k_convert": 4}),
    (98, 98, None, None, {"k_decompress": 1}),
    (28, 28, None, PM, {"k_pmalpha": 1, "k_convert": 1}),
]


@pytest.mark.parametrize("bf,df,ch,steps,per_chunk", ARRAYS, ids=["bc1_bc3", "rgba8_rgba16f", "bc7_pass", "rgba8_copy_pm"])
def test_arrays_over_chunks_and_launches(bf, df, ch, steps, per_chunk):
    """Arrays of 1024^2 chains (11 levels) over several 80 MiB chunks: every item equals the separate calls, and each chunk runs
    every enabled step as one launch over all its levels (the alpha scan included), no mip or coverage kernel"""
    sizes = chain_sizes(1024, 1024)
    scan = df in AO.PIXEL_FORMATS or df in AO.BLOCK_FORMATS
    front = bf in F.BLOCK_BYTES and not passes_through(bf, df, None, ch, steps)
    items = 8
    while len(chunks_of(bf, df, sizes, items, front, scan)) < 3:
        items += 8
    n = len(chunks_of(bf, df, sizes, items, front, scan))
    uniq = make_chains("bc" if bf in F.BLOCK_BYTES else "alpha", bf, sizes, 2, bf + df)
    chs = CS.steps(**ch) if ch is not None else None
    (outs, opaque), ran = launches(capi.levels_from, [uniq[i % 2] for i in range(items)], sizes, bf, df, None, chs, 0, 0, 0.5, steps)
    want, want_opaque = separate(uniq, sizes, bf, None, ch, df, 0, 0, 0.5, steps)
    for i in range(items):
        for l in range(len(sizes)):
            assert np.array_equal(outs[i][l], want[i % 2][l]), (i, l)
    assert opaque == want_opaque
    assert not any(k.startswith(NOT_IN_LEVELS) for k in ran), ran
    fam = {}
    for k, v in ran.items():
        f = k[:-2] if k.endswith("_t") else k[:-4] if k.endswith("_vec") else k
        fam[f] = fam.get(f, 0) + v
    assert fam == {k: v * n for k, v in per_chunk.items()}, (fam, n)


def test_sharded_equals_one_device():
    """With every GPU initialised, the call shards items over the devices and equals one device's result."""
    n = L.dxb200_device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    bases = make_chains("bc", 77, C32, 4 * n, 5)
    chs = CS.steps(swizzle=(2, 1, 0, 3), invert_y=True)
    one, o1 = capi.levels_from(bases, C32, 77, 98, None, chs, 0, 0, 0.5, PM)
    capi.init_devices(list(range(n)))
    try:
        many, o2 = capi.levels_from(bases, C32, 77, 98, None, chs, 0, 0, 0.5, PM)
    finally:
        L.dxb200_shutdown()
        assert L.dxb200_init(0) == 0
    assert o1 == o2
    for a, b in zip(one, many):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def _held(arrays, sizes, fmt, extra, skew):
    """host copies of `arrays` at levels above 0 with rows `extra` bytes wider than tight, the first pixel `skew` bytes into a
    buffer; (images, buffers, views of the rows)"""
    imgs, held = [], []
    for l, (a, (w, h)) in enumerate(zip(arrays, sizes)):
        row, sl = F.compute_pitch(fmt, w, h)
        rows = sl // row
        e, k = (extra, skew) if l else (0, 0)
        buf = np.full(k + (row + e) * rows, 0x5A, np.uint8)
        view = buf[k:].reshape(rows, row + e)
        view[:, :row] = np.ascontiguousarray(a).view(np.uint8).reshape(rows, row)
        held.append((buf, view, row))
        imgs.append(capi.Image(w, h, fmt, row + e, (row + e) * rows, buf.ctypes.data + k))
    return imgs, held


@pytest.mark.parametrize("bf,df,ch,extra,skew", [
    (28, 77, dict(invert_y=True), 16, 0),       # the base uploaded as the working images, BC dst rows 16 bytes wider
    (28, 10, None, 4, 4),                       # a Convert from a base 4 bytes off
    (71, 28, dict(swizzle=(2, 1, 0, 3)), 16, 0),  # Decompress from wider block rows into wider dst rows
    (28, 28, dict(color_key=0x4080C0), 4, 4),    # the base copied into dst in device memory, both 4 bytes off
    (71, 71, None, 16, 0),                      # a passed-through BC chain at wider block rows
])
def test_caller_pitches(bf, df, ch, extra, skew):
    """base and dst levels above 0 at row pitches wider than tight (and 4 bytes off their buffer's start) give the pixels of the
    tight call, which equals the separate calls"""
    sizes = C40
    bases = make_chains("bc" if bf in F.BLOCK_BYTES else "alpha", bf, sizes, 2, 3)
    chs = CS.steps(**ch) if ch is not None else None
    want, _ = capi.levels_from(bases, sizes, bf, df, None, chs)
    sep, _ = separate(bases, sizes, bf, None, ch, df, 0, 0, 0.5, None)
    for a, b in zip(want, sep):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    src, dst, held_out = [], [], []
    keep = []
    for item in bases:
        imgs, held = _held(item, sizes, bf, extra if bf not in F.BLOCK_BYTES or extra % F.BLOCK_BYTES[bf] == 0 else 0, skew)
        src += imgs
        keep.append(held)
        imgs, held = _held([np.zeros(F.compute_pitch(df, w, h)[1], np.uint8) for (w, h) in sizes], sizes, df, extra, skew if df not in F.BLOCK_BYTES else 0)
        dst += imgs
        held_out.append(held)
    hr = L.dxb200_levels_from(capi.images(src), 2, len(sizes), None, C.byref(chs) if chs is not None else None, df, 0, 0, 0.5, None,
                              capi.images(dst), None)
    assert F.hr_u32(hr) == 0, capi.last_error()
    for i, held in enumerate(held_out):
        for l, (buf, view, row) in enumerate(held):
            assert np.array_equal(view[:, :row].reshape(-1), want[i][l]), (i, l)
