"""GPU suite: texconv's -alpha (demultiply) and -f BC3n / DXT5nm / RXGB steps inside dxb200_mipmaps_compress_from_channels_ex,
dxb200_mipmaps_convert_from_ex and dxb200_levels_from_ex, with every intermediate kept in device memory.

Every level of every item and the alpha answer equal the separate host calls in texconv's order: dxb200_decompress ->
dxb200_premultiply_alpha(REVERSE) -> the call without _ex on the demultiplied base; or the call without _ex into the working format
-> dxb200_apply_channel_steps with the layout's swizzle and masks -> dxb200_compress to BC3.  Item 0 also equals the reference's
composed calls (PremultiplyAlpha REVERSE, Resize, TransformImage through tests/cpp/channel_steps_probe.cpp, GenerateMipMaps,
PremultiplyAlpha, Compress) bit for bit, or within one code where an sRGB step runs into an uncompressed target.  Each chunk runs
exactly one more k_pmalpha* launch for a demultiply and one more k_convert launch for a layout than the call without them."""
import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import channel_steps_lib as CS, oracle_lib
from tests.test_cpu_channel_steps import _texconv_pick
from tests.test_gpu_chain_steps import alpha_image, launches
from tests.test_gpu_channel_steps import _bases as channel_bases
from tests.test_gpu_levels_from import opaque_images, steps_images
from tests.test_gpu_mipmaps_compress_from import DEFAULT, bc_base

pytestmark = pytest.mark.gpu
L = capi.lib
REVERSE = 0x2
RXGB_DDS = 0x80000                  # DDS_FLAGS_FORCE_DXT5_RXGB
LAYOUT = {1: dict(swizzle=(0, 1, 2, 0), zero_mask=0x4, one_mask=0x1), 2: dict(swizzle=(3, 1, 2, 0))}
PM = capi.chain_steps(0.0, True)


@pytest.fixture(autouse=True)
def one_device():
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0


@pytest.fixture(scope="module")
def probe(tmp_path_factory, oracle):
    return CS.Probe(tmp_path_factory.mktemp("texconv_steps_ref"))


def sizes_of(w, h, levels):
    out = []
    for _ in range(levels):
        out.append((w, h))
        w, h = max(1, w >> 1), max(1, h >> 1)
    return out


def working_format(bf, source, ch, layout):
    """the format Decompress writes: the caller's, else texconv's pick for the channel steps and the layout, else the default"""
    if bf not in F.BLOCK_BYTES:
        return bf
    if (source or {}).get("decompress_format"):
        return source["decompress_format"]
    if layout and bf in (80, 81, 83, 84):
        return 31 if bf in (81, 84) else 28
    return _texconv_pick(bf, CS.steps(**(ch or {}))) or DEFAULT[bf]


def make_bases(kind, bf, sizes, items, seed):
    """items lists of one image per size: BC5 normal maps, BC blocks of alpha content, or alpha images"""
    rng = np.random.default_rng(seed)
    if kind in ("bc5", "bc5s"):
        per = [channel_bases(kind, w, h, items) for (w, h) in sizes]
        return [[per[l][i] for l in range(len(sizes))] for i in range(items)]
    if bf in (80, 81):
        return [[capi.compress(alpha_image(28, w, h, rng), w, h, 28, bf) for (w, h) in sizes] for _ in range(items)]
    if bf in F.BLOCK_BYTES:
        return [[bc_base(bf, w, h, rng) for (w, h) in sizes] for _ in range(items)]
    if bf == 24:                    # R10G10B10A2: random codes, two-bit alpha
        return [[oracle_lib.random_image(bf, w, h, rng) for (w, h) in sizes] for _ in range(items)]
    return [[alpha_image(bf, w, h, rng) for (w, h) in sizes] for _ in range(items)]


def one_call(entry, bases, sizes, bf, df, source, ch, steps, ts, levels):
    """(outs[i] = the list of item i's levels, alpha answer) of the _ex call"""
    src = capi.chain_source(**source) if source is not None else None
    chs = CS.steps(**ch) if ch is not None else None
    if entry == "lev":
        return capi.levels_from(bases, sizes, bf, df, src, chs, 0, 0, 0.5, steps, texconv=ts)
    (w, h), flat = sizes[0], [item[0] for item in bases]
    if entry == "gen":
        outs, opaque = capi.mipmaps_compress_from_channels(flat, w, h, bf, df, src, chs, 0, levels, 0, steps, texconv=ts)
    else:
        outs, opaque = capi.mipmaps_convert_from(flat, w, h, bf, df, src, chs, 0, 0.5, 0, levels, steps, texconv=ts)
    ow, oh = (source["width"], source["height"]) if source and source.get("width") else (w, h)
    return [unpack(o, df, ow, oh, levels) for o in outs], opaque


def unpack(packed, fmt, w, h, levels):
    layout, _ = capi.texture_layout(fmt, w, h, 1, levels)
    return [packed[off:off + sl] for (off, _, _, _, sl) in layout]


def separate(entry, bases, sizes, bf, df, source, ch, steps, tk, levels):
    """the separate host calls: (outs[i][l], alpha answer)"""
    n, layout = len(bases), tk.get("bc3_layout", 0)
    fmt = working_format(bf, source, ch, layout)
    source = dict(source) if source is not None else None
    if tk.get("demultiply"):
        flat = [a for item in bases for a in item]
        szs = sizes * n
        if bf in F.BLOCK_BYTES and (entry == "lev" or source is not None):
            flat = capi.decompress_images(flat, szs, bf, fmt)
            bf = fmt
            if source is not None:
                source.pop("decompress_format", None)
        flat = capi.premultiply_alpha_images(flat, szs, bf, REVERSE | tk.get("demultiply_flags", 0))
        bases = [flat[i * len(sizes):(i + 1) * len(sizes)] for i in range(n)]
    if not layout:
        return one_call(entry, bases, sizes, bf, df, source, ch, steps, None, levels)
    if bf in F.BLOCK_BYTES:
        source = dict(source or {}, decompress_format=fmt)
    chains, _ = one_call("conv" if entry == "gen" else entry, bases, sizes, bf, fmt, source, ch, steps, None, levels)
    ow, oh = (source["width"], source["height"]) if source and source.get("width") else sizes[0]
    csz = sizes_of(ow, oh, levels) if entry != "lev" else sizes
    flat = steps_images([a for c in chains for a in c], csz * n, fmt, CS.steps(**LAYOUT[layout]))
    out = capi.compress_images(flat, csz * n, fmt, df)
    out = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in out]
    return [out[i * levels:(i + 1) * levels] for i in range(n)], opaque_images(out, csz * n, df)


def reference(oracle, probe, entry, item, sizes, bf, df, source, ch, steps, tk, levels):
    """the reference's composed calls on one item (GenerateMipMaps with the default filter for a generated chain)"""
    layout = tk.get("bc3_layout", 0)
    fmt = working_format(bf, source, ch, layout)
    imgs = []
    for img, (w, h) in zip(item, sizes):
        if bf in F.BLOCK_BYTES:
            hr, img = oracle.decompress(img, w, h, bf, fmt)
            assert hr == 0
        if tk.get("demultiply"):
            hr, img = oracle.premultiply_alpha(img, w, h, fmt, REVERSE | tk.get("demultiply_flags", 0))
            assert hr == 0
        if source and source.get("width"):
            hr, img = oracle.resize(img, w, h, fmt, source["width"], source["height"], source.get("resize_filter", 0))
            assert hr == 0
            w, h = source["width"], source["height"]
        if ch:
            img = probe.apply(fmt, w, h, [img], CS.steps(**ch))[0]
        imgs.append((np.ascontiguousarray(img).view(np.uint8).reshape(-1), w, h))
    if entry != "lev":
        img, w, h = imgs[0]
        if df not in F.BLOCK_BYTES and df != fmt:
            hr, img = oracle.convert(img, w, h, fmt, df)
            assert hr == 0
            fmt = df
        hr, chain = oracle.generate_mipmaps(img, w, h, fmt, 0, levels)
        assert hr == 0
        imgs = [(a, lw, lh) for a, lw, lh in zip(unpack(chain, fmt, w, h, levels), *zip(*sizes_of(w, h, levels)))]
    elif df not in F.BLOCK_BYTES and df != fmt:
        conv = []
        for img, w, h in imgs:
            hr, img = oracle.convert(img, w, h, fmt, df)
            assert hr == 0
            conv.append((img, w, h))
        imgs, fmt = conv, df
    out = []
    for img, w, h in imgs:
        if steps is not None and steps.premultiply:
            hr, img = oracle.premultiply_alpha(img, w, h, fmt, steps.pmalphaFlags)
            assert hr == 0
        if layout:
            img = probe.apply(fmt, w, h, [img], CS.steps(**LAYOUT[layout]))[0]
        if df in F.BLOCK_BYTES:
            hr, img = oracle.compress(img, w, h, fmt, df)
            assert hr == 0
        out.append(np.ascontiguousarray(img).view(np.uint8).reshape(-1))
    return out


def family(ran, prefix):
    return sum(v for k, v in ran.items() if k == prefix or k.startswith(prefix + "_"))


SRGB = F.TEX_FILTER_SRGB
# (name, entry, base kind, base fmt, w, h, items, levels, dst fmt, source kwargs, channel-steps kwargs, chain steps, texconv kwargs,
#  codes the reference may differ by (None: not compared))
CASES = [
    ("BC5 -> BC3n + invert Y", "gen", "bc5", 83, 64, 64, 2, 7, 77, dict(), dict(invert_y=True), None, dict(bc3_layout=1), 0),
    ("BC5 -> RXGB + reconstruct Z", "gen", "bc5", 83, 64, 32, 2, 6, 77, dict(), dict(reconstruct_z=True), None, dict(bc3_layout=2), 0),
    ("BC5_SNORM -> BC3n", "gen", "bc5s", 84, 64, 64, 2, 7, 77, dict(), None, None, dict(bc3_layout=1), 0),
    ("BC5_SNORM -> RXGB + invert Y", "gen", "bc5s", 84, 32, 32, 2, 6, 77, dict(), dict(invert_y=True), None, dict(bc3_layout=2), 0),
    ("BC4 -> BC3n", "gen", "bc", 80, 64, 64, 2, 7, 77, dict(), None, None, dict(bc3_layout=1), 0),
    ("BC4_SNORM -> RXGB", "gen", "bc", 81, 32, 32, 1, 6, 77, dict(), None, None, dict(bc3_layout=2), 0),
    ("RGBA8 -> BC3n + coverage + premultiply", "gen", "alpha", 28, 64, 64, 2, 7, 77, None, None, capi.chain_steps(0.5, True),
     dict(bc3_layout=1), None),
    ("RGBA16F -> BC3n + premultiply", "gen", "alpha", 10, 64, 32, 2, 6, 77, None, None, PM, dict(bc3_layout=1), 0),
    ("RGBA32F -> RXGB + premultiply", "gen", "alpha", 2, 32, 32, 2, 6, 77, None, None, PM, dict(bc3_layout=2), 0),
    ("R10G10B10A2 -> BC3n + coverage", "gen", "alpha", 24, 32, 32, 2, 6, 77, None, None, capi.chain_steps(0.5), dict(bc3_layout=1), None),
    ("BC3 -alpha -> BC7 + premultiply", "gen", "bc", 77, 64, 64, 2, 7, 98, dict(), None, PM, dict(demultiply=True), None),
    ("BC3 -alpha -> BC3 + premultiply", "gen", "bc", 77, 64, 64, 2, 7, 77, dict(), None, PM, dict(demultiply=True), 0),
    ("BC7 -alpha sRGB + resize -> BC3 + premultiply", "gen", "bc", 98, 64, 64, 2, 5, 77,
     dict(width=24, height=40, resize_filter=F.TEX_FILTER_LINEAR), None, PM, dict(demultiply=True, demultiply_flags=SRGB), None),
    ("RGBA8_SRGB -alpha -> BC7 + premultiply", "gen", "alpha", 29, 64, 64, 2, 7, 98, None, None, PM, dict(demultiply=True), None),
    ("RGBA8 -alpha sRGB -> BC3 + premultiply", "gen", "alpha", 28, 32, 32, 2, 6, 77, None, None, PM,
     dict(demultiply=True, demultiply_flags=SRGB), None),
    ("RGBA16F -alpha + resize -> BC3 + premultiply", "gen", "alpha", 10, 50, 30, 2, 5, 77, dict(width=32, height=32), None, PM,
     dict(demultiply=True), 0),
    ("BC3 -alpha -> RGBA8 + premultiply", "conv", "bc", 77, 64, 64, 2, 7, 28, dict(), None, PM, dict(demultiply=True), 0),
    ("RGBA8 -alpha sRGB -> BGRA8 + premultiply", "conv", "alpha", 28, 64, 32, 2, 6, 87, None, None, PM,
     dict(demultiply=True, demultiply_flags=SRGB), 1),
    ("RGBA8_SRGB -alpha + resize -> RGBA8 + premultiply", "conv", "alpha", 29, 40, 40, 2, 5, 28,
     dict(width=20, height=24, resize_filter=F.TEX_FILTER_CUBIC), None, PM, dict(demultiply=True), 1),
    ("RGBA16F -alpha -> BGRA8 + premultiply", "conv", "alpha", 10, 32, 32, 2, 6, 87, None, None, PM, dict(demultiply=True), 0),
    ("kept BC5 -> BC3n + invert Y", "lev", "bc5", 83, 64, 64, 2, 7, 77, None, dict(invert_y=True), None, dict(bc3_layout=1), 0),
    ("kept BC5_SNORM -> RXGB + reconstruct Z", "lev", "bc5s", 84, 32, 32, 2, 6, 77, None, dict(reconstruct_z=True), None,
     dict(bc3_layout=2), 0),
    ("kept BC4 -> RXGB + invert Y", "lev", "bc", 80, 40, 24, 2, 6, 77, None, dict(invert_y=True), None, dict(bc3_layout=2), 0),
    ("kept BC3 -alpha -> BC3 + premultiply", "lev", "bc", 77, 64, 64, 2, 7, 77, None, None, PM, dict(demultiply=True), 0),
    ("kept BC7 -alpha -> BGRA8 + premultiply", "lev", "bc", 98, 40, 40, 2, 6, 87, None, None, PM, dict(demultiply=True), 0),
    ("kept RGBA8 -alpha -> RGBA8 + premultiply", "lev", "alpha", 28, 32, 32, 2, 6, 28, None, None, PM, dict(demultiply=True), 0),
    ("kept RGBA16F -alpha + layout -> BC3n", "lev", "alpha", 10, 32, 32, 2, 6, 77, None, None, None,
     dict(demultiply=True, bc3_layout=1), 0),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_equals_separate_calls_and_reference(oracle, probe, case):
    name, entry, kind, bf, w, h, items, levels, df, source, ch, steps, tk, codes = case
    sizes = sizes_of(w, h, levels) if entry == "lev" else [(w, h)]
    bases = make_bases(kind, bf, sizes, items, len(name))
    (outs, opaque), ran = launches(one_call, entry, bases, sizes, bf, df, source, ch, steps, capi.texconv_steps(**tk), levels)
    want, want_opaque = separate(entry, bases, sizes, bf, df, source, ch, steps, tk, levels)
    for i in range(items):
        for l in range(levels):
            assert np.array_equal(outs[i][l], want[i][l]), (name, i, l)
    assert opaque == want_opaque, name
    # one chunk: exactly one more premultiply launch for the demultiply and one more k_convert launch for the layout than the call
    # without them, where that call does not pass a BC chain through
    if not (entry == "lev" and bf == df and bf in F.BLOCK_BYTES and ch is None and steps is None):
        _, bare = launches(one_call, entry, bases, sizes, bf, df, source, ch, steps, None, levels)
        assert family(ran, "k_pmalpha") == family(bare, "k_pmalpha") + (1 if tk.get("demultiply") else 0), (name, ran, bare)
        assert family(ran, "k_convert") == family(bare, "k_convert") + (1 if tk.get("bc3_layout") else 0), (name, ran, bare)
    if codes is None:
        return
    chain = reference(oracle, probe, entry, bases[0], sizes, bf, df, source, ch, steps, tk, levels)
    for l, (a, b) in enumerate(zip(outs[0], chain)):
        if codes:
            d = np.abs(a.astype(np.int16) - b.astype(np.int16))
            assert d.max() <= codes, (name, l, int(d.max()))
        else:
            assert np.array_equal(a, b), (name, l, int(np.count_nonzero(a != b)))
    if tk.get("bc3_layout") == 2 and entry != "lev":
        ow, oh = sizes[0]
        mine = capi.dds_save(np.concatenate(outs[0]), 77, ow, oh, 1, levels, flags=RXGB_DDS)
        hr, theirs = oracle.dds_save(np.concatenate(chain), 77, ow, oh, 1, levels, flags=RXGB_DDS)
        assert hr == 0 and np.array_equal(mine, theirs), name


@pytest.mark.parametrize("layout", [1, 2])
@pytest.mark.parametrize("entry", ["gen", "lev"])
def test_layout_is_the_permutation(layout, entry):
    """on RGBA32F chains the layout is exactly (1, y, 0, x) or (a, g, b, r), checked in numpy before the library's Compress"""
    w = h = 32
    levels = 6
    sizes = sizes_of(w, h, levels) if entry == "lev" else [(w, h)]
    rng = np.random.default_rng(layout)
    bases = [[(rng.random((lh, lw, 4), dtype=np.float32) * 1.5 - 0.25).astype(np.float32) for (lw, lh) in sizes] for _ in range(2)]
    outs, _ = one_call(entry, bases, sizes, 2, 77, None, None, None, capi.texconv_steps(bc3_layout=layout), levels)
    chains, _ = one_call("conv" if entry == "gen" else entry, bases, sizes, 2, 2, None, None, None, None, levels)
    for i in range(2):
        for l, (lw, lh) in enumerate(sizes_of(w, h, levels)):
            p = np.asarray(chains[i][l]).view(np.float32).reshape(lh, lw, 4)
            q = np.empty_like(p)
            if layout == 1:
                q[..., 0], q[..., 1], q[..., 2], q[..., 3] = 1.0, p[..., 1], 0.0, p[..., 0]
            else:
                q[..., 0], q[..., 1], q[..., 2], q[..., 3] = p[..., 3], p[..., 1], p[..., 2], p[..., 0]
            want = capi.compress(np.ascontiguousarray(q), lw, lh, 2, 77)
            assert np.array_equal(outs[i][l], want), (layout, entry, i, l)


@pytest.mark.parametrize("pitch,offset", [(0, 0), (16, 0), (4, 4)])
def test_caller_pitches(pitch, offset):
    """level 0 at a tight row pitch, 16 bytes wider, and 4 bytes wider at a pointer 4 bytes off: the same bytes as tight"""
    w, h, items, levels = 48, 40, 3, 6
    rng = np.random.default_rng(7)
    imgs = [alpha_image(28, w, h, rng) for _ in range(items)]
    ts = capi.texconv_steps(demultiply=True, bc3_layout=1)
    want, want_opaque = capi.mipmaps_compress_from_channels(imgs, w, h, 28, 77, None, None, 0, levels, 0, PM, texconv=ts)
    row = w * 4 + pitch
    laid = []
    for img in imgs:
        buf = np.zeros(row * h + offset, np.uint8)
        view = buf[offset:].reshape(h, row)
        view[:, :w * 4] = img.reshape(h, w * 4)
        laid.append(buf[offset:])
    got, opaque = capi.mipmaps_compress_from_channels(laid, w, h, 28, 77, None, None, 0, levels, 0, PM, row_pitch=row, texconv=ts)
    assert opaque == want_opaque
    for a, b in zip(got, want):
        assert np.array_equal(a, b), (pitch, offset)


EX = {"gen": "dxb200_mipmaps_compress_from_channels_ex", "conv": "dxb200_mipmaps_convert_from_ex", "lev": "dxb200_levels_from_ex"}


@pytest.mark.parametrize("entry", ["gen", "conv", "lev"])
def test_null_and_zero_steps_are_the_call_without_ex(entry, monkeypatch):
    """NULL and all-zero steps give the bytes, the alpha answer and the kernel launches of the call without _ex"""
    w = h = 64
    levels = 7
    sizes = sizes_of(w, h, levels) if entry == "lev" else [(w, h)]
    bases = make_bases("bc", 77, sizes, 2, 3)
    df = 87 if entry == "conv" else 98
    source = dict() if entry != "lev" else None
    runs = [launches(one_call, entry, bases, sizes, 77, df, source, None, PM, ts, levels) for ts in (None, capi.texconv_steps())]
    plain = getattr(L, EX[entry][:-3])
    monkeypatch.setattr(L, EX[entry], lambda *a: plain(*a[:-1]))          # the binding's call without its last argument
    (old, old_opaque), old_ran = launches(one_call, entry, bases, sizes, 77, df, source, None, PM, None, levels)
    for (new, opaque), ran in runs:
        assert ran == old_ran and opaque == old_opaque, (entry, ran, old_ran)
        for a, b in zip(new, old):
            assert np.array_equal(np.concatenate(a), np.concatenate(b)), entry


@pytest.mark.parametrize("entry,w,items", [("gen", 1024, 40), ("lev", 1024, 40)])
def test_chunks_launch_counts(entry, w, items):
    """an array over several chunks: one premultiply launch for the demultiply and one k_convert launch for the layout per
    chunk, beside one Compress launch per chunk, and every item equals the separate calls"""
    levels = 4
    sizes = sizes_of(w, w, levels) if entry == "lev" else [(w, w)]
    bases = make_bases("alpha", 28, sizes, items, 5)
    tk = dict(demultiply=True, bc3_layout=2)
    (outs, opaque), ran = launches(one_call, entry, bases, sizes, 28, 77, None, None, PM, capi.texconv_steps(**tk), levels)
    (_, _), bare = launches(one_call, entry, bases, sizes, 28, 77, None, None, PM, None, levels)
    chunks = family(ran, "k_compress_bc15")
    assert chunks > 1 and chunks == family(bare, "k_compress_bc15"), (ran, bare)
    assert family(ran, "k_pmalpha") == family(bare, "k_pmalpha") + chunks, (ran, bare)
    assert family(ran, "k_convert") == family(bare, "k_convert") + chunks, (ran, bare)
    want, want_opaque = separate(entry, bases, sizes, 28, 77, None, None, PM, tk, levels)
    assert opaque == want_opaque
    for i in range(items):
        for l in range(levels):
            assert np.array_equal(outs[i][l], want[i][l]), (entry, i, l)


def test_two_devices():
    """items sharded over two devices give the bytes of one device"""
    if L.dxb200_device_count() < 2:
        pytest.skip("needs two devices")
    w, items, levels = 256, 8, 5
    sizes = [(w, w)]
    bases = make_bases("bc5", 83, sizes, items, 9)
    ts = capi.texconv_steps(bc3_layout=2)
    one, one_opaque = one_call("gen", bases, sizes, 83, 77, dict(), dict(invert_y=True), None, ts, levels)
    L.dxb200_shutdown()
    capi.init_devices([0, 1])
    two, two_opaque = one_call("gen", bases, sizes, 83, 77, dict(), dict(invert_y=True), None, ts, levels)
    assert one_opaque == two_opaque
    for a, b in zip(one, two):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
