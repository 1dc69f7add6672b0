"""GPU suite: texconv's channel steps on the device equal the reference's TransformImage (tests/cpp/channel_steps_probe.cpp linked
with the reference build) on the corpus of the CPU suite: through the host call (one image, an array over several chunks, one image
cut into bands, sharded over the devices) and through the _device call, in place and at wide pitches.  dxb200_mipmaps_compress_from_
channels equals dxb200_decompress + dxb200_resize + dxb200_apply_channel_steps + dxb200_mipmaps_compress_from_ex, blocks and
alpha-opaque answer, and the reference's composed calls where those are bit-exact (BC1-BC5 targets), on texconv's sequences.  Every
call runs only the generic k_convert for the steps: one launch per chunk, and none when no step is enabled."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F, synth
from tests import channel_steps_lib as CS
from tests import special_values as SV

pytestmark = pytest.mark.gpu
L = capi.lib


@pytest.fixture(scope="module")
def ref(tmp_path_factory, oracle):
    assert L.dxb200_init(0) == 0
    return CS.Probe(tmp_path_factory.mktemp("channel_ref"))


def counted(fn, *args, **kw):
    """(fn's result, all launches, k_convert launches) of one call"""
    n0, k0 = capi.launch_count(), capi.kernel_launch_count("k_convert")
    out = fn(*args, **kw)
    return out, capi.launch_count() - n0, capi.kernel_launch_count("k_convert") - k0


@pytest.mark.parametrize("config", sorted(CS.CONFIGS))
@pytest.mark.parametrize("fmt", CS.FORMATS)
def test_host_call_equals_reference(fmt, config, ref):
    s = CS.steps(**CS.CONFIGS[config])
    img = CS.corpus(fmt)
    want = ref.apply(fmt, CS.W, CS.H, [img], s)[0]
    (got,), n, k = counted(capi.apply_channel_steps, [img], CS.W, CS.H, fmt, s)
    SV.assert_same(got, want, fmt, "%d %s" % (fmt, config))
    assert n == k == 1, (fmt, config, n, k)


def test_array_over_several_chunks_and_one_image_in_bands(ref):
    """24 x 1024^2 RGBA8 images (8 MiB of source and destination each: several 48 MiB chunks) and one 4096^2 RGBA8 image (four 32
    MiB bands), with all four steps"""
    s = CS.steps(**CS.CONFIGS["all"])
    imgs = [CS.corpus(28, 1024, 1024, seed=k) for k in range(24)]
    want = ref.apply(28, 1024, 1024, imgs, s)
    got, n, k = counted(capi.apply_channel_steps, imgs, 1024, 1024, 28, s)
    for i, (a, b) in enumerate(zip(got, want)):
        SV.assert_same(a, b, 28, "item %d" % i)
    assert n == k and k > 1, (n, k)
    big = CS.corpus(28, 4096, 4096, seed=7)
    want = ref.apply(28, 4096, 4096, [big], s)[0]
    (got,), n, k = counted(capi.apply_channel_steps, [big], 4096, 4096, 28, s)
    SV.assert_same(got, want, 28, "bands")
    assert n == k and k >= 4, (n, k)


@pytest.mark.parametrize("fmt", (28, 2, 10, 31, 86, 41, 85))
def test_device_call_in_place_and_at_wide_pitches(ref, fmt):
    """dxb200_apply_channel_steps_device: in place (dst == src) at the tight pitch, and from a +16 pitch into a +4 pitch whose base
    is 4 bytes off"""
    torch = pytest.importorskip("torch")
    w, h = 97, 61
    bpp = F.BYTES_PER_PIXEL[fmt]
    row = w * bpp
    s = CS.steps(**CS.CONFIGS["all"])
    img = CS.corpus(fmt, w, h, seed=3)
    want = ref.apply(fmt, w, h, [img], s)[0].reshape(h, row)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def upload(extra, off):
        pitch = row + extra
        buf = torch.zeros(off + pitch * h + 64, dtype=torch.uint8, device="cuda")
        view = np.zeros((h, pitch), np.uint8)
        view[:, :row] = img.reshape(h, row)
        buf[off:off + pitch * h] = torch.from_numpy(view.reshape(-1)).cuda()
        return buf, capi.Image(w, h, fmt, pitch, pitch * h, buf.data_ptr() + off)

    def rows(buf, im, off):
        return buf.cpu().numpy()[off:off + im.rowPitch * h].reshape(h, im.rowPitch)[:, :row]

    buf, im = upload(0, 0)
    imgs = capi.images([im])
    hr, n, k = counted(L.dxb200_apply_channel_steps_device, imgs, 1, C.byref(s), imgs, stream)
    torch.cuda.synchronize()
    assert F.hr_u32(hr) == 0 and n == k == 1, (fmt, hex(F.hr_u32(hr)), capi.last_error())
    SV.assert_same(rows(buf, im, 0), want, fmt, "in place")
    sbuf, sim = upload(16, 0)
    dbuf, dim = upload(4, 4)
    hr, n, k = counted(L.dxb200_apply_channel_steps_device, capi.images([sim]), 1, C.byref(s), capi.images([dim]), stream)
    torch.cuda.synchronize()
    assert F.hr_u32(hr) == 0 and n == k == 1
    SV.assert_same(rows(dbuf, dim, 4), want, fmt, "pitches")


def test_sharded_over_devices(ref):
    if L.dxb200_device_count() < 2:
        pytest.skip("one device")
    capi.init_devices(list(range(min(4, L.dxb200_device_count()))))
    s = CS.steps(**CS.CONFIGS["all"])
    imgs = [CS.corpus(87, 512, 512, seed=k) for k in range(8)]
    want = ref.apply(87, 512, 512, imgs, s)
    got = capi.apply_channel_steps(imgs, 512, 512, 87, s)
    for a, b in zip(got, want):
        SV.assert_same(a, b, 87, "sharded")


# ---- the pipeline ----------------------------------------------------------------------------------------------------------------
def _normals(w, h, seed):
    """RGBA8 tangent-space normal maps: x, y from a smooth field, some with x*x + y*y > 1 (as after a resize)"""
    img = synth.content_ldr("gradient", w, h, seed=seed)
    out = np.zeros((h, w, 4), np.uint8)
    out[..., :2] = (img[..., :2] * 255).round().astype(np.uint8)
    out[..., 2:] = 255
    return out


def _bases(kind, w, h, items):
    if kind in ("bc5", "bc5s"):
        fmt = 83 if kind == "bc5" else 84
        rg = [_normals(w, h, s) for s in range(items)]
        if kind == "bc5s":
            return [capi.compress((img.astype(np.float32) / 127.5 - 1.0).astype(np.float32), w, h, 2, fmt) for img in rg]
        return [capi.compress(img, w, h, 28, fmt) for img in rg]
    img = [(synth.content_ldr("cutout", w, h, seed=s) * 255).round().astype(np.uint8) for s in range(items)]
    if kind == "bgra":
        return [np.ascontiguousarray(i[..., [2, 1, 0, 3]]) for i in img]
    return img


SEQUENCES = [
    # (name, base kind, items, w, h, base fmt, level-0 fmt, dst fmt, source kwargs, channel steps kwargs, chain steps)
    ("BC5 -> invert Y -> BC5", "bc5", 3, 64, 64, 83, 49, 83, dict(), dict(invert_y=True), None),
    ("BC5 -> reconstruct Z -> BC7", "bc5", 3, 64, 64, 83, 28, 98, dict(), dict(reconstruct_z=True), None),
    ("BC5 -> reconstruct Z -> BC1", "bc5", 3, 64, 64, 83, 28, 71, dict(), dict(reconstruct_z=True), None),
    ("BC5 SNORM -> invert Y, reconstruct Z -> BC5 SNORM", "bc5s", 2, 64, 64, 84, 31, 84, dict(), dict(invert_y=True, reconstruct_z=True), None),
    ("RGBA8 cut-outs -> colour key -> coverage + premultiply -> BC3", "rgba", 3, 64, 48, 28, 28, 77, None, dict(color_key=0x000000),
     capi.chain_steps(0.5, True)),
    ("BGRA8 swizzle -> resize -> BC7", "bgra", 2, 96, 64, 87, 87, 98, dict(width=64, height=32, resize_filter=F.TEX_FILTER_LINEAR),
     dict(swizzle=(2, 1, 0, 3), one_mask=0b1000), None),
    ("RGBA8 all four steps, 40 items over chunks -> BC3", "rgba", 40, 1024, 1024, 28, 28, 77, None, CS.CONFIGS["all"], None),
]


def _separate(bases, w, h, bf, fmt, df, source, channels, steps):
    """the separate calls: decompress (to fmt), resize, apply_channel_steps, mipmaps_compress_from_ex; (chains, opaque, level 0)"""
    lw, lh = w, h
    imgs = bases
    if bf in F.BLOCK_BYTES:
        imgs = capi.decompress_images(bases, [(w, h)] * len(bases), bf, fmt)
    if source and source.get("width"):
        lw, lh = source["width"], source["height"]
        imgs = capi.resize_images(imgs, w, h, fmt, lw, lh, source.get("resize_filter", 0))
    imgs = capi.apply_channel_steps(imgs, lw, lh, fmt, CS.steps(**channels))
    outs, opaque = capi.mipmaps_compress_from_ex(imgs, lw, lh, fmt, df, steps=steps)
    return outs, opaque, imgs


@pytest.mark.parametrize("seq", SEQUENCES, ids=[s[0] for s in SEQUENCES])
def test_from_channels_equals_the_separate_calls(ref, oracle, seq):
    name, kind, items, w, h, bf, fmt, df, source, channels, steps = seq
    bases = _bases(kind, w, h, items)
    src = capi.chain_source(**source) if source is not None else None
    ch = CS.steps(**channels)
    (outs, opaque), n_ch, k_ch = counted(capi.mipmaps_compress_from_channels, bases, w, h, bf, df, source=src, channels=ch, steps=steps)
    # _from_ex with the same decompress format runs the same kernels but the steps' k_convert, one launch per chunk
    src_ex = capi.chain_source(fmt if bf in F.BLOCK_BYTES else 0, src.width, src.height, src.resizeFilter) if src is not None else None
    (outs_ex, _), n_ex, k_ex = counted(capi.mipmaps_compress_from_ex, bases, w, h, bf, df, source=src_ex, steps=steps)
    chunks = n_ch - n_ex
    assert chunks >= 1 and k_ch - k_ex == chunks, (name, n_ch, n_ex, k_ch, k_ex)
    if items == 40:
        assert chunks > 1, name
    want, want_opaque, level0 = _separate(bases, w, h, bf, fmt, df, source, channels, steps)
    for a, b in zip(outs, want):
        assert np.array_equal(a, b), name
    assert opaque == want_opaque, name
    # the reference's composed calls for BC1-BC5 targets, level 0 of item 0: its steps on the same level 0, then its Compress
    if df in (71, 77, 83, 84) and steps is None:
        lw, lh = (source["width"], source["height"]) if source and source.get("width") else (w, h)
        if bf in F.BLOCK_BYTES:
            hr, dec = oracle.decompress(bases[0], w, h, bf, fmt)
            assert hr == 0
            assert np.array_equal(dec, np.asarray(capi.decompress_images(bases[:1], [(w, h)], bf, fmt)[0]).reshape(-1)), name
            pre = dec
        else:
            pre = np.ascontiguousarray(bases[0]).view(np.uint8).reshape(-1)
        stepped = ref.apply(fmt, lw, lh, [pre], ch)[0]
        assert np.array_equal(stepped, np.asarray(level0[0]).view(np.uint8).reshape(-1)), name
        hr, blocks = oracle.compress(stepped, lw, lh, fmt, df)
        assert hr == 0
        assert np.array_equal(blocks, outs[0][:blocks.size]), name


def test_no_step_enabled_launches_nothing_more(ref):
    bases = _bases("rgba", 64, 48, 3)
    for ch in (None, CS.steps()):
        (outs, opaque), n_ch, k_ch = counted(capi.mipmaps_compress_from_channels, bases, 64, 48, 28, 77, channels=ch)
        (outs_ex, opaque_ex), n_ex, k_ex = counted(capi.mipmaps_compress_from_ex, bases, 64, 48, 28, 77)
        assert n_ch == n_ex and k_ch == k_ex
        assert opaque == opaque_ex and all(np.array_equal(a, b) for a, b in zip(outs, outs_ex))
