"""GPU suite: IsAlphaAllOpaque on the device answers like the reference (tests/cpp/alpha_opaque_probe.cpp linked with the
reference build) on the corpus of the CPU suite: through the host call (one device, sharded, an array over several chunks, one
image cut into bands), through the _device call at several pitches, through the mirror's ScratchImage::IsAlphaAllOpaque, and as
the answer dxb200_mipmaps_compress_from_ex returns with blocks identical to dxb200_mipmaps_compress_from's.  Every call runs only
the generic k_convert or k_decompress, once per chunk, and formats without alpha launch nothing."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F, synth
from tests import alpha_opaque_lib as A

pytestmark = pytest.mark.gpu
L = capi.lib
KERNEL = {True: "k_decompress", False: "k_convert"}


@pytest.fixture(scope="module")
def ref(tmp_path_factory, oracle):
    return A.Probe(tmp_path_factory.mktemp("alpha_ref"), reference=True)


@pytest.fixture(scope="module")
def mirror(tmp_path_factory):
    assert L.dxb200_init(0) == 0
    return A.Probe(tmp_path_factory.mktemp("alpha_ours"), reference=False)


def launches():
    return capi.launch_count(), {k: capi.kernel_launch_count(k) for k in ("k_convert", "k_decompress")}


def host_opaque(fmt, w, h, pixels, items=1, levels=1, expect_launches=1):
    """dxb200_is_alpha_all_opaque of a texture in ScratchImage layout; asserts the call ran expect_launches launches of the generic
    kernel of its format and nothing else"""
    pixels = np.ascontiguousarray(pixels).view(np.uint8).reshape(-1)
    n0, k0 = launches()
    hr, op = A.call(L.dxb200_is_alpha_all_opaque, A.container_images(fmt, w, h, pixels, items, levels), items * levels)
    n1, k1 = launches()
    assert hr == F.S_OK, (fmt, hex(hr), capi.last_error())
    k = KERNEL[fmt in F.BLOCK_BYTES]
    if expect_launches is not None:
        assert n1 - n0 == expect_launches and k1[k] - k0[k] == expect_launches, (fmt, n1 - n0, k1, k0)
    else:
        assert n1 - n0 == k1[k] - k0[k] >= 1
    return op == 1


def boundary(ref, fmt):
    codes = A.alpha_codes(fmt)
    want = A.per_code(ref.opaque, fmt, codes)
    non, op = A.boundary_codes(fmt, want, codes)
    vals = A.code_values(fmt, codes)
    fill = codes[want][np.argmax(np.where(np.isfinite(vals[want]), vals[want], -1))]
    return non, op, fill


@pytest.mark.parametrize("fmt", A.PIXEL_FORMATS)
def test_pixel_formats_through_the_host_call(ref, mirror, fmt):
    """Boundary codes at the first, middle and last texel of images 1, 5 and 257 wide, alone and as the last image of an array; all
    opaque images; the fp32 special values each alone.  Host call == reference == mirror, one k_convert launch each."""
    non, op, fill = boundary(ref, fmt)
    for w, h in ((1, 1), (5, 3), (257, 2)):
        for code in (non, op):
            for where in ("first", "middle", "last"):
                px = A.placed(fmt, w, h, code, where, fill)
                want = ref.opaque(fmt, w, h, px)
                assert host_opaque(fmt, w, h, px) == want == mirror.opaque(fmt, w, h, px), (fmt, w, h, code, where)
                arr = np.concatenate([A.placed(fmt, w, h, fill, "first", fill)] * 2 + [px])
                assert host_opaque(fmt, w, h, arr, items=3) == ref.opaque(fmt, w, h, arr, items=3) == want
    if fmt == 2:
        _, make = A.alpha_field(fmt)
        for c in A.f32_codes():
            px = make([c])
            assert host_opaque(fmt, 1, 1, px) == ref.opaque(fmt, 1, 1, px), hex(int(c))


@pytest.mark.parametrize("fmt", A.BLOCK_FORMATS)
def test_block_formats_through_the_host_call(ref, mirror, fmt):
    """The CPU suite's blocks by class, as 4x4 and 3x2 images; BC1 transparent texels in the padding of partial blocks; blocks the
    reference's encoder makes.  Host call == reference, one k_decompress launch each; the mirror agrees."""
    rng = np.random.default_rng(fmt)
    for b in A.block_corpus(fmt, rng):
        assert host_opaque(fmt, 4, 4, b) == ref.opaque(fmt, 4, 4, b), (fmt, b.tobytes().hex())
        assert host_opaque(fmt, 3, 2, b) == ref.opaque(fmt, 3, 2, b) == mirror.opaque(fmt, 3, 2, b), (fmt, b.tobytes().hex())
    if fmt in (71, 72):
        for (w, h) in ((1, 1), (2, 3), (5, 7), (13, 9)):
            assert host_opaque(fmt, w, h, A.bc1_partial_image(w, h, False))
            assert not host_opaque(fmt, w, h, A.bc1_partial_image(w, h, True))


@pytest.mark.parametrize("fmt", A.BLOCK_FORMATS)
def test_reference_encoded_containers(ref, mirror, oracle, fmt):
    """Reference-encoded blocks in the containers a caller builds: 2D, an array, a chain and a cube map (the mirror's
    IsAlphaAllOpaque == the reference's on each)."""
    blocks = A.reference_encoded(oracle, fmt, w=32, h=32) + A.reference_encoded(oracle, fmt, w=32, h=32, opaque=True)
    for b in blocks:
        assert host_opaque(fmt, 32, 32, b) == ref.opaque(fmt, 32, 32, b) == mirror.opaque(fmt, 32, 32, b)
    arr = np.concatenate(blocks[3:] + blocks[:1])
    assert mirror.opaque(fmt, 32, 32, arr, items=4) == ref.opaque(fmt, 32, 32, arr, items=4)
    n = capi.texture_layout(fmt, 32, 32, 6, 2)[1]
    cube = np.resize(np.concatenate(blocks[3:]), n)
    assert mirror.opaque(fmt, 32, 32, cube, items=1, levels=2, cube=True) == ref.opaque(fmt, 32, 32, cube, items=1, levels=2, cube=True)
    n = capi.texture_layout(fmt, 32, 32, 2, 3)[1]
    chains = np.resize(np.concatenate(blocks), n)
    assert mirror.opaque(fmt, 32, 32, chains, items=2, levels=3) == ref.opaque(fmt, 32, 32, chains, items=2, levels=3)


def test_formats_without_alpha_launch_nothing(mirror):
    for fmt in A.NO_ALPHA_FORMATS:
        n = capi.texture_layout(fmt, 16, 16, 1, 1)[1]
        px = np.zeros(n, np.uint8)
        n0, _ = launches()
        hr, op = A.call(L.dxb200_is_alpha_all_opaque, A.container_images(fmt, 16, 16, px), 1)
        assert (hr, op) == (F.S_OK, 1) and mirror.opaque(fmt, 16, 16, px)
        assert launches()[0] == n0, fmt


def test_array_over_several_chunks_and_one_image_in_bands(ref, oracle):
    """12 x 1024^2 RGBA32F images (16 MiB each: several 48 MiB chunks) with one non-opaque texel in the last image only; one
    2048 x 4096 RGBA32F image (128 MiB: four bands) with it at its last texel, then opaque; one 4096^2 BC7 image made of opaque
    blocks with one non-opaque block at its end."""
    fmt, w = 2, 1024
    _, make = A.alpha_field(fmt)
    one, below = np.float32(1).view(np.uint32), np.nextafter(np.float32(0.997), np.float32(0)).view(np.uint32)
    img = make([one] * (w * w)).reshape(-1)
    arr = np.tile(img, 12)
    last = arr.size - 16
    arr[last:] = make([below])[0]
    assert host_opaque(fmt, w, w, arr, items=12, expect_launches=None) is False
    assert ref.opaque(fmt, w, w, arr, items=12) is False
    arr[last:] = img[:16]
    assert host_opaque(fmt, w, w, arr, items=12, expect_launches=None) is True
    big = make([one] * (2048 * 4096)).reshape(-1)
    big[-16:] = make([below])[0]
    assert host_opaque(fmt, 2048, 4096, big, expect_launches=None) is False
    assert ref.opaque(fmt, 2048, 4096, big) is False
    big[-16:] = big[:16]
    assert host_opaque(fmt, 2048, 4096, big, expect_launches=None) is True
    hr, white = oracle.compress(np.ones((4, 4, 4), np.float32), 4, 4, 2, 98)
    assert hr == 0 and ref.opaque(98, 4, 4, white)
    blocks = np.tile(white, 1024 * 1024)
    assert host_opaque(98, 4096, 4096, blocks, expect_launches=None) is True
    blocks[-16:] = 0                                        # the reserved mode: zeros, alpha 0
    assert host_opaque(98, 4096, 4096, blocks, expect_launches=None) is False


def _device_copy(host, extra_pitch, row, rows, offset, torch):
    """host rows (row bytes each) copied to device memory at pitch row + extra_pitch, starting `offset` bytes into the buffer"""
    pitch = row + extra_pitch
    buf = torch.zeros(offset + pitch * rows + 64, dtype=torch.uint8, device="cuda")
    view = np.zeros((rows, pitch), np.uint8)
    view[:, :row] = host.reshape(rows, row)
    buf[offset:offset + pitch * rows] = torch.from_numpy(view.reshape(-1)).cuda()
    return buf, pitch


@pytest.mark.parametrize("fmt", (28, 2, 10, 86, 77, 98, 71))
def test_device_call_pitches(ref, fmt):
    """dxb200_is_alpha_all_opaque_device on device images: pitches tight, +16, and (uncompressed) +4 with the base 4 bytes off."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(fmt)
    w, h = 37, 23
    if fmt in F.BLOCK_BYTES:
        cases = [A.bc1_partial_image(w, h, inside) for inside in (False, True)] if fmt == 71 else \
            [np.concatenate([b] * (((w + 3) // 4) * ((h + 3) // 4))) for b in A.block_corpus(fmt, rng)[:6]]
        layouts = ((0, 0), (16, 0))
        row, rows = F.compute_pitch(fmt, w, h)[0], (h + 3) // 4
    else:
        non, op, fill = boundary(ref, fmt)
        cases = [A.placed(fmt, w, h, c, where, fill) for c in (non, op) for where in ("first", "middle", "last")]
        layouts = ((0, 0), (16, 0), (4, 4))
        row, rows = F.compute_pitch(fmt, w, h)[0], h
    stream = torch.cuda.current_stream().cuda_stream
    for px in cases:
        want = ref.opaque(fmt, w, h, px)
        for extra, off in layouts:
            buf, pitch = _device_copy(px, extra, row, rows, off, torch)
            imgs = capi.images([capi.Image(w, h, fmt, pitch, pitch * rows, buf.data_ptr() + off)] * 2)
            n0, k0 = launches()
            opaque = C.c_int32(-1)
            hr = F.hr_u32(L.dxb200_is_alpha_all_opaque_device(imgs, 2, C.byref(opaque), C.c_void_p(stream)))
            n1, k1 = launches()
            assert hr == F.S_OK, (fmt, extra, off, hex(hr), capi.last_error())
            assert (opaque.value == 1) == want, (fmt, extra, off)
            k = KERNEL[fmt in F.BLOCK_BYTES]
            assert n1 - n0 == 1 and k1[k] - k0[k] == 1


def test_sharded_over_devices(ref):
    """With two or more devices the host call shards the bands and ANDs their answers."""
    if L.dxb200_device_count() < 2:
        pytest.skip("one device")
    capi.init_devices(list(range(min(4, L.dxb200_device_count()))))
    fmt, w = 28, 512
    img = np.full((w * w * 8, 4), 255, np.uint8)
    for where in (0, img.shape[0] // 2, img.shape[0] - 1):
        px = img.copy()
        px[where, 3] = 252
        assert host_opaque(fmt, w, w, px, items=8, expect_launches=None) is False
    assert host_opaque(fmt, w, w, img, items=8, expect_launches=None) is True


# ---- the pipeline ----------------------------------------------------------------------------------------------------------------
def compress_launches():
    return sum(capi.kernel_launch_count(k) for k in ("k_compress_bc15", "k_compress_bc15_t", "k_compress_bc7", "k_compress_bc7_tma",
                                                     "k_compress_bc6h"))


def _run(fn, *args, **kw):
    d0, c0 = capi.kernel_launch_count("k_decompress"), compress_launches()
    out = fn(*args, **kw)
    return out, capi.kernel_launch_count("k_decompress") - d0, compress_launches() - c0


SEQUENCES = [
    # (name, bases, w, h, base fmt, dst fmt, source, steps)
    ("BC3 -> resize -> coverage -> premultiply -> BC7", "bc3", 64, 64, 77, 98, dict(width=48, height=32, resize_filter=F.TEX_FILTER_LINEAR),
     capi.chain_steps(0.5, True)),
    ("RGBA8 cutout -> BC1 with a threshold", "cutout", 64, 48, 28, 71, None, None),
    ("RGBA8 opaque -> BC1", "opaque", 64, 48, 28, 71, None, None),
    ("RGBA8 cutout -> BC3, 40 items over chunks", "cutout40", 512, 512, 28, 77, None, None),
    ("RGBA8 cutout -> BC4 (no scan)", "cutout", 64, 48, 28, 80, None, None),
]


def _bases(kind, w, h):
    if kind == "bc3":
        return [capi.compress((synth.content_ldr("cutout", w, h, seed=s) * 255).astype(np.uint8), w, h, 28, 77) for s in range(3)]
    imgs = [(synth.content_ldr("cutout", w, h, seed=s) * 255).round().astype(np.uint8) for s in range(40 if kind == "cutout40" else 3)]
    if kind == "opaque":
        for i in imgs:
            i[..., 3] = 255
    return imgs


@pytest.mark.parametrize("seq", SEQUENCES, ids=[s[0] for s in SEQUENCES])
def test_from_ex_answers_for_its_output(ref, seq):
    """_from_ex's blocks are _from's byte for byte, its answer is the reference's IsAlphaAllOpaque of the output chain, and every
    chunk runs exactly one scan launch (BC4: none)."""
    name, kind, w, h, bf, df, source, steps = seq
    bases = _bases(kind, w, h)
    src = capi.chain_source(**source) if source else None
    cw, ch = (source["width"], source["height"]) if source else (w, h)
    outs, dec_from, comp_from = _run(capi.mipmaps_compress_from, bases, w, h, bf, df, source=src, steps=steps)
    (outs_ex, opaque), dec_ex, comp_ex = _run(capi.mipmaps_compress_from_ex, bases, w, h, bf, df, source=src, steps=steps)
    assert all(np.array_equal(a, b) for a, b in zip(outs, outs_ex)), name
    levels = F.count_mips(cw, ch)
    want = ref.opaque(df, cw, ch, np.concatenate(outs_ex), items=len(bases), levels=levels)
    assert opaque == want, name
    assert comp_ex == comp_from >= 1
    scans = dec_ex - dec_from
    assert scans == (0 if df == 80 else comp_ex), (name, scans, comp_ex)
