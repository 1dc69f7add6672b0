"""CPU suite: IsAlphaAllOpaque (dxb200_is_alpha_all_opaque, its _device twin, dxb200_mipmaps_compress_from_ex and the mirror's
ScratchImage::IsAlphaAllOpaque) without a device.

The HRESULT table runs through the library and through the planner on the host (tests/emul/alpha_opaque.cpp); formats without
alpha are answered on this machine, by the library and by the mirror.  The emulator walks every texel with the rule and the
decoders the device scan runs, and must answer like the reference (tests/cpp/alpha_opaque_probe.cpp linked with the reference
build) on every alpha code of every implemented uncompressed format with alpha, on boundary texels placed anywhere in images and
arrays, and on BC1 / BC2 / BC3 / BC7 blocks by class."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import alpha_opaque_lib as A
from tests.test_cpu_mipmaps_compress_from import TABLE, VALID, Call

L = capi.lib
NO_DEVICE = L.dxb200_device_count() == 0
SCAN_HR = F.E_FAIL if NO_DEVICE else F.S_OK          # what a call that has to scan returns


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    E = A.load_emul(tmp_path_factory.mktemp("alpha_emul"))
    E.emul_plan_mipmaps_compress_from_ex.argtypes = L.dxb200_mipmaps_compress_from_ex.argtypes + [C.POINTER(C.c_int32)]
    E.emul_plan_mipmaps_compress_from_ex.restype = C.c_int32
    return E


@pytest.fixture(scope="module")
def ref(tmp_path_factory, oracle):
    return A.Probe(tmp_path_factory.mktemp("alpha_ref"), reference=True)


@pytest.fixture(scope="module")
def mirror(tmp_path_factory):
    return A.Probe(tmp_path_factory.mktemp("alpha_ours"), reference=False)


def emul_opaque(emul, fmt, w, h, pixels, items=1, levels=1):
    pixels = np.ascontiguousarray(pixels).view(np.uint8).reshape(-1)
    hr, op = A.call(emul.emul_is_alpha_all_opaque, A.container_images(fmt, w, h, pixels, items, levels), items * levels)
    assert hr == F.S_OK, (fmt, w, h, hex(hr))
    return op == 1


def _imgs(specs, keep):
    """dxb200_image array of (w, h, fmt, rowPitch, pixels?) specs; pixels True = a fresh zeroed buffer"""
    out = []
    for (w, h, fmt, row, has) in specs:
        buf = np.zeros(max(row, 1) * (h + 4) + 64, np.uint8)
        keep.append(buf)
        out.append(capi.Image(w, h, fmt, row, row * h, buf.ctypes.data if has else None))
    return capi.images(out)


# (name, image specs (w, h, fmt, rowPitch, has pixels), HRESULT of the planner, opaque when S_OK without a scan)
TABLE_OPAQUE = [
    ("R8G8B8A8", [(8, 8, 28, 32, True)], "scan", None),
    ("BC7 partial", [(5, 3, 98, 32, True)], "scan", None),
    ("array of BC3", [(8, 8, 77, 32, True)] * 3, "scan", None),
    ("no alpha: R32_FLOAT", [(8, 8, 41, 32, True)], F.S_OK, 1),
    ("no alpha: B8G8R8X8", [(8, 8, 88, 32, True)], F.S_OK, 1),
    ("no alpha: BC4", [(8, 8, 80, 16, True)], F.S_OK, 1),
    ("no alpha: BC5", [(8, 8, 83, 32, True)], F.S_OK, 1),
    ("no alpha: BC6H", [(8, 8, 95, 32, True)], F.S_OK, 1),
    ("no alpha, not implemented: R32_UINT", [(8, 8, 42, 32, True)], F.S_OK, 1),
    ("formats differ", [(8, 8, 28, 32, True), (8, 8, 87, 32, True)], F.E_INVALIDARG, None),
    ("formats differ, no alpha", [(8, 8, 41, 32, True), (8, 8, 88, 32, True)], F.E_INVALIDARG, None),
    ("null pixels", [(8, 8, 28, 32, True), (8, 8, 28, 32, False)], F.E_POINTER, None),
    ("null pixels, no alpha", [(8, 8, 41, 32, False)], F.E_POINTER, None),
    ("alpha, not implemented: R8G8B8A8_UINT", [(8, 8, 30, 32, True)], F.HRESULT_E_NOT_SUPPORTED, None),
    ("alpha, not implemented: BC1_TYPELESS", [(8, 8, 70, 16, True)], F.HRESULT_E_NOT_SUPPORTED, None),
    ("alpha, not implemented: R10G10B10_XR_BIAS_A2", [(8, 8, 89, 32, True)], F.HRESULT_E_NOT_SUPPORTED, None),
    ("BC row pitch off the block size", [(8, 8, 77, 40, True)], F.E_INVALIDARG, None),
    ("BC1 row pitch off the block size", [(8, 8, 71, 20, True)], F.E_INVALIDARG, None),
    ("zero width", [(0, 8, 28, 32, True)], F.E_INVALIDARG, None),
    ("zero height", [(8, 0, 98, 32, True)], F.E_INVALIDARG, None),
]


@pytest.mark.parametrize("name,specs,want,answer", TABLE_OPAQUE, ids=[t[0] for t in TABLE_OPAQUE])
def test_hresult_table(emul, name, specs, want, answer):
    """The library's host and _device calls and the host planner agree; formats without alpha answer 1 without a device."""
    keep = []
    imgs = _imgs(specs, keep)
    hr_e, op_e = A.call(emul.emul_is_alpha_all_opaque, imgs, len(specs))
    hr_h, op_h = A.call(L.dxb200_is_alpha_all_opaque, imgs, len(specs))
    opaque = C.c_int32(-1)
    hr_d = F.hr_u32(L.dxb200_is_alpha_all_opaque_device(imgs, len(specs), C.byref(opaque), None))
    if want == "scan":
        assert hr_e == F.S_OK and op_e in (0, 1)
        assert hr_h == SCAN_HR and (NO_DEVICE or op_h == op_e), (name, hex(hr_h))
        return
    assert (hr_e, hr_h, hr_d) == (want, want, want), (name, hex(hr_e), hex(hr_h), hex(hr_d))
    if want == F.S_OK:
        assert op_e == op_h == opaque.value == answer


def test_argument_pointers():
    keep = []
    imgs = _imgs([(8, 8, 41, 32, True)], keep)
    opaque = C.c_int32(-1)
    assert F.hr_u32(L.dxb200_is_alpha_all_opaque(None, 1, C.byref(opaque))) == F.E_INVALIDARG
    assert F.hr_u32(L.dxb200_is_alpha_all_opaque(imgs, 1, None)) == F.E_INVALIDARG
    assert F.hr_u32(L.dxb200_is_alpha_all_opaque(imgs, 0, C.byref(opaque))) == F.E_INVALIDARG
    assert F.hr_u32(L.dxb200_is_alpha_all_opaque_device(imgs, 0, C.byref(opaque), None)) == F.E_INVALIDARG
    assert F.hr_u32(L.dxb200_is_alpha_all_opaque_device(imgs, 1, None, None)) == F.E_INVALIDARG


def test_every_dxgi_value_reads_pixels_only_with_alpha(ref):
    """For DXGI values 0..200: no alpha (the reference's HasAlpha) -> S_OK and 1 without a device; alpha and implemented -> a scan;
    alpha and not implemented -> E_NOT_SUPPORTED."""
    ref.L.probe_has_alpha.argtypes = [C.c_uint32]
    buf = np.zeros(256, np.uint8)
    implemented = set(A.PIXEL_FORMATS) | set(A.BLOCK_FORMATS)
    for fmt in range(201):
        hr, op = A.call(L.dxb200_is_alpha_all_opaque, capi.images([capi.Image(1, 1, fmt, 16, 16, buf.ctypes.data)]), 1)
        if not ref.L.probe_has_alpha(fmt):
            assert (hr, op) == (F.S_OK, 1), (fmt, hex(hr))
        elif fmt in implemented:
            assert hr == SCAN_HR, (fmt, hex(hr))
        else:
            assert hr == F.HRESULT_E_NOT_SUPPORTED, (fmt, hex(hr))


def test_mirror_answers_formats_without_alpha(mirror, ref):
    """ScratchImage::IsAlphaAllOpaque of the mirror: true for every implemented format without alpha (2D, array, cube, chain),
    false for an empty container, as the reference."""
    for fmt in A.NO_ALPHA_FORMATS:
        for (items, levels, cube) in ((1, 1, False), (3, 1, False), (1, 1, True), (2, 4, False)):
            n = capi.texture_layout(fmt, 16, 16, items * (6 if cube else 1), levels)[1]
            px = np.zeros(n, np.uint8)
            assert mirror.opaque(fmt, 16, 16, px, items, levels, cube) and ref.opaque(fmt, 16, 16, px, items, levels, cube), fmt
    mirror.L.probe_empty_is_alpha_all_opaque.restype = ref.L.probe_empty_is_alpha_all_opaque.restype = C.c_int
    assert mirror.L.probe_empty_is_alpha_all_opaque() == 0 and ref.L.probe_empty_is_alpha_all_opaque() == 0


def _from_ex_hr(c, planner):
    """(library HRESULT of dxb200_mipmaps_compress_from_ex with an answer pointer, planner HRESULT, planner's scan flag)"""
    opaque, scan = C.c_int32(-1), C.c_int32(-1)
    hr = F.hr_u32(L.dxb200_mipmaps_compress_from_ex(*c.args(), C.byref(opaque)))
    hp = F.hr_u32(planner.emul_plan_mipmaps_compress_from_ex(*c.args(), C.byref(opaque), C.byref(scan)))
    return hr, hp, scan.value


@pytest.mark.parametrize("name,kw,want", TABLE + [(v[0], v[1], F.S_OK) for v in VALID], ids=[t[0] for t in TABLE] + [v[0] for v in VALID])
def test_from_ex_hresults_are_from_s(emul, name, kw, want):
    """Every case of dxb200_mipmaps_compress_from's table returns the same HRESULT through _from_ex with an answer pointer, and
    with NULL (which is _from)."""
    c = Call(**kw)
    hr_from = F.hr_u32(L.dxb200_mipmaps_compress_from(*c.args()))
    hr, hp, scan = _from_ex_hr(c, emul)
    assert hr == hr_from and F.hr_u32(L.dxb200_mipmaps_compress_from_ex(*c.args(), None)) == hr_from, (name, hex(hr), hex(hr_from))
    assert hp == want, (name, hex(hp))
    if want == F.S_OK:
        assert scan == (1 if c.dst_fmt in A.BLOCK_FORMATS else 0)


def test_from_ex_scans_only_targets_with_alpha(emul):
    for dst, scan in ((71, 1), (77, 1), (98, 1), (80, 0), (83, 0), (95, 0)):
        c = Call(28 if dst != 95 else 10, 32, 32, dst_fmt=dst)
        hr, hp, s = _from_ex_hr(c, emul)
        assert hp == F.S_OK and s == scan, dst


# ---- emulator == reference ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", A.PIXEL_FORMATS)
def test_every_alpha_code(emul, ref, fmt):
    """Every code of the alpha field (fp32: the contract's special values) as a 1x1 image: the emulator answers like the reference,
    and the codes split into a non-opaque range below an opaque range."""
    codes = A.alpha_codes(fmt)
    want = A.per_code(ref.opaque, fmt, codes)
    got = A.per_code(lambda f, w, h, px: emul_opaque(emul, f, w, h, px), fmt, codes)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, (fmt, [int(codes[i]) for i in bad[:8]])
    assert want.any() and (~want).any(), fmt
    non, op = A.boundary_codes(fmt, want, codes)
    vals = A.code_values(fmt, codes)
    assert A.code_values(fmt, [non])[0] < A.code_values(fmt, [op])[0]
    finite = np.isfinite(vals)
    assert np.all(want[finite] == (vals[finite] >= A.code_values(fmt, [op])[0])), fmt


def boundary_cases(probe, fmt):
    """(largest non-opaque code, smallest opaque code, the code of 1.0 or the largest opaque one)"""
    codes = A.alpha_codes(fmt)
    want = A.per_code(probe.opaque, fmt, codes)
    non, op = A.boundary_codes(fmt, want, codes)
    vals = A.code_values(fmt, codes)
    fill = codes[want][np.argmax(np.where(np.isfinite(vals[want]), vals[want], -1))]
    return non, op, fill


@pytest.mark.parametrize("fmt", A.PIXEL_FORMATS)
def test_boundary_texels_anywhere(emul, ref, fmt):
    """The boundary codes at the first, middle and last texel of images 1, 5 and 257 wide, alone and as the last image of an array
    and of a mip chain; all-opaque images.  The emulator answers like the reference."""
    non, op, fill = boundary_cases(ref, fmt)
    for w, h in ((1, 1), (5, 3), (257, 2)):
        for code in (non, op):
            for where in ("first", "middle", "last"):
                px = A.placed(fmt, w, h, code, where, fill)
                assert emul_opaque(emul, fmt, w, h, px) == ref.opaque(fmt, w, h, px), (fmt, w, h, code, where)
                arr = np.concatenate([A.placed(fmt, w, h, fill, "first", fill)] * 2 + [px])
                assert emul_opaque(emul, fmt, w, h, arr, items=3) == ref.opaque(fmt, w, h, arr, items=3), (fmt, w, h, code, where)
        levels = min(3, F.count_mips(w, h))
        n = capi.texture_layout(fmt, w, h, 1, levels)[1] // F.BYTES_PER_PIXEL[fmt]
        chain = A.placed(fmt, n, 1, non, "last", fill)
        assert not ref.opaque(fmt, w, h, chain, levels=levels)
        assert emul_opaque(emul, fmt, w, h, chain, levels=levels) is False
        full = A.placed(fmt, w, h, fill, "first", fill)
        assert emul_opaque(emul, fmt, w, h, full) and ref.opaque(fmt, w, h, full)


@pytest.mark.parametrize("fmt", A.BLOCK_FORMATS)
def test_blocks_by_class(emul, ref, fmt):
    """Single blocks: random streams (BC7: stratified by mode 0-7 and the reserved mode), BC1 three-colour blocks, BC2 nibbles 13-15,
    BC3 palettes around 252 / 253 in both endpoint orders.  Each is a 4x4 image, a 3x2 image (partial block) and the last image
    of an array.  The emulator answers like the reference, and the classes reach both answers."""
    rng = np.random.default_rng(fmt)
    seen = set()
    opaque_block = None
    for b in A.block_corpus(fmt, rng):
        want = ref.opaque(fmt, 4, 4, b)
        seen.add(want)
        assert emul_opaque(emul, fmt, 4, 4, b) == want, (fmt, b.tobytes().hex())
        assert emul_opaque(emul, fmt, 3, 2, b) == ref.opaque(fmt, 3, 2, b), (fmt, b.tobytes().hex())
        if want and opaque_block is None:
            opaque_block = b
    assert seen == {False, True}, fmt
    for b in A.block_corpus(fmt, rng)[:16]:
        arr = np.concatenate([opaque_block, opaque_block, b])
        assert emul_opaque(emul, fmt, 4, 4, arr, items=3) == ref.opaque(fmt, 4, 4, arr, items=3)


@pytest.mark.parametrize("w,h", [(1, 1), (2, 3), (5, 7), (13, 9)])
@pytest.mark.parametrize("fmt", (71, 72))
def test_bc1_transparent_texels_in_the_padding(emul, ref, fmt, w, h):
    """BC1 three-colour blocks whose index-3 (transparent) texels lie only in the padding of partial blocks are opaque; one such
    texel inside the image is not."""
    pad = A.bc1_partial_image(w, h, inside=False)
    assert ref.opaque(fmt, w, h, pad) and emul_opaque(emul, fmt, w, h, pad)
    inside = A.bc1_partial_image(w, h, inside=True)
    assert not ref.opaque(fmt, w, h, inside) and not emul_opaque(emul, fmt, w, h, inside)


@pytest.mark.parametrize("fmt", A.BLOCK_FORMATS)
def test_reference_encoded_classes(emul, ref, oracle, fmt):
    """Blocks the reference's encoder makes from the contract's content classes, with alpha and made opaque, 32x32 and cut to
    30x29, as single images and as a chain."""
    for opaque in (False, True):
        for blocks in A.reference_encoded(oracle, fmt, opaque=opaque):
            for (w, h) in ((32, 32), (30, 29)):
                want = ref.opaque(fmt, w, h, blocks)
                assert emul_opaque(emul, fmt, w, h, blocks) == want, (fmt, opaque, w, h)
    blocks = A.reference_encoded(oracle, fmt, kinds=("alpha_uncorr",))[0]
    n = capi.texture_layout(fmt, 32, 32, 1, 3)[1]
    chain = np.zeros(n, np.uint8)           # level 0 the encoded blocks, the smaller levels zero blocks
    chain[:blocks.nbytes] = blocks
    assert emul_opaque(emul, fmt, 32, 32, chain, levels=3) == ref.opaque(fmt, 32, 32, chain, levels=3)
