"""GPU suite for the kernel routes of GenerateMipMaps and Resize.

dxb_launch_mip_chain (dxb_k_rows.cu) runs every level on one of five kernel families: k_mip_box3 (three BOX or 2:1 LINEAR
levels per pass), k_mip_tail (the levels from 64x64 down, one CTA per item), k_mip_sep (separable CUBIC), k_mip_tile (2D tiles)
or the generic k_mip_level.  The specialised families are compiled per filter, sRGB-ness and UNORM twin of a hot format (an sRGB
format runs its twin's kernels).  CASES is one table:
each case names its format, size, item count, filter flags, memory layout and the families it must launch, and every case runs

  - with DXB200_OPT_MIP_KERNELS = 0 (the routing users get): the per-family launch counters must move for exactly those families;
  - with DXB200_OPT_MIP_KERNELS = 1: only k_mip_level may launch, and the result must equal option 0's bit for bit.  Both options
    use the same device powf, so this checks the specialised kernels with sRGB too;
  - against the oracle (the unmodified reference): bit for bit without sRGB.  With sRGB the generic route is compared one level
    at a time (a levels = 2 call on the oracle's previous level, so errors do not add up): alpha exactly, RGB within one code for
    8-bit formats, one ulp for half and 2^-20 for fp32 (DESIGN.md section 3).

tests/test_cpu_mip_routes.py checks, without a GPU, that the table reaches every specialised instantiation the launcher compiles."""
import collections
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import oracle_lib

BOX, LIN, CUB, TRI, PT = F.TEX_FILTER_BOX, F.TEX_FILTER_LINEAR, F.TEX_FILTER_CUBIC, F.TEX_FILTER_TRIANGLE, F.TEX_FILTER_POINT
SRGB, SRGB_IN = F.TEX_FILTER_SRGB, F.TEX_FILTER_SRGB_IN
MODE_MASK = 0xF00000
HOT = (28, 29, 10, 2, 61, 41, 87)                   # on_mip_format in dxb_k_rows.cu
FAMILIES = ("k_mip_box3", "k_mip_tail", "k_mip_sep", "k_mip_tile", "k_mip_level")


def _format_tables():
    """(formats whose filters honour TEX_FILTER_SRGB_IN / _OUT, sRGB formats that always convert, {sRGB format: its UNORM twin}),
    read from dxb_resolve_srgb_linear and dxb_make_linear in dxb_formats.h: the tables the launcher resolves a call's sRGB steps
    and compiles its specialised kernels with"""
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "directxtex_b200", "csrc", "dxb_formats.h")).read()
    value = {k: int(v) for k, v in re.findall(r"\bDXB_FMT_(\w+) = (\d+)", src)}
    body = re.search(r"dxb_resolve_srgb_linear\(uint32_t flags, uint32_t fmt\)\s*\{(.*?)\n\}", src, re.S).group(1)
    always, keep = re.findall(r"((?:case DXB_FMT_\w+:\s*)+)return flags", body)[:2]
    names = lambda block: {value[n] for n in re.findall(r"case DXB_FMT_(\w+):", block)}
    body = re.search(r"dxb_make_linear\(uint32_t fmt\)\s*\{(.*?)\n\}", src, re.S).group(1)
    twin = {value[a]: value[b] for a, b in re.findall(r"case DXB_FMT_(\w+):\s*return DXB_FMT_(\w+);", body)}
    return names(keep), names(always), twin


SRGB_KEEP, SRGB_ALWAYS, TWIN = _format_tables()
BOX3, TAIL, SEP, TILE, LEVEL = FAMILIES

# layout of device images: item -> (row pitch beyond the tight one, offset of the base from a 256-byte boundary)
LAYOUTS = {
    "tight": lambda item: (0, 0),
    "pad16": lambda item: (16, 0),
    "off4": lambda item: (4, 4),
    "mixed": lambda item: (0, 0) if item == 0 else (4, 4),
}

Case = collections.namedtuple("Case", "fmt w h items fl layout resize fams")


def case(fmt, w, h, items, fl, fams, layout="host", resize=None):
    return Case(fmt, w, h, items, fl, layout, resize, frozenset(fams))


def case_id(c):
    op = "resize%dx%d" % c.resize if c.resize else "mips"
    return "%s-f%d-%dx%dx%d-%06x-%s" % (op, c.fmt, c.w, c.h, c.items, c.fl, c.layout)


def _cases():
    cs = []
    # every specialised instantiation: per hot format, sRGB off and on (format 29 is always sRGB)
    for fmt in HOT:
        for s in ((SRGB,) if fmt == 29 else (0, SRGB)):
            cs += [case(fmt, 256, 256, 1, BOX | s, (BOX3, TAIL)),
                   case(fmt, 256, 128, 3, LIN | s, (BOX3, TAIL)),
                   case(fmt, 128, 128, 1, CUB | s, (SEP, TAIL)),
                   case(fmt, 2048, 4, 3, BOX | s, (TILE, TAIL)),             # tile BOX, with the stale-row quirk from level 3 on
                   case(fmt, 333, 97, 1, s, (TILE, TAIL)),                   # filter 0 on a non-power-of-two size = LINEAR
                   case(fmt, 200, 120, 1, CUB | s, (TILE,), resize=(50, 30))]    # CUBIC at 4:1: tile
    # filters, sRGB variants and a non-hot format on the generic kernel
    for fl in (TRI, PT, TRI | SRGB, LIN | SRGB_IN, BOX | SRGB_IN, CUB | SRGB_IN):
        cs += [case(28, 128, 64, 3, fl, (LEVEL,)), case(2, 64, 64, 1, fl, (LEVEL,))]
    cs += [case(29, 96, 80, 1, CUB | SRGB_IN, (SEP, TAIL)),                   # format 29 turns SRGB_IN into both steps
           case(88, 256, 256, 1, BOX | SRGB, (LEVEL,)), case(88, 100, 60, 3, CUB, (LEVEL,)),
           case(28, 128, 128, 3, CUB | F.TEX_FILTER_WRAP, (SEP, TAIL)), case(10, 128, 64, 1, CUB | F.TEX_FILTER_MIRROR, (SEP, TAIL)),
           case(28, 256, 256, 1, LIN | F.TEX_FILTER_WRAP, (BOX3, TAIL))]
    # the packed formats whose sRGB steps run on the generic kernel only
    cs += [case(26, 64, 32, 3, BOX | SRGB, (LEVEL,)), case(67, 40, 24, 1, CUB | SRGB, (LEVEL,)), case(85, 40, 24, 3, 0 | SRGB, (LEVEL,)),
           case(86, 64, 32, 1, TRI | SRGB, (LEVEL,)), case(115, 64, 32, 3, LIN | SRGB, (LEVEL,)), case(115, 40, 24, 1, CUB | SRGB, (LEVEL,), resize=(20, 30))]
    # partial tiles, wide / short, tall
    cs += [case(28, 1023, 767, 1, 0, (TILE, TAIL)), case(41, 1023, 767, 1, CUB, (SEP, TAIL)), case(10, 66, 130, 3, CUB | SRGB, (SEP, TAIL)),
           case(61, 333, 97, 3, CUB, (SEP, TAIL)), case(2, 66, 130, 1, 0, (TILE, TAIL)),
           case(61, 1024, 2, 3, BOX, (TILE, TAIL)), case(2, 1024, 2, 1, BOX | SRGB, (TILE, TAIL)), case(87, 2048, 4, 3, LIN, (TILE, TAIL)),
           case(28, 4, 2048, 3, BOX, (TILE, TAIL)), case(10, 4, 2048, 1, CUB, (SEP, TAIL)), case(61, 1, 4096, 1, BOX, (TILE, TAIL)),
           case(41, 1, 4096, 3, LIN | SRGB, (TILE, TAIL)),
           case(61, 1, 1 << 20, 1, BOX, (LEVEL, TILE, TAIL)), case(61, 1, 1 << 20, 1, LIN, (LEVEL, TILE, TAIL))]   # tile g.y > 65535
    # caller layouts on the device API
    for lay in ("tight", "pad16"):
        cs += [case(61, 256, 256, 3, BOX, (BOX3, TAIL), lay), case(28, 256, 128, 1, LIN | SRGB, (BOX3, TAIL), lay),
               case(2, 128, 128, 3, CUB, (SEP, TAIL), lay), case(10, 2048, 4, 1, BOX, (TILE, TAIL), lay)]
    cs += [case(61, 256, 256, 3, BOX, (TILE, TAIL), "off4"), case(28, 256, 128, 1, LIN | SRGB, (TILE, TAIL), "off4"),
           case(87, 128, 128, 3, CUB, (SEP, TAIL), "off4"), case(10, 128, 128, 1, CUB, (TILE, TAIL), "off4"),
           case(2, 2048, 4, 3, BOX, (TILE, TAIL), "off4"), case(41, 333, 97, 1, 0, (TILE, TAIL), "off4"),
           case(28, 256, 256, 2, BOX | SRGB, (TILE, TAIL), "mixed"), case(2, 1024, 2, 2, BOX, (TILE, TAIL), "mixed"),
           case(10, 128, 128, 2, CUB | SRGB, (TILE, TAIL), "mixed"), case(61, 128, 128, 2, CUB, (SEP, TAIL), "mixed")]
    # resize routes
    cs += [case(28, 300, 90, 3, CUB, (SEP,), resize=(100, 30)), case(2, 300, 90, 1, CUB | SRGB, (SEP,), resize=(100, 30)),
           case(28, 301, 91, 3, CUB, (TILE,), resize=(100, 30)), case(10, 400, 120, 1, CUB | SRGB, (TILE,), resize=(100, 30)),
           case(61, 40, 30, 3, CUB, (SEP,), resize=(120, 90)), case(41, 97, 61, 1, CUB | F.TEX_FILTER_MIRROR, (SEP,), resize=(97, 61)),
           case(87, 128, 64, 3, 0, (TILE,), resize=(64, 32)), case(2, 128, 64, 1, BOX | SRGB, (TILE,), resize=(64, 32)),
           case(29, 100, 60, 1, LIN, (TILE,), resize=(37, 91)), case(10, 100, 60, 3, LIN | F.TEX_FILTER_WRAP, (TILE,), resize=(300, 20)),
           case(28, 100, 60, 1, TRI, (LEVEL,), resize=(37, 91)), case(61, 100, 60, 3, PT, (LEVEL,), resize=(37, 91)),
           case(28, 128, 64, 2, BOX, (TILE,), "mixed", resize=(64, 32)), case(10, 200, 120, 3, CUB, (TILE,), "pad16", resize=(50, 30)),
           case(28, 300, 90, 1, CUB | SRGB, (SEP,), "off4", resize=(100, 30)), case(2, 300, 90, 1, CUB, (TILE,), "off4", resize=(100, 30))]
    # large extents: fp32 coordinates lose their fraction above 2^23 (DESIGN.md section 0, a17 / f-2)
    cs += [case(61, 8388616, 8, 1, 0, (TILE, TAIL)), case(61, 8388616, 8, 1, LIN, (TILE, TAIL)),
           case(41, 12582912, 1, 1, CUB, (TILE,), resize=(12582912, 1)), case(41, 12582913, 1, 1, CUB, (TILE,), resize=(12582912, 1))]
    # more items than one grid's z extent: uniform_batch declines, k_mip_level covers the levels above the tail
    cs += [case(61, 128, 8, 70000, BOX, (LEVEL, TAIL), "tight")]
    return cs


CASES = _cases()


# ---- what a case exercises ------------------------------------------------------------------------------------------------
def ispow2(x):
    return x > 0 and not (x & (x - 1))


def srgb_bits(fmt, fl):
    """the sRGB steps the filters take (dxb_resolve_srgb_linear)"""
    if fmt in SRGB_ALWAYS:
        return SRGB
    return fl & SRGB if fmt in SRGB_KEEP else 0


def mode_of(c):
    m = c.fl & MODE_MASK
    if m:
        return m
    if c.resize:
        return BOX if (c.resize[0] * 2, c.resize[1] * 2) == (c.w, c.h) else LIN
    return BOX if ispow2(c.w) and ispow2(c.h) else LIN


def instantiations(c):
    """(family, format, mode, sRGB, LIN) of every specialised kernel the case launches with option 0; format is the case's
    UNORM twin (dxb_make_linear), mode is 0 where the template has no mode parameter (k_mip_box3, k_mip_sep)"""
    fmt, srgb, mode = TWIN.get(c.fmt, c.fmt), srgb_bits(c.fmt, c.fl) == SRGB, mode_of(c)
    out = set()
    for fam in c.fams:
        if fam == BOX3:
            out.add(("box3", fmt, 0, srgb, mode == LIN))
        elif fam == SEP:
            out.add(("sep", fmt, 0, srgb, False))
        elif fam in (TILE, TAIL):
            out.add((fam[len("k_mip_"):], fmt, mode, srgb, False))
    return out


# ---- running a case -------------------------------------------------------------------------------------------------------
def levels_of(c):
    return [(c.w, c.h), c.resize] if c.resize else [(lw, lh) for (_, lw, lh, _, _) in F.mip_chain_layout(c.fmt, c.w, c.h)[0]]


def sources(c):
    """level 0 of each item: different content per item, at most 3 distinct images (item i uses source i % 3)"""
    rng = np.random.default_rng(zlib.crc32(case_id(c).encode()))
    return [oracle_lib.random_image(c.fmt, c.w, c.h, rng).view(np.uint8).reshape(-1) for _ in range(min(c.items, 3))]


def tight_bytes(fmt, w, h):
    return F.compute_pitch(fmt, w, h)[1]


def run_host(c, srcs):
    """per level, an (items, bytes) array of the tight images (level 0 included)"""
    items = [srcs[i % len(srcs)] for i in range(c.items)]
    if c.resize:
        return [np.stack(items), np.stack(capi.resize_images(items, c.w, c.h, c.fmt, c.resize[0], c.resize[1], c.fl))]
    layout, _ = F.mip_chain_layout(c.fmt, c.w, c.h)
    chains = np.stack(capi.generate_mipmaps_images(items, c.w, c.h, c.fmt, c.fl))
    return [chains[:, off:off + sl] for (off, _, _, _, sl) in layout]


def run_device(c, srcs):
    """the device API on torch buffers laid out per c.layout: one buffer per level holding every item at a 16-byte-aligned
    stride; same result structure as run_host"""
    import torch
    fmt, bpp, sizes = c.fmt, F.BYTES_PER_PIXEL[c.fmt], levels_of(c)
    geo = [LAYOUTS[c.layout](i) for i in range(c.items)]
    groups = [(g, np.array([i for i in range(c.items) if geo[i] == g])) for g in sorted(set(geo))]
    strides = [((max(base + (lw * bpp + pad) * lh for (pad, base) in set(geo)) + 15) & ~15) for (lw, lh) in sizes]
    bufs = [torch.zeros(c.items * st_, dtype=torch.uint8, device="cuda") for st_ in strides]

    def view(host, l, pad, base, idx):
        """the pixel rows of items idx at level l: (items, height, width * bpp), a copy"""
        lw, lh = sizes[l]
        pitch = lw * bpp + pad
        return host.reshape(c.items, strides[l])[idx, base:base + pitch * lh].reshape(len(idx), lh, pitch)[:, :, :lw * bpp]
    host0 = np.zeros(c.items * strides[0], np.uint8)
    src = np.stack(srcs)
    (w0, h0) = sizes[0]
    for (pad, base), idx in groups:          # level 0: one padded host image of every item, one upload
        img = src[idx % len(srcs)].reshape(len(idx), h0, w0 * bpp)
        host0.reshape(c.items, strides[0])[idx, base:base + (w0 * bpp + pad) * h0] = np.pad(img, ((0, 0), (0, 0), (0, pad))).reshape(len(idx), -1)
    bufs[0].copy_(torch.from_numpy(host0))
    recs = np.zeros((len(sizes), c.items, 6), np.uint64)        # dxb200_image: width, height, format, rowPitch, slicePitch, pixels
    for l, (lw, lh) in enumerate(sizes):
        pitch = np.array([lw * bpp + pad for (pad, _) in geo], np.uint64)
        recs[l, :, 0], recs[l, :, 1], recs[l, :, 2], recs[l, :, 3], recs[l, :, 4] = lw, lh, fmt, pitch, pitch * np.uint64(lh)
        recs[l, :, 5] = np.uint64(bufs[l].data_ptr()) + np.arange(c.items, dtype=np.uint64) * np.uint64(strides[l]) + \
            np.array([base for (_, base) in geo], np.uint64)
    assert C.sizeof(capi.Image) == 48
    P = C.POINTER(capi.Image)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if c.resize:
        s_, d_ = np.ascontiguousarray(recs[0]), np.ascontiguousarray(recs[1])
        hr = capi.lib.dxb200_resize_device(s_.ctypes.data_as(P), c.items, c.fl, d_.ctypes.data_as(P), st)
    else:
        t = np.ascontiguousarray(recs.transpose(1, 0, 2))      # item-major, mip-minor
        hr = capi.lib.dxb200_generate_mipmaps_device(t.ctypes.data_as(P), c.items, len(sizes), c.fl, st)
    assert F.hr_u32(hr) == 0, (case_id(c), hex(F.hr_u32(hr)), capi.last_error())
    torch.cuda.synchronize()
    out = []
    for l, (lw, lh) in enumerate(sizes):
        host = bufs[l].cpu().numpy()
        lvl = np.empty((c.items, lw * lh * bpp), np.uint8)
        for (pad, base), idx in groups:
            lvl[idx] = view(host, l, pad, base, idx).reshape(len(idx), -1)
        out.append(lvl)
    return out


def run(c, srcs, option):
    """(per level an (items, bytes) array, {family: launches}) with DXB200_OPT_MIP_KERNELS = option"""
    before = {f: capi.kernel_launch_count(f) for f in FAMILIES}
    assert capi.lib.dxb200_set_option(capi.OPT_MIP_KERNELS, option) == 0
    try:
        got = run_host(c, srcs) if c.layout == "host" else run_device(c, srcs)
    finally:
        capi.lib.dxb200_set_option(capi.OPT_MIP_KERNELS, 0)
    return got, {f: capi.kernel_launch_count(f) - before[f] for f in FAMILIES if capi.kernel_launch_count(f) != before[f]}


def oracle_levels(oracle, c, src):
    if c.resize:
        hr, out = oracle.resize(src, c.w, c.h, c.fmt, c.resize[0], c.resize[1], c.fl)
        assert hr == 0, (case_id(c), hex(hr))
        return [src, out]
    hr, chain = oracle.generate_mipmaps(src, c.w, c.h, c.fmt, c.fl)
    assert hr == 0, (case_id(c), hex(hr))
    return [chain[off:off + sl] for (off, _, _, _, sl) in F.mip_chain_layout(c.fmt, c.w, c.h)[0]]


# ---- the sRGB tolerance (DESIGN.md section 3) -----------------------------------------------------------------------------
# packed formats: (shift, bits) of the colour fields, of the alpha field (None: no alpha).  R11G11B10's fields are unsigned small
# floats, so their codes are ordered like their values and one code is one ulp.
PACKED = {85: (((11, 5), (5, 6), (0, 5)), None), 86: (((10, 5), (5, 5), (0, 5)), (15, 1)), 115: (((8, 4), (4, 4), (0, 4)), (12, 4)),
          26: (((0, 11), (11, 11), (22, 10)), None)}


def srgb_diff(fmt, got, want):
    """largest RGB difference in the format's unit (codes, half ulps, mantissa steps of R9G9B9E5's larger shared exponent, or
    absolute fp32); asserts that alpha is identical"""
    if fmt in PACKED or fmt == 67:
        dt = np.uint16 if F.BYTES_PER_PIXEL[fmt] == 2 else np.uint32
        g, w = got.view(dt).astype(np.int64), want.view(dt).astype(np.int64)
        field = lambda a, f: (a >> f[0]) & ((1 << f[1]) - 1)
        if fmt == 67:
            eg, ew = field(g, (27, 5)), field(w, (27, 5))
            step = np.exp2(np.maximum(eg, ew) - 24.0)
            return max(float((np.abs(field(g, (k, 9)) * np.exp2(eg - 24.0) - field(w, (k, 9)) * np.exp2(ew - 24.0)) / step).max())
                       for k in (0, 9, 18))
        colour, alpha = PACKED[fmt]
        if alpha:
            assert np.array_equal(field(g, alpha), field(w, alpha)), "alpha differs"
        return int(max(np.abs(field(g, f) - field(w, f)).max() for f in colour))
    bpp = F.BYTES_PER_PIXEL[fmt]
    dt = {2: np.float32, 41: np.float32, 10: np.uint16}.get(fmt, np.uint8)
    n = bpp // np.dtype(dt).itemsize
    assert bpp in (1, 4, 8, 16) and n in (1, 4), fmt
    if n == 4:
        assert np.array_equal(got.reshape(-1, bpp)[:, bpp * 3 // 4:], want.reshape(-1, bpp)[:, bpp * 3 // 4:]), "alpha differs"
    g, w = got.view(dt).reshape(-1, n)[:, :3], want.view(dt).reshape(-1, n)[:, :3]
    if dt == np.float32:
        return float(np.abs(g.astype(np.float64) - w).max())
    if dt == np.uint16:            # half: distance in ulps on the sign-magnitude order
        key = lambda a: np.where(a & 0x8000, -(a.astype(np.int32) & 0x7FFF), a.astype(np.int32))
        return int(np.abs(key(g) - key(w)).max())
    return int(np.abs(g.astype(np.int32) - w).max())


SRGB_BOUND = {2: 2.0 ** -20, 41: 2.0 ** -20}      # every other format here: one code / ulp / mantissa step


def check_srgb_generic(oracle, c, srcs, want):
    """the generic kernel one level at a time on the oracle's previous level, against the oracle's level; returns the largest
    RGB difference.  Levels whose BOX source is one row high read the stale row of an earlier level (dxb_mip_box) that a
    levels = 2 call does not have: those are checked through option 0 == option 1 and the non-sRGB cases only."""
    fmt, worst, sizes = c.fmt, 0, levels_of(c)
    bound = SRGB_BOUND.get(fmt, 1)
    fl = (c.fl & ~MODE_MASK) | mode_of(c)          # a lower level alone could resolve filter 0 to another mode
    assert capi.lib.dxb200_set_option(capi.OPT_MIP_KERNELS, 1) == 0
    try:
        for l in range(1, len(sizes)):
            (sw, sh), (dw, dh) = sizes[l - 1], sizes[l]
            if mode_of(c) == BOX and sh == 1 and sw > 1 and not c.resize:
                continue
            prev = [want[k][l - 1] for k in range(len(srcs))]
            if c.resize:
                got = capi.resize_images(prev, sw, sh, fmt, dw, dh, fl)
            else:
                chains = capi.generate_mipmaps_images(prev, sw, sh, fmt, fl, levels=2)
                got = [ch[tight_bytes(fmt, sw, sh):] for ch in chains]
            for k in range(len(srcs)):
                d = srgb_diff(fmt, got[k], want[k][l])
                assert d <= bound, (case_id(c), l, k, d)
                worst = max(worst, d)
    finally:
        capi.lib.dxb200_set_option(capi.OPT_MIP_KERNELS, 0)
    return worst


pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _init():
    assert capi.lib.dxb200_init(0) == 0


def check_route_and_result(oracle, c, srcs):
    """case c on level-0 images srcs (run's item i takes srcs[i % len(srcs)]): option 0 launches exactly c.fams, option 1 only
    k_mip_level, the two agree bit for bit and both agree with the oracle (sRGB: check_srgb_generic).  Returns option 0's levels."""
    got0, fam0 = run(c, srcs, 0)
    got1, fam1 = run(c, srcs, 1)
    print("%s option 0: %s  option 1: %s" % (case_id(c), fam0, fam1))
    assert set(fam0) == set(c.fams), (case_id(c), fam0)
    assert set(fam1) == {LEVEL}, (case_id(c), fam1)
    for l in range(len(got0)):
        assert np.array_equal(got0[l], got1[l]), (case_id(c), "option 0 != option 1", l)
    want = [oracle_levels(oracle, c, s) for s in srcs]
    if srgb_bits(c.fmt, c.fl):
        print("%s largest sRGB difference %s" % (case_id(c), check_srgb_generic(oracle, c, srcs, want)))
        return got0
    pick = np.arange(c.items) % len(srcs)
    for l in range(len(got0)):
        bad = np.nonzero((got0[l] != np.stack([w[l] for w in want])[pick]).any(1))[0]
        assert bad.size == 0, (case_id(c), "differs from the oracle", "level", l, "items", bad[:5])
    return got0


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_route_and_result(oracle, c):
    check_route_and_result(oracle, c, sources(c))
