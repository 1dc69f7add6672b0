"""A dense sweep of Resize and GenerateMipMaps extents: one case list shared by tests/test_cpu_resize_sweep.py and
tests/test_gpu_resize_sweep.py.

Every filter chooses its taps from fp32 coordinates that depend only on the (source, destination) extent pair of an axis
(dxb_linear_entry / dxb_cubic_entry in dxb_mips.cuh, dxb_sep_entry in dxb_k_rows.cu, POINT's 16.16 step in dxb_mip_point,
TRIANGLE's host gather lists), and the specialised kernels depend on the pair too: k_mip_sep fills 32 x 16 destination tiles
from row buffers sized for 3:1, the CUBIC k_mip_tile reuses filtered rows across DXB_CUBIC_KY outputs, k_mip_tail runs the ends
of chains, launch_box3 declines sizes that are not multiples of 8.  The sweep walks the pairs where tile edges meet ratio edges.
Resize pairs are per axis: one axis sweeps while the other holds a small fixed pair, plus a diagonal set where both vary:

  dense      every (s, d) with 1 <= s, d <= 48;
  boundary   s at the tile edges 31 .. 4097, d in {s, s +- 1, s / 2 both ways, ceil(s / 3), ceil(s / 3) - 1 (just past 3:1),
             s / 3 + 1, 2s, 3s, 7s}; and d at the tile edges 7 .. 65 with s = 3d, 3d + 1 and 4d + 3;
  random     seeded pairs up to 4096, up and down;
  long       s in {65535, 65536, 65537, 131073} with the other axis 1, 2 or 3 pixels (POINT's sw << 16 leaves 32 bits); BOX
             with the other axis 2 -> 1, so that it runs where the long axis halves;
  diagonal   a seeded subset of dense pairs on both axes at once.

Each runs POINT, LINEAR, CUBIC, TRIANGLE, filter 0 and BOX (which the reference refuses with E_FAIL unless both axes are
exactly 2:1), on R32G32B32A32_FLOAT and R8G8B8A8_UNORM.  LINEAR, CUBIC, TRIANGLE and filter 0 also run every per-axis WRAP /
MIRROR word of tests/address_modes.py on every one-axis pair with an extent of 5 or less (on one of the two formats, in turn),
and WRAP and MIRROR on a seeded eighth of their other resizes; R16G16B16A16_FLOAT, R10G10B10A2_UNORM (generic
kernel only) and R8G8B8A8_UNORM with TEX_FILTER_SRGB on seeded subsets.  Mip chains: every base width 1 .. 130 with height
1, 2, 3, 7 or 64, the transposes and the squares, under every filter, except BOX chains of one-row bases wider than a pixel,
where the reference reads a scanline it never wrote (box_row_undefined).

route() states which kernel family dxb_launch_mip_chain launches for each level, from the same facts it reads (hot format,
filter mode, sRGB steps, uniform batch, pixel alignment, source <= 3 x destination, the extent limit of k_mip_sep and the
grid's y limit); its constants are read from dxb_k_rows.cu and tests/test_cpu_resize_sweep.py pins its predicates there and
holds it to every case of the route tables of tests/test_gpu_mip_routes.py and tests/address_modes.py."""
import collections
import functools
import hashlib
import os
import re

import numpy as np

from directxtex_b200 import formats as F
from tests import address_modes as A, test_gpu_mip_routes as R
from tests.test_cpu_mip_routes import _sep_constants

BOX, LIN, CUB, TRI, PT = R.BOX, R.LIN, R.CUB, R.TRI, R.PT
SRGB = R.SRGB
BOX3, TAIL, SEP, TILE, LEVEL = R.FAMILIES
FILTERS = (PT, LIN, CUB, TRI, 0, BOX)
FILTER_NAME = {PT: "POINT", LIN: "LINEAR", CUB: "CUBIC", TRI: "TRIANGLE", 0: "default", BOX: "BOX"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- what dxb_launch_mip_chain reads ----------------------------------------------------------------------------------
def filter_of(c):
    return c.fl & R.MODE_MASK


def _cubic_rows():
    src = open(os.path.join(ROOT, "directxtex_b200", "csrc", "dxb_k_rows.cu")).read()
    return int(re.search(r"#define DXB_CUBIC_KY (\d+)u", src).group(1))


SEP_TW, SEP_TH, SEP_MAXC, SEP_MAXR, SEP_MAX_EXTENT = _sep_constants()      # read from dxb_k_rows.cu
CUBIC_KY = _cubic_rows()
TILE_ROWS = 8               # rows of a k_mip_tile / k_mip_box3 CTA (blk = 32 x 8)
GRID_Y = 65535              # largest gridDim.y
UNIFORM_ITEMS = 65535       # uniform_batch: at most one grid's z extent of items
TAIL_EXTENT = 64            # k_mip_tail from the first level whose source is at most 64 x 64
BOX3_LIN_EXTENT = 1 << 23   # launch_box3 declines LINEAR above this extent


def _aligned(layout, items, fmt, width, bytes_):
    """vec_aligned of every item's image `width` pixels wide, under the test_gpu_mip_routes layout (host staging: tight rows on
    256-byte boundaries; device buffers hold items at 16-byte-aligned strides)"""
    v = min(bytes_, 16)
    bpp = F.BYTES_PER_PIXEL[fmt]
    geo = {(0, 0)} if layout == "host" else {R.LAYOUTS[layout](i) for i in range(items)}
    return all(base % v == 0 and (width * bpp + pad) % v == 0 for (pad, base) in geo)


def _box3(c, sizes, l, lin):
    (sw, sh), bpp = sizes[l - 1], F.BYTES_PER_PIXEL[c.fmt]
    if sw % 8 or sh % 8 or sw < 8 or sh < 8 or c.items > UNIFORM_ITEMS:
        return False
    if sizes[l:l + 3] != [(sw >> k, sh >> k) for k in (1, 2, 3)]:
        return False
    if not all(_aligned(c.layout, c.items, c.fmt, sw >> k, b) for k, b in ((0, 8 * bpp), (1, 4 * bpp), (2, 2 * bpp), (3, bpp))):
        return False
    if lin and max(sw, sh) > BOX3_LIN_EXTENT:
        return False
    return -(-(sh // 8) // TILE_ROWS) <= GRID_Y


def _level(c, sizes, l, special, mode):
    (sw, sh), (dw, dh) = sizes[l - 1], sizes[l]
    if special and c.items <= UNIFORM_ITEMS:
        pix = _aligned(c.layout, c.items, c.fmt, sw, F.BYTES_PER_PIXEL[c.fmt])
        if (mode == CUB and pix and max(sw, sh, dw, dh) <= SEP_MAX_EXTENT and sw <= 3 * dw and sh <= 3 * dh and
                -(-dh // SEP_TH) <= GRID_Y):
            return SEP
        if -(-dh // (TILE_ROWS * CUBIC_KY if mode == CUB else TILE_ROWS)) <= GRID_Y:
            return TILE
    return LEVEL


def route(c, option=0):
    """[(family, first level, levels)] of the launches of case c (a test_gpu_mip_routes.Case) with DXB200_OPT_MIP_KERNELS =
    option; [] when the call fails in planning (BOX on sizes that do not halve exactly: E_FAIL)"""
    sizes, mode = R.levels_of(c), R.mode_of(c)
    (sw, sh), (dw, dh) = sizes[0], sizes[1]
    if mode == BOX and not ((sw, sh) == (2 * dw, 2 * dh) if c.resize else R.ispow2(sw) and R.ispow2(sh)):
        return []
    levels = len(sizes)
    special = (option == 0 and c.fmt in R.HOT and mode in (BOX, LIN, CUB) and R.srgb_bits(c.fmt, c.fl) in (0, SRGB))
    tail_start = next((l for l in range(1, levels) if max(sizes[l - 1]) <= TAIL_EXTENT), levels)
    tail = special and levels - tail_start >= 2
    fused = special and mode != CUB and levels >= 4
    out, l = [], 1
    while l < levels:
        if fused and l + 2 < levels and max(sizes[l - 1]) > TAIL_EXTENT and _box3(c, sizes, l, mode == LIN):
            out.append((BOX3, l, 3))
            l += 3
        elif tail and l >= tail_start:
            out.append((TAIL, l, levels - l))
            break
        else:
            out.append((_level(c, sizes, l, special, mode), l, 1))
            l += 1
    return out


def families(c, option=0):
    return frozenset(f for (f, _, _) in route(c, option))


def case(fmt, w, h, fl, resize=None, layout="host", items=1):
    """a test_gpu_mip_routes.Case whose families are route()'s"""
    c = R.case(fmt, w, h, items, fl, (), layout, resize)
    return c._replace(fams=families(c))


def with_layout(c, layout):
    return case(c.fmt, c.w, c.h, c.fl, c.resize, layout, c.items)


# ---- the pairs --------------------------------------------------------------------------------------------------------
EDGES = (31, 32, 33, 47, 48, 49, 63, 64, 65, 95, 96, 97, 127, 129, 255, 257, 1023, 1025, 4097)
LONG = (65535, 65536, 65537, 131073)
THIN = ((1, 1), (2, 3), (3, 1))                  # the other axis of the long pairs
DENSE = [(s, d) for s in range(1, 49) for d in range(1, 49)]


def boundary_dests(s):
    c3 = -(-s // 3)
    return sorted({s, s - 1, s + 1, s // 2, -(-s // 2), c3, c3 - 1, s // 3 + 1, 2 * s, 3 * s, 7 * s} - {0})


def long_dests(s):
    """7s: from 131073 on, 8-row tiles of the destination exceed the grid's y limit (k_mip_level takes LINEAR and BOX)"""
    c3 = -(-s // 3)
    return sorted({s, s - 1, s + 1, s // 2, c3, c3 - 1, 2 * s, 7 * s})


BOUNDARY = [(s, d) for s in EDGES for d in boundary_dests(s)]
# destinations at the tile edges reduced at exactly 3:1, just past it and at 4:1 + 3
BOUNDARY += [(s, d) for d in (7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65) for s in (3 * d, 3 * d + 1, 4 * d + 3)]
_rng = np.random.default_rng(2024)
RANDOM = [(int(a), int(b)) for a, b in _rng.integers(1, 4097, (300, 2))]
_perm = _rng.permutation(len(DENSE))
DIAGONAL = [(DENSE[i], DENSE[_perm[i]]) for i in range(0, len(DENSE), 4)]


def fixed_pair(flt):
    """the other axis of a one-axis sweep: 2:1 where BOX (and filter 0 = BOX) needs it, else 5 -> 3"""
    return (6, 3) if flt in (BOX, 0) else (5, 3)


def thin_pairs(flt, i, j):
    """the other axis of long pair j of long extent i: every THIN pair for POINT, 2 -> 1 for BOX (so that the 2:1 long pairs
    run), one THIN pair in turn for the other filters"""
    return {PT: THIN, BOX: ((2, 1),)}.get(flt, (THIN[(i + j) % len(THIN)],))


def _pick(key, n):
    """a seeded 1-in-n choice"""
    return int.from_bytes(hashlib.blake2b(key.encode(), digest_size=8).digest(), "little") % n == 0


def _resize_base(fmt, flt):
    """[(case, the swept (s, d) pair, the swept axis)]: every pair on the U axis (0) and on the V axis (1), the other axis at
    fixed_pair; the long pairs on both axes over thin_pairs and the diagonal set (axis None: no single swept axis)"""
    fs, fd = fixed_pair(flt)
    out = []
    for s, d in DENSE + BOUNDARY + RANDOM:
        out += [(case(fmt, s, fs, flt, (d, fd)), (s, d), 0), (case(fmt, fs, s, flt, (fd, d)), (s, d), 1)]
    for i, s in enumerate(LONG):
        for j, d in enumerate(long_dests(s)):
            for ts, td in thin_pairs(flt, i, j):
                out += [(case(fmt, s, ts, flt, (d, td)), (s, d), None), (case(fmt, ts, s, flt, (td, d)), (s, d), None)]
    for (s, d), (t, e) in DIAGONAL:
        if flt in (BOX, 0):
            t = 2 * e                   # BOX / filter 0: the second axis at 2:1
        out.append((case(fmt, s, t, flt, (d, e)), (s, d), None))
    return out


# Address words.  On a one-axis sweep whose pair has an extent of 5 or less, every word of tests/address_modes.py, on one of the
# two formats (word_format); on every other resize of those two formats, WRAP and MIRROR for a seeded eighth.  BOX and POINT
# read no address bit.
WORD_FILTERS = (LIN, CUB, TRI, 0)
WORDS = tuple(w for w in A.WORDS if w)


def small_pair(pair, axis):
    return axis is not None and min(pair) <= 5


def word_format(pair, axis):
    """the format that runs every word on a small pair: R32G32B32A32_FLOAT and R8G8B8A8_UNORM in turn"""
    return (2, 28)[(pair[0] + pair[1] + axis) % 2]


def _words(c, pair, axis):
    if filter_of(c) not in WORD_FILTERS:
        return []
    if small_pair(pair, axis):
        return list(WORDS) if c.fmt == word_format(pair, axis) else []
    return [A.WRAP, A.MIRROR] if _pick(R.case_id(c) + "wrap", 8) else []


def _resize_cases():
    cs = []
    for flt in FILTERS:
        for fmt in (2, 28):
            for c, pair, axis in _resize_base(fmt, flt):
                cs += [c] + [case(fmt, c.w, c.h, c.fl | w, c.resize) for w in _words(c, pair, axis)]
        # the other formats and sRGB on seeded subsets of the base pairs
        for c, _, _ in _resize_base(2, flt):
            if max(c.w * c.h, c.resize[0] * c.resize[1]) > 1 << 20:
                continue
            for fmt, fl, n in ((10, 0, 8), (24, 0, 12), (28, SRGB, 12)):
                if _pick("%s-%d-%x" % (R.case_id(c), fmt, fl), n):
                    cs.append(case(fmt, c.w, c.h, c.fl | fl, c.resize))
    return list(dict.fromkeys(cs))          # the families overlap (dense and boundary pairs up to 48): once each


def chain_shapes():
    shapes = {(w, h) for w in range(1, 131) for h in (1, 2, 3, 7, 64)}
    shapes |= {(h, w) for (w, h) in shapes} | {(s, s) for s in range(1, 131)}
    return sorted(shapes - {(1, 1)})            # a 1 x 1 base has no second level


def box_row_undefined(c):
    """a BOX chain whose base is one row high and wider than one pixel: the reference's BOX filter reads the second row of its
    scanline buffer, which no level of such a chain ever wrote (dxb_mip_box), so its result is not defined"""
    return not c.resize and R.mode_of(c) == BOX and c.h == 1 and c.w > 1


def _chain_cases():
    cs = []
    for flt in FILTERS:
        for w, h in chain_shapes():
            cs += [case(2, w, h, flt), case(28, w, h, flt)]
            for fmt, fl, n in ((10, 0, 8), (24, 0, 12), (28, SRGB, 12)):
                if _pick("mips-%d-%d-%d-%x-%x" % (w, h, fmt, fl, flt), n):
                    cs.append(case(fmt, w, h, flt | fl))
    return [c for c in cs if not box_row_undefined(c)]


# The case lists are built on first use, not at import: collecting either sweep file (also when -m deselects it) stays cheap.
@functools.lru_cache(maxsize=None)
def resize_cases():
    return tuple(_resize_cases())


@functools.lru_cache(maxsize=None)
def chain_cases():
    return tuple(_chain_cases())


def cases():
    return resize_cases() + chain_cases()


@functools.lru_cache(maxsize=None)
def device_cases():
    """a seeded tenth of the cases that run, at the pad16 and off4 device layouts"""
    return tuple(with_layout(c, lay) for c in cases() if c.fams and _pick(R.case_id(c) + "device", 10) for lay in ("pad16", "off4"))


def srgb_of(c):
    return bool(R.srgb_bits(c.fmt, c.fl))


def group_key(c):
    """(operation, filter name, format, sRGB) of a case: the unit the GPU file runs per test"""
    return ("resize" if c.resize else "mips", FILTER_NAME[filter_of(c)], c.fmt, srgb_of(c))


# every group_key of the sweep: operation x filter x (the two swept formats, R16G16B16A16_FLOAT, R10G10B10A2_UNORM, and
# R8G8B8A8_UNORM with TEX_FILTER_SRGB)
GROUP_KEYS = tuple((op, FILTER_NAME[f], fmt, srgb) for op in ("resize", "mips") for f in FILTERS
                   for (fmt, srgb) in ((2, False), (28, False), (10, False), (24, False), (28, True)))


def groups(cs):
    out = collections.OrderedDict()
    for c in cs:
        out.setdefault(group_key(c), []).append(c)
    return out


@functools.lru_cache(maxsize=None)
def host_groups():
    out = collections.OrderedDict((k, []) for k in GROUP_KEYS)
    for c in cases():
        out[group_key(c)].append(c)
    return out


# the device tenth is grouped per operation and filter only: some (format, sRGB) groups have no case in it
DEVICE_KEYS = tuple((op, FILTER_NAME[f]) for op in ("resize", "mips") for f in FILTERS)


@functools.lru_cache(maxsize=None)
def device_groups():
    out = collections.OrderedDict((k, []) for k in DEVICE_KEYS)
    for c in device_cases():
        out[group_key(c)[:2]].append(c)
    return out


def group_id(key):
    """resize-CUBIC-f2, mips-LINEAR-f28-srgb ...; a DEVICE_KEYS key has no format: resize-CUBIC"""
    if len(key) == 2:
        return "%s-%s" % key
    op, name, fmt, srgb = key
    return "%s-%s-f%d%s" % (op, name, fmt, "-srgb" if srgb else "")


def host_bytes(c):
    return c.items * sum(F.compute_pitch(c.fmt, w, h)[1] for (w, h) in R.levels_of(c))
