"""The per-axis address modes of GenerateMipMaps and Resize: one case table shared by tests/test_cpu_address_modes.py and
tests/test_gpu_address_modes.py.

The reference reads TEX_FILTER_WRAP_U / WRAP_V / MIRROR_U / MIRROR_V separately for each axis: CreateLinearFilter and
CreateTriangleFilter take the axis's wrap bit, CreateCubicFilter its wrap and mirror bits (bounduvw: wrap wins over mirror),
BOX and POINT read none, and a 2D image never reads the W bits.  The library makes the same choice in dxb_mips.cuh (k_mip_level,
k_mip_tail, the non-CUBIC k_mip_tile), in k_mip_tile's CUBIC branch, in k_mip_sep and in the TRIANGLE gather lists of dxb_plan.h.
A route that swaps the axes, ORs them or drops one is only visible on content whose edges differ from each other and on extents
where the boundary rule reaches a result:

  LINEAR   the wrap bit moves a tap only where the axis is enlarged from at least 2 pixels (a reduced axis never reads outside
           [0, source - 1], so LINEAR mip chains are the same under every word);
  CUBIC    wrap moves a tap where source >= 2 and the ratio source / dest is below 3 and not 1 (from 3:1 on, and at 1:1, the outer
           taps are inside the image or carry weight 0; at 2 -> 1 wrap swaps the two outer taps, whose weights are equal, so only
           the rounding may move); mirror differs from clamp only beyond the last pixel but one, which a
           weighted tap reaches only where the axis is enlarged from at least 2 pixels;
  TRIANGLE wrap changes the weights wherever source and destination have 2 pixels or more; with one destination pixel every
           source pixel still lands in it, and with one source pixel every tap reads it, so the weights only round differently
           and the result may or may not move.

acting() states these rules and the teeth test holds the reference to them for every case: the result of a word equals the
result of 0, of its U/V swap, of the word without either axis's bits and of the word without any one bit exactly when the
rules say the two read the same taps.  A case whose words cannot be told apart where the rules say they act fails there."""
import collections

import numpy as np

from directxtex_b200 import formats as F
from tests import test_gpu_mip_routes as R

WU, WV, WW = F.TEX_FILTER_WRAP_U, F.TEX_FILTER_WRAP_V, 0x4
MU, MV, MW = F.TEX_FILTER_MIRROR_U, F.TEX_FILTER_MIRROR_V, 0x40
WRAP, MIRROR = F.TEX_FILTER_WRAP, F.TEX_FILTER_MIRROR
BOX, LIN, CUB, TRI, PT = R.BOX, R.LIN, R.CUB, R.TRI, R.PT
SRGB = R.SRGB
U_BITS, V_BITS = WU | MU, WV | MV

# every word that can behave differently per axis, the W bits alone (no-ops on 2D images) and the two whole-image words
WORDS = (0, WU, WV, MU, MV, WU | MV, MU | WV, WU | MU, WV | MV, WRAP | MIRROR, WW, MW, WRAP, MIRROR)
# the shorter list of the large cases: closed under the U/V swap
SHORT = (0, WU, WV, WU | MV, MU | WV)
BOX3, TAIL, SEP, TILE, LEVEL = R.FAMILIES
HOT = R.HOT


def swap_uv(word):
    return (word & ~(U_BITS | V_BITS)) | ((word & U_BITS) << 1) | ((word & V_BITS) >> 1)


def asymmetric(word):
    return (word & (U_BITS | V_BITS)) != (swap_uv(word) & (U_BITS | V_BITS))


def variants(word):
    """the words the teeth test compares `word` with: 0, the U/V swap, the word without its U bits, without its V bits and
    without each one of its bits"""
    out = {0, swap_uv(word), word & ~U_BITS, word & ~V_BITS}
    out |= {word & ~b for b in (WU, WV, WW, MU, MV, MW) if word & b}
    out.discard(word)
    return sorted(out)


# ---- the case table ---------------------------------------------------------------------------------------------------
# mode: the filter (0 = the reference's default for the extents); fl: other flags (sRGB); words: the address words it runs;
# fams: the kernel families option 0 launches (test_gpu_mip_routes.FAMILIES); resize: destination (w, h), None = a mip chain
Case = collections.namedtuple("Case", "fmt w h items mode fl words fams resize")


def case(fmt, w, h, mode, fams, words=WORDS, resize=None, items=1, fl=0):
    return Case(fmt, w, h, items, mode, fl, tuple(words), frozenset(fams), resize)


def case_id(c):
    op = "resize%dx%d" % c.resize if c.resize else "mips"
    return "%s-f%d-%dx%dx%d-%06x" % (op, c.fmt, c.w, c.h, c.items, c.mode | c.fl)


def route_case(c, word, layout="host"):
    """the test_gpu_mip_routes case that runs `c` with `word`"""
    return R.case(c.fmt, c.w, c.h, c.items, c.mode | c.fl | word, c.fams, layout, c.resize)


def _cases():
    cs = []
    for fmt in HOT:
        s = SRGB if fmt == 29 else 0
        cs += [
            # k_mip_box3: LINEAR at 2:1 and BOX read no address bit
            case(fmt, 256, 128, LIN, (BOX3, TAIL), SHORT, fl=s), case(fmt, 256, 256, BOX, (BOX3, TAIL), SHORT, fl=s),
            # k_mip_sep at 2:1 (wrap acts at both ends of both axes), then k_mip_tail
            case(fmt, 160, 96, CUB, (SEP, TAIL), fl=s),
            # k_mip_sep enlarging: wrap and mirror act; 40x30 -> 120x90 and 7x5 -> 20x13
            case(fmt, 40, 30, CUB, (SEP,), resize=(120, 90), fl=s), case(fmt, 7, 5, CUB, (SEP,), resize=(20, 13), fl=s),
            # k_mip_tile CUBIC: one axis above 3:1 (no address bit acts there), the other reduced below 3:1 or enlarged
            case(fmt, 200, 60, CUB, (TILE,), resize=(50, 30), fl=s), case(fmt, 60, 200, CUB, (TILE,), resize=(30, 50), fl=s),
            case(fmt, 200, 30, CUB, (TILE,), resize=(50, 90), fl=s), case(fmt, 30, 200, CUB, (TILE,), resize=(90, 50), fl=s),
            # k_mip_tile LINEAR enlarging (wrap acts), and on an odd chain (filter 0 = LINEAR, no level 2:1), then k_mip_tail
            case(fmt, 40, 30, LIN, (TILE,), resize=(120, 90), fl=s), case(fmt, 333, 97, 0, (TILE, TAIL), SHORT, fl=s),
            # k_mip_tail alone: a chain from 64 x 64 down, odd sizes and 1-pixel axes
            case(fmt, 61, 37, CUB, (TAIL,), fl=s), case(fmt, 5, 3, CUB, (TAIL,), fl=s), case(fmt, 9, 2, CUB, (TAIL,), fl=s),
        ]
    # CUBIC at 4:1 (nothing acts), at non-integer ratios and one axis of 1, 2, 3 and 5 pixels
    cs += [case(28, 200, 120, CUB, (TILE,), resize=(50, 30)), case(10, 100, 60, CUB, (SEP,), resize=(37, 91)),
           case(2, 97, 61, CUB, (SEP,), resize=(41, 26)), case(28, 1, 40, CUB, (TAIL,)), case(87, 40, 1, CUB, (TAIL,)),
           case(61, 2, 48, CUB, (TAIL,)), case(41, 3, 17, CUB, (TAIL,)), case(2, 48, 5, CUB, (TAIL,)),
           case(10, 1, 9, CUB, (SEP,), resize=(2, 20)), case(28, 3, 5, CUB, (SEP,), resize=(7, 2))]
    # LINEAR resizes: enlarging one axis only, 7 -> 20
    cs += [case(28, 7, 40, LIN, (TILE,), resize=(20, 20)), case(10, 40, 7, LIN, (TILE,), resize=(20, 20)),
           case(2, 7, 7, LIN, (TILE,), resize=(20, 20)), case(61, 5, 3, 0, (TILE,), resize=(9, 8))]
    # partial tiles: k_mip_sep and k_mip_tile on wide, short, tall and odd sizes
    cs += [case(28, 1023, 767, CUB, (SEP, TAIL), SHORT), case(10, 2048, 4, CUB, (SEP, TAIL), SHORT), case(41, 4, 2048, CUB, (SEP, TAIL), SHORT),
           case(87, 1023, 767, CUB, (TILE,), SHORT, resize=(200, 380)), case(61, 767, 1023, CUB, (TILE,), SHORT, resize=(380, 200)),
           case(2, 1023, 767, 0, (TILE, TAIL), SHORT), case(28, 2048, 4, BOX, (TILE, TAIL), SHORT)]
    # TRIANGLE and POINT run the generic kernel on every format
    cs += [case(28, 96, 40, TRI, (LEVEL,)), case(2, 37, 22, TRI, (LEVEL,)), case(61, 1, 24, TRI, (LEVEL,)),
           case(10, 40, 30, TRI, (LEVEL,), resize=(120, 90)), case(87, 100, 60, TRI, (LEVEL,), resize=(37, 91)),
           case(28, 48, 20, PT, (LEVEL,)), case(41, 30, 40, PT, (LEVEL,), resize=(70, 20))]
    # formats without specialised kernels: the generic kernel on every filter
    cs += [case(88, 160, 96, CUB, (LEVEL,)), case(88, 40, 30, CUB, (LEVEL,), resize=(120, 90)), case(88, 40, 30, LIN, (LEVEL,), resize=(120, 90)),
           case(24, 96, 40, TRI, (LEVEL,)), case(24, 7, 5, CUB, (LEVEL,), resize=(20, 13)), case(24, 333, 97, 0, (LEVEL,), SHORT)]
    # sRGB on the linear twin's specialised kernels
    cs += [case(28, 160, 96, CUB, (SEP, TAIL), SHORT, fl=SRGB), case(28, 200, 30, CUB, (TILE,), SHORT, resize=(50, 90), fl=SRGB),
           case(28, 40, 30, LIN, (TILE,), SHORT, resize=(120, 90), fl=SRGB), case(28, 96, 40, TRI, (LEVEL,), SHORT, fl=SRGB)]
    # arrays: per-item records on k_mip_sep, k_mip_tile and k_mip_tail (one CTA per item)
    cs += [case(28, 160, 96, CUB, (SEP, TAIL), SHORT, items=5), case(10, 61, 37, CUB, (TAIL,), SHORT, items=4),
           case(87, 200, 30, CUB, (TILE,), SHORT, resize=(50, 90), items=3), case(2, 40, 30, TRI, (LEVEL,), SHORT, items=3)]
    return cs


CASES = _cases()

# TRIANGLE resizes between every source and destination extent from 1 to 9, one axis at a time (the other axis 6 -> 4, where
# its wrap bit acts): the gather lists are built on the host for each pair
TRI_WORDS = (0, WU, WV, WRAP)
TRI_GRID = [case(2, s, 6, TRI, (LEVEL,), TRI_WORDS, resize=(d, 4)) for s in range(1, 10) for d in range(1, 10)] + \
           [case(2, 6, s, TRI, (LEVEL,), TRI_WORDS, resize=(4, d)) for s in range(1, 10) for d in range(1, 10) if (s, d) != (6, 4)]


# ---- what the reference's filters read --------------------------------------------------------------------------------
def levels_of(c):
    return R.levels_of(route_case(c, 0))


def axis_pairs(c):
    """the (source, destination) extents of every level of the U axis and of the V axis"""
    sizes = levels_of(c)
    return [(a[0], b[0]) for a, b in zip(sizes, sizes[1:])], [(a[1], b[1]) for a, b in zip(sizes, sizes[1:])]


def _any(vals):
    """True when some level's taps move, None when none does but some level's weights may round differently, else False"""
    vals = list(vals)
    return True if True in vals else (None if None in vals else False)


def acting(c):
    """{bit: True / False / None}: whether the reference's result on case c's extents depends on each of the U / V address bits
    (None: only in the rounding of TRIANGLE's weights).  The rules of the module docstring."""
    mode = R.mode_of(route_case(c, 0))
    out = {}
    for (wrap, mirror), pairs in zip(((WU, MU), (WV, MV)), axis_pairs(c)):
        if mode == LIN:
            out[wrap], out[mirror] = _any(d > s >= 2 for s, d in pairs), False
        elif mode == CUB:
            out[wrap] = _any((None if (s, d) == (2, 1) else True) if s >= 2 and s != d and s < 3 * d else False for s, d in pairs)
            out[mirror] = _any(d > s >= 2 for s, d in pairs)
        elif mode == TRI:
            out[wrap], out[mirror] = _any(True if d >= 2 and s >= 2 else None for s, d in pairs), False
        else:
            out[wrap] = out[mirror] = False
    return out


def effective(c, word):
    """(the bits of `word` that change the reference's result on case c, the bits that may change only its rounding)"""
    act = acting(c)
    if word & WU:
        word &= ~MU                     # bounduvw: wrap wins over mirror on the same axis
    if word & WV:
        word &= ~MV
    sure = sum(b for b in act if word & b and act[b])
    maybe = sum(b for b in act if word & b and act[b] is None)
    return sure, maybe


def same_taps(c, a, b):
    """True when words a and b read the same taps on case c, False when they do not, None when they differ only in rounding"""
    (sa, ma), (sb, mb) = effective(c, a), effective(c, b)
    if sa != sb:
        return False
    return True if ma == mb else None


# ---- content with teeth -----------------------------------------------------------------------------------------------
def content_rgba(w, h, item=0):
    """h x w x 4 floats in [0, 1]: a random interior, a distinct ramp along each edge and a bright 1-pixel column on the left
    edge only, so that wrapping, mirroring or clamping either axis reads different values.  Item k > 0 is a different draw, its
    left / right edges swapped for odd k."""
    rng = np.random.default_rng(1000 + 7 * item + w * 131 + h)
    img = rng.uniform(0.2, 0.8, (h, w, 4))
    x, y = np.linspace(0.0, 1.0, w), np.linspace(0.0, 1.0, h)
    ch = np.array([1.0, 0.8, 0.6, 0.9])
    img[0, :, :] = (0.05 + 0.15 * x)[:, None] * ch                        # top: dark ramp
    img[h - 1, :, :] = (0.55 + 0.25 * x[::-1])[:, None] * ch              # bottom: mid ramp, the other way
    img[:, w - 1, :] = (0.3 + 0.4 * y)[:, None] * ch[::-1]                # right: ramp down the edge
    img[:, 0, :] = 1.0 - 0.1 * y[:, None]                                 # left: bright column
    if item % 2:
        img = img[:, ::-1]
    return np.clip(img, 0.0, 1.0)


def encode(fmt, rgba):
    """the h x w x 4 floats in `fmt` as bytes"""
    r = lambda v, n: np.rint(v * n).astype(np.uint32)
    if fmt in (28, 29):
        return r(rgba, 255).astype(np.uint8).reshape(-1)
    if fmt in (87, 88):
        v = r(rgba[..., [2, 1, 0, 3]], 255).astype(np.uint8)
        if fmt == 88:
            v[..., 3] = 255
        return v.reshape(-1)
    if fmt == 10:
        return rgba.astype(np.float16).view(np.uint8).reshape(-1)
    if fmt == 2:
        return rgba.astype(np.float32).view(np.uint8).reshape(-1)
    if fmt == 61:
        return r(rgba[..., 0], 255).astype(np.uint8).reshape(-1)
    if fmt == 41:
        return np.ascontiguousarray(rgba[..., 0]).astype(np.float32).view(np.uint8).reshape(-1)
    if fmt == 24:
        v = r(rgba[..., 0], 1023) | r(rgba[..., 1], 1023) << 10 | r(rgba[..., 2], 1023) << 20 | r(rgba[..., 3], 3) << 30
        return v.astype(np.uint32).view(np.uint8).reshape(-1)
    raise ValueError(fmt)


def sources(c):
    """level 0 of each item, as test_gpu_mip_routes.run takes it: at most 3 distinct images, item i uses source i % 3"""
    return [encode(c.fmt, content_rgba(c.w, c.h, k)) for k in range(min(c.items, 3))]


def oracle_result(oracle, c, word, src):
    """the reference's levels 1 .. of one item with `word`, concatenated"""
    return np.concatenate(R.oracle_levels(oracle, route_case(c, word), src)[1:])
