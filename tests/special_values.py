"""TEST INFRASTRUCTURE: a deterministic special-value corpus and the comparison rule used with it.

Everything is generated from code (nothing is stored): the fp32 edge list, images that put every edge value in every
channel position (with +Inf and -Inf inside the same 2x2 / 4x4 neighbourhoods), every non-NaN half bit pattern, every
16-bit pattern of the packed 16-bit formats and a seeded sample of R11G11B10 / R9G9B9E5 patterns.  NaN inputs are outside
the contract (DESIGN.md section 3): no generator here emits one.  Never imported by the product."""
import numpy as np

from directxtex_b200 import formats as F

F32_FORMATS = (2, 6, 16, 41)
F16_FORMATS = (10, 34, 54)
FLOAT_FORMATS = F32_FORMATS + F16_FORMATS + (26, 67)
PACKED16 = (85, 86, 115)
SRGB_FORMATS = (29, 91, 93)
CHANNELS = {2: 4, 6: 3, 16: 2, 41: 1, 10: 4, 34: 2, 54: 1}
STORE_SCALES = (255, 127, 65535, 32767, 1023, 3, 31, 63, 15)

_f32 = np.float32


def _ulp_neighbours(v):
    v = _f32(v)
    return [np.nextafter(v, _f32(-np.inf)), v, np.nextafter(v, _f32(np.inf))]


def f32_edges():
    """The fp32 edge list: signed zeros and units, denormals, the half range limits and overflow points, FLT_MAX, +-Inf,
    neighbours of 0.5 and 1, the sRGB thresholds, the rounding ties (k + 1/2) / scale +-1 ulp of every UNORM / SNORM
    store scale, and the R11G11B10 / R9G9B9E5 limits.  Sorted by bit pattern, no duplicates, no NaN."""
    fi = np.finfo(np.float32)
    pos = [1.0, 0.5, 2.0, fi.smallest_subnormal, fi.tiny, 2.0 ** -24, 1023 * 2.0 ** -24, 6.1035156e-05,
           65504.0, 65519.0, 65520.0, 65536.0, 1e5, 1e10, fi.max, np.inf, 0.0031308, 0.04045,
           65024.0, np.nextafter(_f32(65024.0), _f32(np.inf)), float(0x1FF << 7), 2.0 ** -16]
    pos += _ulp_neighbours(0.5) + _ulp_neighbours(1.0)
    for s in STORE_SCALES:
        for k in (0, 1, s - 1):
            pos += _ulp_neighbours(_f32(k + 0.5) / _f32(s))
    vals = np.array([_f32(v) for v in pos] + [_f32(0.0)], np.float32)
    vals = np.concatenate([vals, -vals])
    bits = np.unique(vals.view(np.uint32))
    out = bits.view(np.float32)
    assert not np.isnan(out).any()
    return out


def edge_image(w, h, seed=0, values=None):
    """(h, w, 4) float32 image.  Every value of `values` (default f32_edges()) sits once in each of the four channel
    positions, with the other channels drawn at random from the same list; the top-left 4x4 tile (and one further tile
    per 64 pixels of width) is a +Inf / -Inf checkerboard, so box, linear, cubic and triangle filters and the block
    encoders all meet Inf - Inf.  The rest is filled with random list values."""
    vals = f32_edges() if values is None else np.asarray(values, np.float32)
    rng = np.random.default_rng(seed)
    n = len(vals)
    px = vals[rng.integers(0, n, (4 * n, 4))]
    for c in range(4):
        px[c * n:(c + 1) * n, c] = vals[rng.permutation(n)]
    px = px[rng.permutation(4 * n)]
    img = np.zeros((h, w, 4), np.float32)
    tiles = np.zeros((h, w), bool)
    inf = np.where((np.arange(4)[:, None] + np.arange(4)[None, :]) % 2 == 0, np.float32(np.inf), np.float32(-np.inf))
    for x0 in range(0, max(1, w - 3), 64):
        tile = img[0:4, x0:x0 + 4]
        th, tw = tile.shape[:2]
        tiles[0:4, x0:x0 + 4] = True
        for c in range(4):
            tile[..., c] = np.roll(inf, c, axis=1)[:th, :tw]
    free = int((~tiles).sum())
    if free > len(px):
        px = np.concatenate([px, vals[rng.integers(0, n, (free - len(px), 4))]])
    img[~tiles] = px[:free]                                     # row-major, around the Inf tiles
    return img


def f32_image(fmt, w, h, seed=0):
    """edge_image as fp32 format `fmt` (R32G32B32A32 / R32G32B32 / R32G32 / R32): the leading channels"""
    return np.ascontiguousarray(edge_image(w, h, seed)[..., :CHANNELS[fmt]])


def half_patterns():
    """every non-NaN binary16 pattern: the 63 488 finite ones and +-Inf (uint16)"""
    p = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    return p[(p & 0x7FFF) <= 0x7C00]


def half_image(fmt=10, w=256, seed=0):
    """all non-NaN half patterns as a `fmt` image (RGBA16F / RG16F / R16F) of width w; channel c of pixel i holds pattern
    (i + c * N / C) mod N, so every pattern appears in every channel position.  Returns (uint16 array (h, w, C), h)."""
    c = CHANNELS[fmt]
    p = half_patterns()
    n = len(p)
    rng = np.random.default_rng(seed)
    base = rng.permutation(n)
    idx = np.stack([(base + k * (n // c)) % n for k in range(c)], -1)
    h = -(-n // w)
    pad = rng.integers(0, n, (w * h - n, c))
    idx = np.concatenate([idx, pad])
    return np.ascontiguousarray(p[idx].reshape(h, w, c)), h


def packed_patterns(fmt, seed=0, count=65536):
    """source patterns of a packed format: every 16-bit value for B5G6R5 / B5G5R5A1 / B4G4R4A4; for R11G11B10_FLOAT and
    R9G9B9E5_SHAREDEXP every channel's exponent-31 patterns with zero mantissa (Inf for R11G11B10) plus a seeded sample of
    the rest (R11G11B10 exponent-31 patterns with a mantissa are NaN and stay out)."""
    if fmt in PACKED16:
        return np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    rng = np.random.default_rng(seed)
    v = rng.integers(0, 1 << 32, count, dtype=np.uint64).astype(np.uint32)
    if fmt == 26:
        fields = ((0, 6), (11, 6), (22, 5))                     # (offset, mantissa bits); 5 exponent bits follow each mantissa
        for off, mb in fields:
            m = (v >> np.uint32(off)) & np.uint32((1 << mb) - 1)
            e = (v >> np.uint32(off + mb)) & np.uint32(0x1F)
            nan = (e == 31) & (m != 0)
            v = np.where(nan, v & ~np.uint32(((1 << mb) - 1) << off), v)
        specials = []
        for off, mb in fields:
            specials.append(np.uint32(0x1F << (off + mb)))      # +Inf in this channel, zero elsewhere
        allinf = np.uint32(0)
        for s in specials:
            allinf |= s
        specials.append(allinf)
        specials += [np.uint32(0), np.uint32(0x7BF | (0x7BF << 11) | (0x3DF << 22))]     # zero, largest finite
        v = np.concatenate([np.array(specials, np.uint32), v])
    elif fmt == 67:
        specials = [np.uint32(31 << 27), np.uint32((31 << 27) | 0x7FFFFFF), np.uint32(0), np.uint32(0x7FFFFFF)]
        v = np.concatenate([np.array(specials, np.uint32), v])
    else:
        raise ValueError(fmt)
    return v[:count]


def _int_codes(fmt, n, seed):
    """every code of each channel of an integer format, cycled with a seeded rotation per channel"""
    bpp = F.BYTES_PER_PIXEL[fmt]
    rng = np.random.default_rng(seed)
    if bpp in (1, 2) and fmt not in PACKED16 and fmt not in (49, 51):
        dt = np.uint8 if bpp == 1 else np.uint16
        codes = np.arange(1 << (8 * bpp), dtype=np.uint32).astype(dt)
        return np.resize(codes[rng.permutation(len(codes))], n).view(np.uint8)
    if fmt in (49, 51):                                         # R8G8: two byte channels
        b = np.arange(256, dtype=np.uint8)
        return np.stack([np.resize(b[rng.permutation(256)], n), np.resize(b[rng.permutation(256)], n)], -1).reshape(-1)
    if bpp == 4 and fmt not in (26, 67, 24):                    # four byte channels or two 16-bit channels
        b = np.arange(256, dtype=np.uint8)
        return np.stack([np.resize(b[rng.permutation(256)], n) for _ in range(4)], -1).reshape(-1)
    if fmt == 24:
        return rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.uint8)
    if bpp == 8:                                                # four 16-bit channels
        c = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
        return np.stack([np.resize(c[rng.permutation(len(c))], n) for _ in range(4)], -1).reshape(-1).view(np.uint8)
    raise ValueError(fmt)


def source_image(fmt, w, h, seed=0):
    """A w x h source of any supported pixel format as tightly packed bytes: the fp32 corpus for the fp32 formats, all
    half patterns for the half formats (cycled), the packed patterns for 85 / 86 / 115 / 26 / 67 and every code of each
    channel for the integer formats."""
    n = w * h
    if fmt in F32_FORMATS:
        return f32_image(fmt, w, h, seed).view(np.uint8).reshape(-1)
    if fmt in F16_FORMATS:
        c = CHANNELS[fmt]
        img, _ = half_image(fmt, 256, seed)
        flat = img.reshape(-1, c)
        rng = np.random.default_rng(seed)
        start = int(rng.integers(0, len(flat)))
        return np.ascontiguousarray(np.resize(np.roll(flat, -start, 0), (n, c))).view(np.uint8).reshape(-1)
    if fmt in PACKED16 or fmt in (26, 67):
        p = packed_patterns(fmt, seed)
        rng = np.random.default_rng(seed + 1)
        return np.ascontiguousarray(np.resize(p[rng.permutation(len(p))], n)).view(np.uint8).reshape(-1)
    return np.ascontiguousarray(_int_codes(fmt, n, seed))


# ---- comparison -----------------------------------------------------------------------------------------------------
def _float_elements(buf, fmt):
    """(elements, NaN mask) of a float-format buffer, or None for formats whose NaN bit pattern is not free"""
    if fmt in F32_FORMATS:
        a = buf.view(np.uint32)
        return a, (a & np.uint32(0x7FFFFFFF)) > np.uint32(0x7F800000)
    if fmt in F16_FORMATS:
        a = buf.view(np.uint16)
        return a, (a & np.uint16(0x7FFF)) > np.uint16(0x7C00)
    if fmt == 26:
        a = buf.view(np.uint32)
        ch = np.stack([a & 0x7FF, (a >> 11) & 0x7FF, a >> 22], -1)
        nan = np.stack([((ch[:, 0] >> 6) == 31) & ((ch[:, 0] & 0x3F) != 0), ((ch[:, 1] >> 6) == 31) & ((ch[:, 1] & 0x3F) != 0),
                        ((ch[:, 2] >> 5) == 31) & ((ch[:, 2] & 0x1F) != 0)], -1)
        return ch, nan
    return None


def mismatches(got, want, fmt):
    """Boolean mask of the elements that differ, under the suite's one comparison rule: outputs are compared bit for bit,
    except that where the destination is a float format and BOTH sides hold a NaN, any NaN matches any NaN (the NaN bit
    pattern that Inf - Inf or 0 * Inf produces is not pinned between x86 and CUDA).  NaN INPUTS are out of contract and
    must not be fed to this rule's callers."""
    a = np.ascontiguousarray(got).view(np.uint8).reshape(-1)
    b = np.ascontiguousarray(want).view(np.uint8).reshape(-1)
    assert a.size == b.size, (a.size, b.size)
    fa = _float_elements(a, fmt)
    if fa is None:
        return a != b
    ea, na = fa
    eb, nb = _float_elements(b, fmt)
    return (ea != eb) & ~(na & nb)


def assert_same(got, want, fmt, ctx=""):
    bad = mismatches(got, want, fmt)
    if bad.any():
        idx = np.flatnonzero(bad.reshape(len(bad), -1).any(-1) if bad.ndim > 1 else bad)
        raise AssertionError("%s: %d of %d elements differ (fmt %d), first at %s" % (ctx, len(idx), len(bad), fmt, idx[:8].tolist()))


# one code of the destination, in decoded (R32G32B32A32) units: the sRGB paths go through powf, which differs in the last
# ulp between glibc and CUDA's libm; the contract there is +-1 code (DESIGN.md section 3)
def _code_tolerance(fmt, v):
    scale = {11: 65535, 35: 65535, 56: 65535, 13: 32767, 37: 32767, 58: 32767, 31: 127, 51: 127, 63: 127, 85: 31, 86: 31,
             115: 15, 24: 1023}.get(fmt, 255)
    if fmt in FLOAT_FORMATS:
        mbits = {10: 10, 34: 10, 54: 10, 26: 5, 67: 8}.get(fmt, 20)
        return np.abs(v) * np.float32(2.0 ** -mbits) + np.float32(1e-30)
    return np.float32(1.0001 / scale)


def assert_within_one_code(oracle, got, want, w, h, fmt, ctx=""):
    """the sRGB rule: one destination code per channel.  8- and 16-bit channel formats compare their stored codes; the
    others are decoded to RGBA32F with the reference (float destinations: a relative 2^-(mantissa bits), a few ulps of
    powf's last-place difference after scaling)"""
    if np.array_equal(np.asarray(got).view(np.uint8).reshape(-1), np.asarray(want).view(np.uint8).reshape(-1)):
        return
    raw = {28: np.uint8, 29: np.uint8, 87: np.uint8, 88: np.uint8, 91: np.uint8, 93: np.uint8, 49: np.uint8, 61: np.uint8, 65: np.uint8,
           31: np.int8, 51: np.int8, 63: np.int8, 11: np.uint16, 35: np.uint16, 56: np.uint16, 13: np.int16, 37: np.int16, 58: np.int16}
    if fmt in raw:                                              # one code per channel, on the stored codes
        a = np.ascontiguousarray(got).view(raw[fmt]).astype(np.int32)
        b = np.ascontiguousarray(want).view(raw[fmt]).astype(np.int32)
        bad = np.abs(a - b) > 1
        assert not bad.any(), "%s: %d channels beyond one code (fmt %d), first at %s" % (ctx, int(bad.sum()), fmt, np.flatnonzero(bad)[:8].tolist())
        return
    if fmt == 2:
        a, b = np.asarray(got).view(np.float32), np.asarray(want).view(np.float32)
    else:
        hr1, a = oracle.convert(got, w, h, fmt, 2)
        hr2, b = oracle.convert(want, w, h, fmt, 2)
        assert hr1 == 0 and hr2 == 0
        a, b = a.view(np.float32), b.view(np.float32)
    both_nan = np.isnan(a) & np.isnan(b)
    with np.errstate(invalid="ignore"):                         # Inf - Inf where both sides hold the same Inf (a == b below)
        d = np.abs(a.astype(np.float64) - b.astype(np.float64))
    mag = np.maximum(np.abs(a), np.abs(b))
    if fmt == 67:                                               # one shared exponent: a code is relative to the pixel's largest channel
        mag = np.repeat(mag.reshape(-1, 4)[:, :3].max(1), 4)
    tol = _code_tolerance(fmt, mag)
    bad = ~both_nan & ~(d <= tol) & ~(a == b)
    assert not bad.any(), "%s: %d channels beyond one code (fmt %d), first at %s" % (ctx, int(bad.sum()), fmt, np.flatnonzero(bad)[:8].tolist())


def convert_refused(dst_fmt, flags):
    """the pairs the library refuses (dxb_plan.h plan_convert): dithered stores to the 16-bit packed formats"""
    return bool(flags & (F.TEX_FILTER_DITHER | F.TEX_FILTER_DITHER_DIFFUSION)) and dst_fmt in PACKED16


def involves_srgb(sf, df, flags):
    return sf in SRGB_FORMATS or df in SRGB_FORMATS or bool(flags & F.TEX_FILTER_SRGB)


# ---- sRGB inputs on which glibc's and CUDA's powf agree -------------------------------------------------------------------
SNORM_FORMATS = (13, 31, 37, 51, 58, 63, 81, 84)
SRGB_BLOCK_FORMATS = (72, 75, 78, 99)


def resolve_srgb(flags, in_fmt, out_fmt):
    """the sRGB bits ConvertScanline runs with (DirectXTexConvert.cpp:3121-3167), restated here independently of
    dxb_resolve_srgb_convert: an sRGB format adds its side's bit, A8 drops it, and IN together with OUT cancel"""
    f = flags & F.TEX_FILTER_SRGB
    srgb = SRGB_FORMATS + SRGB_BLOCK_FORMATS
    if in_fmt in srgb:
        f |= F.TEX_FILTER_SRGB_IN
    elif in_fmt == 65:
        f &= ~F.TEX_FILTER_SRGB_IN
    if out_fmt in srgb:
        f |= F.TEX_FILTER_SRGB_OUT
    elif out_fmt == 65:
        f &= ~F.TEX_FILTER_SRGB_OUT
    if f == F.TEX_FILTER_SRGB:
        f = 0
    return f


def powf_direction(flags, in_fmt, out_fmt):
    """TEX_FILTER_SRGB_IN or _OUT when a Convert / Compress / Decompress from in_fmt to out_fmt with these flags runs a pixel
    through powf, else 0.  sRGB -> linear runs on FLOAT and UNORM inputs, linear -> sRGB on FLOAT and UNORM outputs
    (dxb_convert_pixel); every supported format is FLOAT, UNORM or SNORM."""
    f = resolve_srgb(flags, in_fmt, out_fmt)
    if f & F.TEX_FILTER_SRGB_IN and in_fmt not in SNORM_FORMATS:
        return F.TEX_FILTER_SRGB_IN
    if f & F.TEX_FILTER_SRGB_OUT and out_fmt not in SNORM_FORMATS:
        return F.TEX_FILTER_SRGB_OUT
    return 0


def _fields(fmt):
    """[(bit offset, bits, kind, decoded channel or None)] of one pixel of `fmt`, or None for R9G9B9E5 (shared exponent: whole
    pixels).  kind: 'f32', 'f16', 'f11' (an R11G11B10 field) or 'int'.  Every field decodes into one channel alone, which
    _probe checks on the oracle's decoding."""
    if fmt in F32_FORMATS:
        return [(32 * c, 32, "f32", c) for c in range(CHANNELS[fmt])]
    if fmt in F16_FORMATS:
        return [(16 * c, 16, "f16", c) for c in range(CHANNELS[fmt])]
    if fmt == 67:
        return None
    bgra = [(0, 8, "int", 2), (8, 8, "int", 1), (16, 8, "int", 0)]
    fixed = {26: [(0, 11, "f11", 0), (11, 11, "f11", 1), (22, 10, "f11", 2)],
             24: [(0, 10, "int", 0), (10, 10, "int", 1), (20, 10, "int", 2), (30, 2, "int", 3)],
             85: [(0, 5, "int", 2), (5, 6, "int", 1), (11, 5, "int", 0)],
             86: [(0, 5, "int", 2), (5, 5, "int", 1), (10, 5, "int", 0), (15, 1, "int", 3)],
             115: [(0, 4, "int", 2), (4, 4, "int", 1), (8, 4, "int", 0), (12, 4, "int", 3)],
             87: bgra + [(24, 8, "int", 3)], 91: bgra + [(24, 8, "int", 3)], 88: bgra + [(24, 8, "int", None)], 93: bgra + [(24, 8, "int", None)],
             65: [(0, 8, "int", 3)]}
    if fmt in fixed:
        return fixed[fmt]
    size = 16 if fmt in (11, 13, 35, 37, 56, 58) else 8
    return [(size * c, size, "int", c) for c in range(F.BYTES_PER_PIXEL[fmt] * 8 // size)]


def _field_pool(kind, bits, rng):
    """candidate values of one field: every pattern up to 16 bits (NaN patterns excluded), a seeded pool for fp32"""
    if kind == "f32":
        pool = np.concatenate([f32_edges(), rng.random(6144, dtype=np.float32), (rng.random(2048) * 1.4 - 0.2).astype(np.float32)])
        return np.unique(pool.view(np.uint32))
    if kind == "f16":
        return half_patterns().astype(np.uint32)
    v = np.arange(1 << bits, dtype=np.uint32)
    if kind == "f11":
        mb = bits - 5
        v = v[~(((v >> np.uint32(mb)) == 31) & ((v & np.uint32((1 << mb) - 1)) != 0))]
    return v


def _pack(fmt, fields, cols):
    """pixels of `fmt` as bytes (n, bpp) from one value column per field"""
    n, bpp = len(cols[0]), F.BYTES_PER_PIXEL[fmt]
    out = np.zeros((n, bpp), np.uint8)
    word = np.zeros(n, np.uint32)
    for (off, bits, _, _), col in zip(fields, cols):
        if bits in (8, 16, 32) and off % 8 == 0:
            out[:, off // 8:(off + bits) // 8] = col.astype("<u%d" % (bits // 8)).view(np.uint8).reshape(n, bits // 8)
        else:
            word |= col.astype(np.uint32) << np.uint32(off)
    if any(not (bits in (8, 16, 32) and off % 8 == 0) for (off, bits, _, _) in fields):
        out |= word.view(np.uint8).reshape(n, 4)[:, :bpp]
    return out


def _device_convert():
    """capi.convert when a CUDA device is present, else None"""
    try:
        from directxtex_b200 import capi
        if capi.lib.dxb200_device_count() > 0 and capi.lib.dxb200_init(0) == 0:
            return capi.convert
    except Exception:
        pass
    return None


_SAFE = {}
SRGB_SAFE_FRACTIONS = {}


def _probe(fmt, direction):
    """(fields, pools, safe masks) of `fmt` for one sRGB direction; cached"""
    key = (fmt, direction)
    if key in _SAFE:
        return _SAFE[key]
    from tests import oracle_lib
    oracle = oracle_lib.load_ref()
    rng = np.random.default_rng(fmt * 7 + direction)
    fields = _fields(fmt)
    if fields is None:
        pools = [packed_patterns(fmt, seed=fmt)]
        cols = pools
        n = len(pools[0])
        pixels = pools[0].astype("<u4").view(np.uint8).reshape(n, 4)
    else:
        pools = [_field_pool(kind, bits, rng) for (_, bits, kind, _) in fields]
        n = max(len(p) for p in pools)
        cols = [np.resize(p[rng.permutation(len(p))], n) for p in pools]
        pixels = _pack(fmt, fields, cols)
    # the value each channel enters the sRGB function with: the pixel as loaded (the oracle's bit-exact Convert to
    # R32G32B32A32; for an sRGB format with both flags, which cancel its own sRGB -> linear step), and for linear -> sRGB
    # from an SNORM source after its mapping to UNORM, v * 0.5 + 0.5 unfused
    if fmt == 2:
        dec = pixels
    else:
        hr, dec = oracle.convert(pixels, n, 1, fmt, 2, F.TEX_FILTER_SRGB if fmt in SRGB_FORMATS else 0)
        assert hr == 0
    u = np.ascontiguousarray(dec).view(np.float32).reshape(n, 4).copy()
    if direction == F.TEX_FILTER_SRGB_OUT and fmt in SNORM_FORMATS:
        u = (u * np.float32(0.5)).astype(np.float32) + np.float32(0.5)
    # every distinct value through device and oracle Convert(R32_FLOAT -> R32G32B32A32_FLOAT) with the sRGB flag: the same
    # dxb_convert_pixel the block encoders run, on the same inputs; a value is safe where both give the same bits
    ubits = u[:, :3].view(np.uint32)
    vals = np.unique(ubits)
    device = _device_convert()
    if device is None:
        safe_vals = vals
    else:
        m = -(-len(vals) // 256) * 256
        probe = np.zeros(m, np.uint32)
        probe[:len(vals)] = vals
        hr, want = oracle.convert(probe.view(np.float32), 256, m // 256, 41, 2, direction)
        assert hr == 0
        got = device(probe.view(np.float32), 256, m // 256, 41, 2, direction)
        same = got.view(np.uint32).reshape(m, 4)[:, 0] == want.view(np.uint32).reshape(m, 4)[:, 0]
        safe_vals = vals[same[:len(vals)]]
    chan_safe = np.isin(ubits, safe_vals)
    if fields is None:
        masks = [chan_safe.all(1)]
        kept, total = int(masks[0].sum()), n
    else:
        masks, kept, total = [], 0, 0
        for (off, bits, kind, ch), pool, col in zip(fields, pools, cols):
            if ch is None or ch == 3:                           # alpha and X never go through powf
                masks.append(np.ones(len(pool), bool))
                continue
            # the field alone decides its channel (checks the layout of _fields)
            pairs = np.unique(np.stack([col, ubits[:, ch]], 1), axis=0)
            assert len(pairs) == len(np.unique(col)), (fmt, off)
            bad = np.unique(col[~chan_safe[:, ch]])
            masks.append(~np.isin(pool, bad))
            kept += int(masks[-1].sum())
            total += len(pool)
    frac = kept / total if total else 1.0
    SRGB_SAFE_FRACTIONS[key] = (kept, total)
    print("srgb_safe_image: format %d %s: %d of %d values kept (%.1f %%)%s" % (
        fmt, "SRGB_IN" if direction == F.TEX_FILTER_SRGB_IN else "SRGB_OUT", kept, total, 100.0 * frac, "" if device else " (oracle only)"))
    assert frac >= 0.25, (fmt, direction, frac)
    _SAFE[key] = (fields, pools, masks)
    return _SAFE[key]


def srgb_safe_image(fmt, direction, w, h, seed=0):
    """A w x h source of `fmt` (tightly packed bytes) whose every channel value gives the same bits through CUDA's powf as
    through glibc's, in the given direction (TEX_FILTER_SRGB_IN: sRGB -> linear on the loaded value; TEX_FILTER_SRGB_OUT:
    linear -> sRGB after the conversion to UNORM).  A single ulp of difference can change a BC block, so an sRGB compress
    or convert is compared bit for bit only on such inputs.  The candidates are every pattern of each field up to 16 bits
    (every code of the 8-, 10- and 16-bit formats, every non-NaN half) and a seeded fp32 pool with the edge list; each
    field's values are drawn independently from its safe set (R9G9B9E5: whole safe patterns).  Without a CUDA device
    every value is kept."""
    fields, pools, masks = _probe(fmt, direction)
    rng = np.random.default_rng(seed)
    n = w * h
    cols = []
    for pool, mask in zip(pools, masks):
        keep = pool[mask]
        cols.append(np.resize(keep[rng.permutation(len(keep))], n))
    if fields is None:
        return np.ascontiguousarray(cols[0].astype("<u4").view(np.uint8))
    return np.ascontiguousarray(_pack(fmt, fields, cols).reshape(-1))
