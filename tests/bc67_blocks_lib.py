"""TEST INFRASTRUCTURE: per-block checks of the BC6H and BC7 encoders against the reference decoder (tests/test_cpu_bc67_blocks.py,
tests/test_gpu_bc67_blocks.py).

tests/bc67_blocks/record_host.cpp is the host emulator plus the encoders' host-only record and force hooks: for every block it returns
what the encoder chose (mode, shape, rotation, index selector, endpoints, indices) and the texels those choices must decode to.  This
module holds
  - record(): one recorded encode, optionally with per-block forcing;
  - a reader of the BC6H / BC7 bit streams written from the format description (the mode fields, the partition / rotation / index
    selector fields and the index fields), with the partition and anchor tables probed from the reference decoder rather than
    taken from the encoder's tables;
  - check_bc7() / check_bc6h(): the reference decoder returns the recorded texels exactly, the stream's fields equal the record,
    and every index is the exhaustive nearest entry of the recorded palette (lowest index on ties);
  - the structured corpora and the forced cells;
  - stratified random block streams for the decoders (every mode, every endpoint order)."""
import ctypes as C

import numpy as np

from directxtex_b200 import formats as F
from tests import bc7_ranking_build as B, oracle_lib

BC7, UF16, SF16 = 98, 95, 96
REC = 80
HERE = B.os.path.join(B.ROOT, "tests", "bc67_blocks")


# ---- the recording harness ---------------------------------------------------------------------------------------------------
def load(out_dir):
    L = B.host_lib("record_host.cpp", out_dir, HERE)
    L.record_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.record_compress.restype = C.c_int32
    return L


def record(L, emul, src, w, h, sf, df, flags=0, force=None):
    """(blocks, record [blocks, REC] int32).  Unforced, the blocks must equal emul.compress: recording changes nothing."""
    src = np.ascontiguousarray(src)
    nb = ((w + 3) // 4) * ((h + 3) // 4)
    blocks = np.zeros(nb * 16, np.uint8)
    rec = np.zeros((nb, REC), np.int32)
    fp = None
    if force is not None:
        force = np.ascontiguousarray(force, np.int32)
        assert force.shape == (nb, 5 if df == BC7 else 2)
        fp = force.ctypes.data
    hr = L.record_compress(src.ctypes.data, w, h, sf, df, flags, fp, blocks.ctypes.data, rec.ctypes.data)
    assert hr == 0, hex(F.hr_u32(hr))
    if force is None:
        he, want = emul.compress(src, w, h, sf, df, flags)
        assert he == 0 and np.array_equal(blocks, want), "recording changed the blocks"
    return blocks, rec


def bc7_fields(rec):
    r = rec.view(np.uint32)
    tex = r[:, 46:62].copy().view(np.uint8).reshape(-1, 16, 4)
    return dict(mode=r[:, 0].astype(np.int64), shape=r[:, 1].astype(np.int64), rot=r[:, 2].astype(np.int64), idx=r[:, 3].astype(np.int64),
                q0=r[:, 4:7], q1=r[:, 7:10], pb=r[:, 10:13].astype(np.int64), err=r[:, 13].astype(np.int64),
                idxC=r[:, 14:30].astype(np.int64), idxA=r[:, 30:46].astype(np.int64), texel=tex.astype(np.int64))


def bc6h_fields(rec):
    return dict(mode=rec[:, 0].astype(np.int64), shape=rec[:, 1].astype(np.int64), wq=rec[:, 2:14].astype(np.int64).reshape(-1, 4, 3),
                idx=rec[:, 14:30].astype(np.int64), texel=rec[:, 30:78].astype(np.int64).reshape(-1, 16, 3))


# ---- the format, from its description ---------------------------------------------------------------------------------------
# BC7 modes: subsets, partition bits, rotation bits, index-selector bits, colour bits, alpha bits, p-bits per endpoint, shared
# p-bits per subset, index bits, second index bits
BC7_MODES = {0: (3, 4, 0, 0, 4, 0, 1, 0, 3, 0), 1: (2, 6, 0, 0, 6, 0, 0, 1, 3, 0), 2: (3, 6, 0, 0, 5, 0, 0, 0, 2, 0),
             3: (2, 6, 0, 0, 7, 0, 1, 0, 2, 0), 4: (1, 0, 2, 1, 5, 6, 0, 0, 2, 3), 5: (1, 0, 2, 0, 7, 8, 0, 0, 2, 2),
             6: (1, 0, 0, 0, 7, 7, 1, 0, 4, 0), 7: (2, 6, 0, 0, 5, 5, 1, 0, 2, 0)}
# BC6H modes 1..14 (record index 0..13): mode field, regions, endpoint precision, delta bits R G B (0: not transformed)
BC6H_MODES = [(0x00, 2, 10, (5, 5, 5)), (0x01, 2, 7, (6, 6, 6)), (0x02, 2, 11, (5, 4, 4)), (0x06, 2, 11, (4, 5, 4)),
              (0x0A, 2, 11, (4, 4, 5)), (0x0E, 2, 9, (5, 5, 5)), (0x12, 2, 8, (6, 5, 5)), (0x16, 2, 8, (5, 6, 5)),
              (0x1A, 2, 8, (5, 5, 6)), (0x1E, 2, 6, (0, 0, 0)), (0x03, 1, 10, (0, 0, 0)), (0x07, 1, 11, (9, 9, 9)),
              (0x0B, 1, 12, (8, 8, 8)), (0x0F, 1, 16, (4, 4, 4))]
BC6H_CODE_TO_MODE = {m[0]: i for i, m in enumerate(BC6H_MODES)}
BC6H_RESERVED = (0x13, 0x17, 0x1B, 0x1F)
WEIGHTS = {2: [0, 21, 43, 64], 3: [0, 9, 18, 27, 37, 46, 55, 64], 4: [0, 4, 9, 13, 17, 21, 26, 30, 34, 38, 43, 47, 51, 55, 60, 64]}


def bits_of(blocks):
    """[n, 128] bits of 16-byte blocks, LSB of byte 0 first"""
    return np.unpackbits(np.ascontiguousarray(blocks, np.uint8).reshape(-1, 16), axis=1, bitorder="little").astype(np.int64)


def field(bits, pos, n):
    v = np.zeros(bits.shape[0], np.int64)
    for k in range(n):
        v |= bits[:, pos + k] << k
    return v


class Tables:
    """Partition and anchor tables probed from the reference decoder: mode-1 (two subsets) and mode-2 (three subsets) blocks whose
    subsets decode to distinct colours give each pixel's subset; the same blocks with every index bit set decode the anchors (whose
    index field is one bit shorter) to a different palette entry than the other pixels."""

    def __init__(self, ref):
        self.part2, self.anchor2 = self._probe(ref, 1)
        self.part3, self.anchor3 = self._probe(ref, 2)

    @staticmethod
    def _probe(ref, mode):
        ns, pbits, _, _, cb, _, _, spb, ib, _ = BC7_MODES[mode]
        part, anchor = np.zeros((64, 16), np.int64), np.zeros((64, 3), np.int64)
        top = (1 << cb) - 1
        for ones in (False, True):
            blocks = np.zeros((64, 128), np.uint8)
            for s in range(64):
                b = blocks[s]
                b[mode] = 1
                pos = mode + 1
                for k in range(pbits):
                    b[pos + k] = (s >> k) & 1
                pos += pbits
                for c in range(3):                      # endpoint 0 of subset j: j * top / (ns - 1) in channel 0; endpoint 1 = top
                    for j in range(ns):
                        for e in range(2):
                            v = top if (ones and e == 1) else ((j * top) // (ns - 1) if c == 0 else 0)
                            for k in range(cb):
                                b[pos + k] = (v >> k) & 1
                            pos += cb
                pos += spb * ns
                if ones:
                    b[pos:] = 1
            packed = np.packbits(blocks, axis=1, bitorder="little")
            dec = np.rint(ref.decode_blocks(BC7, packed.reshape(-1), 4 * 64, 4) * 255).astype(np.int64)
            dec = dec.reshape(4, 64, 4, 4).transpose(1, 0, 2, 3).reshape(64, 16, 4)
            if not ones:
                part = np.rint(dec[:, :, 0] * (ns - 1) / 255.0).astype(np.int64)
            else:
                full = dec[:, :, 1] > 200                  # index 2^ib - 1 -> endpoint 1 (G near 255); anchors hold 2^(ib-1) - 1
                for s in range(64):
                    for j in range(ns):
                        a = np.nonzero((part[s] == j) & ~full[s])[0]
                        assert a.size == 1, (mode, s, j, a)
                        anchor[s, j] = a[0]
        return part, anchor


def parse_bc7(bits, T):
    """mode (8 = reserved), partition, rotation, index selector, and the colour / alpha index of every pixel as stored"""
    n = bits.shape[0]
    mode = np.full(n, 8, np.int64)
    for m in range(7, -1, -1):
        mode[bits[:, m] == 1] = m
    out = dict(mode=mode, shape=np.zeros(n, np.int64), rot=np.zeros(n, np.int64), isel=np.zeros(n, np.int64),
               idxC=np.zeros((n, 16), np.int64), idxA=np.zeros((n, 16), np.int64))
    for m, (ns, pbits, rbits, ibits, cb, ab, epb, spb, ib, ib2) in BC7_MODES.items():
        sel = np.nonzero(mode == m)[0]
        if sel.size == 0:
            continue
        b = bits[sel]
        pos = m + 1
        shape = field(b, pos, pbits); pos += pbits
        rot = field(b, pos, rbits); pos += rbits
        isel = field(b, pos, ibits); pos += ibits
        pos += 2 * ns * (3 * cb + ab) + 2 * ns * epb + ns * spb
        anchors = np.zeros((sel.size, 3), np.int64)
        if ns == 2:
            anchors[:, :2] = T.anchor2[shape][:, :2]
        elif ns == 3:
            anchors = T.anchor3[shape]
        first = np.zeros((sel.size, 16), np.int64)
        starts = np.full(sel.size, pos, np.int64)                 # the anchors differ per block, so do the field positions
        for i in range(16):
            anch = np.any(anchors[:, :ns] == i, axis=1)
            for r in range(sel.size):
                nbits = ib - 1 if anch[r] else ib
                first[r, i] = sum(int(b[r, starts[r] + k]) << k for k in range(nbits))
                starts[r] += nbits
        second = np.zeros((sel.size, 16), np.int64)
        if ib2:
            p2 = pos + 16 * ib - 1
            for i in range(16):
                nbits = ib2 - 1 if i == 0 else ib2
                second[:, i] = field(b, p2, nbits)
                p2 += nbits
        swap = (m == 4) & (isel == 1)
        out["shape"][sel] = shape; out["rot"][sel] = rot; out["isel"][sel] = isel
        out["idxC"][sel] = np.where(swap[:, None], second, first)
        out["idxA"][sel] = np.where(swap[:, None], first, second)
    return out


def parse_bc6h(bits, T):
    """mode index 0..13 (-1 = reserved code), shape, and the index of every pixel as stored"""
    n = bits.shape[0]
    code = np.where(field(bits, 0, 2) < 2, field(bits, 0, 2), field(bits, 0, 5))
    mode = np.array([BC6H_CODE_TO_MODE.get(int(c), -1) for c in code], np.int64)
    two = np.array([BC6H_MODES[m][1] == 2 if m >= 0 else False for m in mode])
    shape = np.where(two, field(bits, 77, 5), 0)
    idx = np.zeros((n, 16), np.int64)
    for r in range(n):
        pos, ib = (82, 3) if two[r] else (65, 4)
        anchors = (0, int(T.anchor2[shape[r], 1])) if two[r] else (0,)
        for i in range(16):
            nbits = ib - 1 if i in anchors else ib
            idx[r, i] = sum(int(bits[r, pos + k]) << k for k in range(nbits))
            pos += nbits
    return dict(code=code, mode=mode, shape=shape, idx=idx)


# ---- per-block checks ---------------------------------------------------------------------------------------------------------
def block_pixels(img, w, h):
    """[blocks, 16, C] pixels of the full 4x4 blocks of an (h, w, C) image and the mask of full blocks (partial blocks: zeros)"""
    nbx, nby = (w + 3) // 4, (h + 3) // 4
    pad = np.zeros((nby * 4, nbx * 4) + img.shape[2:], img.dtype)
    pad[:h, :w] = img
    px = pad.reshape(nby, 4, nbx, 4, -1).transpose(0, 2, 1, 3, 4).reshape(nbx * nby, 16, -1)
    full = np.zeros((nby, nbx), bool)
    full[:h // 4, :w // 4] = True
    return px, full.reshape(-1)


def decoded_blocks(ref, fmt, blocks):
    nb = blocks.size // 16
    return ref.decode_blocks(fmt, blocks, 4 * nb, 4).reshape(4, nb, 4, 4).transpose(1, 0, 2, 3).reshape(nb, 16, 4)


def _fail(ctx, what, bad, detail=""):
    bad = np.nonzero(bad)[0]
    assert bad.size == 0, "%s: %s in %d blocks; first block %d %s" % (ctx, what, bad.size, bad[0], detail(bad[0]) if callable(detail) else detail)


def bc7_expected_stored(R, T):
    """the recorded indices after the anchor fix-up: a subset whose anchor index has its top bit set is stored mirrored"""
    n = R["mode"].size
    idxC, idxA = R["idxC"].copy(), R["idxA"].copy()
    for r in range(n):
        m, isel = int(R["mode"][r]), int(R["idx"][r])
        ns, _, _, _, _, _, _, _, ib, ib2 = BC7_MODES[m]
        ibc = 3 if (m == 4 and isel) else ib
        iba = (2 if isel else 3) if m == 4 else ib2
        s = int(R["shape"][r])
        part = T.part2[s] if ns == 2 else T.part3[s] if ns == 3 else np.zeros(16, np.int64)
        anchors = [0] + ([int(T.anchor2[s, 1])] if ns == 2 else [int(T.anchor3[s, 1]), int(T.anchor3[s, 2])] if ns == 3 else [])
        for j, a in enumerate(anchors):
            if (R["idxC"][r, a] >> (ibc - 1)) & 1:
                sub = part == j
                idxC[r, sub] = (1 << ibc) - 1 - R["idxC"][r, sub]
        if iba and (R["idxA"][r, 0] >> (iba - 1)) & 1:
            idxA[r] = (1 << iba) - 1 - R["idxA"][r]
    return idxC, idxA


def bc7_palettes(R, T):
    """[blocks, 16 pixels, 16 entries, 4 slots] colour palette and [blocks, 16, 8, 4] alpha palette of every pixel, slot order, from
    the recorded fields dequantised as the format describes (field << (8 - bits) | field >> (2 bits - 8), p-bit as the lowest bit)"""
    n = R["mode"].size
    palC = np.zeros((n, 16, 16, 4), np.int64)
    palA = np.zeros((n, 16, 8, 4), np.int64)
    nC, nA = np.zeros(n, np.int64), np.zeros(n, np.int64)
    for r in range(n):
        m, isel, s = int(R["mode"][r]), int(R["idx"][r]), int(R["shape"][r])
        ns, _, _, _, cb, ab, epb, spb, ib, ib2 = BC7_MODES[m]
        ibc = 3 if (m == 4 and isel) else ib
        iba = (2 if isel else 3) if m == 4 else ib2
        part = T.part2[s] if ns == 2 else T.part3[s] if ns == 3 else np.zeros(16, np.int64)
        for j in range(ns):
            ends = []
            for e, q in enumerate((R["q0"][r, j], R["q1"][r, j])):
                fq = [(int(q) >> (8 * c)) & 0xFF for c in range(4)]
                p = (int(R["pb"][r, j]) >> e) & 1 if (epb or spb) else None
                ch = []
                for c in range(4):
                    bits = cb if c < 3 else ab
                    if bits == 0:
                        ch.append(255)
                        continue
                    v, nb = fq[c], bits
                    if p is not None:
                        v, nb = (v << 1) | p, bits + 1
                    v <<= 8 - nb
                    ch.append(v | (v >> nb))
                ends.append(ch)
            e0, e1 = np.array(ends[0]), np.array(ends[1])
            sub = part == j
            wc = np.array(WEIGHTS[ibc])
            palC[r, sub, :len(wc)] = ((e0[None, :] * (64 - wc[:, None]) + e1[None, :] * wc[:, None] + 32) >> 6)[None]
            if iba:
                wa = np.array(WEIGHTS[iba])
                palA[r, sub, :len(wa)] = ((e0[None, :] * (64 - wa[:, None]) + e1[None, :] * wa[:, None] + 32) >> 6)[None]
        nC[r], nA[r] = 1 << ibc, (1 << iba) if iba else 0
    return palC, palA, nC, nA


def rotate(px, rot):
    """natural RGBA -> slot order (rotation r swaps channel r - 1 with alpha); its own inverse"""
    out = px.copy()
    for r in (1, 2, 3):
        sel = rot == r
        out[sel, ..., r - 1], out[sel, ..., 3] = px[sel, ..., 3], px[sel, ..., r - 1]
    return out


def check_bc7(ref, T, blocks, rec, px=None, ctx=""):
    """(a) the reference decoder returns the recorded texels; (b) the stream's mode, partition, rotation, index selector and indices
    equal the record (indices after the anchor fix-up); (c) with the blocks' LDR pixels px [blocks, 16, 4] (None: skip), every
    recorded index is the exhaustive nearest entry of the recorded palette (ties: lowest index), the palette entries are the recorded
    texels, and the block's decoded squared error is at most the stage-3 error it won with.  Returns the record fields."""
    R = bc7_fields(rec)
    n = R["mode"].size
    dec = np.rint(decoded_blocks(ref, BC7, blocks).astype(np.float64) * 255.0).astype(np.int64)
    _fail(ctx, "reference decode != recorded texels", np.any(dec != R["texel"], axis=(1, 2)),
          lambda b: "mode %d: decoded %s, recorded %s" % (R["mode"][b], dec[b].tolist(), R["texel"][b].tolist()))
    P = parse_bc7(bits_of(blocks), T)
    _fail(ctx, "stream mode != record", P["mode"] != R["mode"])
    hasP = np.isin(R["mode"], (0, 1, 2, 3, 7))
    _fail(ctx, "stream partition != record", hasP & (P["shape"] != R["shape"]))
    _fail(ctx, "stream rotation != record", np.isin(R["mode"], (4, 5)) & (P["rot"] != R["rot"]))
    _fail(ctx, "stream index selector != record", (R["mode"] == 4) & (P["isel"] != R["idx"]))
    eC, eA = bc7_expected_stored(R, T)
    _fail(ctx, "stored colour indices != record", np.any(P["idxC"] != eC, axis=1),
          lambda b: "mode %d shape %d: stored %s, record %s" % (R["mode"][b], R["shape"][b], P["idxC"][b].tolist(), R["idxC"][b].tolist()))
    _fail(ctx, "stored alpha indices != record", np.isin(R["mode"], (4, 5)) & np.any(P["idxA"] != eA, axis=1))
    palC, palA, nC, nA = bc7_palettes(R, T)
    sepA = np.isin(R["mode"], (4, 5))
    i16 = np.arange(16)
    entC = palC[np.arange(n)[:, None], i16[None], R["idxC"]]
    entA = palA[np.arange(n)[:, None], i16[None], R["idxA"]]
    want = np.where(sepA[:, None, None] & (np.arange(4) == 3)[None, None], entA, entC)
    _fail(ctx, "palette entry of the recorded indices != recorded texel", np.any(rotate(want, R["rot"]) != R["texel"], axis=(1, 2)))
    if px is not None:
        p = rotate(px.astype(np.int64), R["rot"])
        cm = np.where(np.isin(R["mode"], (6, 7)), 4, 3)                   # channels of the colour index set (slot order)
        chan = np.arange(4)[None, :] < cm[:, None]
        dC = ((palC - p[:, :, None, :]) ** 2 * chan[:, None, None, :]).sum(-1)
        dC = np.where(np.arange(16)[None, None, :] < nC[:, None, None], dC, 1 << 40)
        dA = (palA[..., 3] - p[:, :, None, 3]) ** 2
        dA = np.where(np.arange(8)[None, None, :] < nA[:, None, None], dA, 1 << 40)
        _fail(ctx, "colour index not the nearest palette entry", np.any(dC.argmin(-1) != R["idxC"], axis=1),
              lambda b: "mode %d: nearest %s, recorded %s" % (R["mode"][b], dC[b].argmin(-1).tolist(), R["idxC"][b].tolist()))
        _fail(ctx, "alpha index not the nearest palette entry", sepA & np.any(dA.argmin(-1) != R["idxA"], axis=1))
        # stage 4 takes the exact nearest entry of the winner's palette per pixel, while the stage-3 error of the same endpoints is
        # the exact integer error of one index choice per pixel (dxb_bc7_eval), so the decoded error can only be lower
        sse = ((dec - px.astype(np.int64)) ** 2).sum((1, 2))
        _fail(ctx, "decoded squared error > the stage-3 error it was chosen by", sse > R["err"],
              lambda b: "mode %d: %d > %d" % (R["mode"][b], sse[b], R["err"][b]))
    return R


def bc6h_unquantize(q, prec, signed):
    """Unquantize + FinishUnquantize of the format description, elementwise"""
    q = np.asarray(q, np.int64)
    if signed:
        a = np.abs(q)
        if prec >= 16:
            u = a
        else:
            u = np.where(a == 0, 0, np.where(a >= (1 << (prec - 1)) - 1, 0x7FFF, ((a << 15) + 0x4000) >> (prec - 1)))
        return np.where(q < 0, -u, u)
    if prec >= 15:
        return q
    return np.where(q == 0, 0, np.where(q == (1 << prec) - 1, 0xFFFF, ((q << 16) + 0x8000) >> prec))


def bc6h_finish(v, signed):
    v = np.asarray(v, np.int64)
    if signed:
        return np.where(v < 0, -(((-v) * 31) >> 5), (v * 31) >> 5)
    return (v * 31) >> 6


def check_bc6h(ref, T, blocks, rec, fmt, px=None, ctx=""):
    """(a) the reference decoder's values, in the INT domain of half bits, equal the recorded texels; (b) the stream's mode, shape
    and indices equal the record; (c) the recorded endpoints interpolated as the format describes give the recorded texels, and
    with the blocks' INT pixels px [blocks, 16, 3] (None: skip) every index is the exhaustive nearest palette entry (anchors: the
    first half of the palette; ties: lowest index) under the encoder's fp32 distance, and within fp32 rounding of the exact nearest.
    Returns the record fields."""
    signed = fmt == SF16
    R = bc6h_fields(rec)
    n = R["mode"].size
    dec = oracle_lib.bc6h_to_int(decoded_blocks(ref, fmt, blocks)[..., :3], signed)
    _fail(ctx, "reference decode != recorded INT texels", np.any(dec != R["texel"], axis=(1, 2)),
          lambda b: "mode %d (%#x): decoded %s, recorded %s" % (R["mode"][b], BC6H_MODES[R["mode"][b]][0], dec[b].tolist(), R["texel"][b].tolist()))
    P = parse_bc6h(bits_of(blocks), T)
    _fail(ctx, "stream mode != record", P["mode"] != R["mode"])
    two = np.array([BC6H_MODES[m][1] == 2 for m in R["mode"]])
    _fail(ctx, "stream shape != record", two & (P["shape"] != R["shape"]))
    _fail(ctx, "stored indices != record", np.any(P["idx"] != R["idx"], axis=1))
    pal = np.zeros((n, 16, 16, 3), np.int64)
    nk = np.zeros((n, 16), np.int64)
    for r in range(n):
        m = int(R["mode"][r])
        _, regions, prec, _ = BC6H_MODES[m]
        ib = 3 if regions == 2 else 4
        s = int(R["shape"][r])
        region = T.part2[s] if regions == 2 else np.zeros(16, np.int64)
        w = np.array(WEIGHTS[ib])
        for j in range(regions):
            ua, ub = bc6h_unquantize(R["wq"][r, 2 * j], prec, signed), bc6h_unquantize(R["wq"][r, 2 * j + 1], prec, signed)
            p = bc6h_finish((ua[None, :] * (64 - w[:, None]) + ub[None, :] * w[:, None] + 32) >> 6, signed)
            pal[r, region == j, :len(w)] = p[None]
        anchors = [0] + ([int(T.anchor2[s, 1])] if regions == 2 else [])
        nk[r] = 1 << ib
        nk[r, anchors] = 1 << (ib - 1)
    ent = pal[np.arange(n)[:, None], np.arange(16)[None], R["idx"]]
    _fail(ctx, "palette entry of the recorded index != recorded texel", np.any(ent != R["texel"], axis=(1, 2)))
    if px is not None:
        # The encoder ranks the entries in fp32, fma(dx, dx, fma(dy, dy, dz dz)) with a strict < over ascending index.  The differences
        # are integers below 2^17, so each product is exact in float64 and so is each sum of a product and an fp32 value: rounding
        # every step to fp32 reproduces the fused operations exactly.  Above a squared distance of 2^24 that metric rounds, so two
        # entries whose exact distances differ by less than its resolution can rank either way: the index must be the nearest under
        # the encoder's metric, and under the exact metric within fp32 rounding of the nearest.
        dd = (pal - px.astype(np.int64)[:, :, None, :]).astype(np.float64)
        f = (dd[..., 2] * dd[..., 2]).astype(np.float32).astype(np.float64)
        f = (dd[..., 1] * dd[..., 1] + f).astype(np.float32).astype(np.float64)
        f = (dd[..., 0] * dd[..., 0] + f).astype(np.float32)
        valid = np.arange(16)[None, None, :] < nk[:, :, None]
        f = np.where(valid, f, np.float32(np.inf))
        _fail(ctx, "index not the nearest palette entry under the encoder's fp32 metric", np.any(f.argmin(-1) != R["idx"], axis=1),
              lambda b: "mode %d: nearest %s, recorded %s" % (R["mode"][b], f[b].argmin(-1).tolist(), R["idx"][b].tolist()))
        d = np.where(valid, (dd ** 2).sum(-1), np.inf)
        got = np.take_along_axis(d, R["idx"][..., None], -1)[..., 0]
        _fail(ctx, "index farther than fp32 rounding from the exact nearest palette entry", np.any(got > d.min(-1) * (1 + 2.0 ** -21), axis=1))
    return R


# ---- corpora ------------------------------------------------------------------------------------------------------------------
def blocks_to_image(px, nbx, nby):
    """[nbx * nby, 16, C] block pixels (raster block order) -> (4 nby, 4 nbx, C) image"""
    return np.ascontiguousarray(px.reshape(nby, nbx, 4, 4, -1).transpose(0, 2, 1, 3, 4).reshape(nby * 4, nbx * 4, -1))


def structured_ldr(T, n, seed, alpha, shapes=None, nsub=None):
    """[n, 16, 4] LDR blocks (floats 0..1): per block one, two or three subsets on a BC7 partition (random, or `shapes` with `nsub`),
    each subset two flat colours or one line with its pixels at random positions on it; near-equal colours in a quarter of the
    blocks; alpha 255 unless `alpha`"""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 16, 4))
    for b in range(n):
        ns = int(nsub if nsub is not None else rng.integers(1, 4))
        s = int(shapes[b] if shapes is not None else rng.integers(0, 16 if ns == 3 and rng.random() < 0.3 else 64))
        part = T.part2[s] if ns == 2 else T.part3[s] if ns == 3 else np.zeros(16, np.int64)
        near = rng.random() < 0.25
        base = rng.integers(0, 256, 4)
        for j in range(ns):
            c0 = np.clip(base + rng.integers(-3, 4, 4), 0, 255) if near else rng.integers(0, 256, 4)
            c1 = np.clip(c0 + rng.integers(-2, 3, 4), 0, 255) if near else rng.integers(0, 256, 4)
            t = rng.integers(0, 2, 16) if rng.random() < 0.5 else rng.random(16)
            v = c0[None, :] + t[:, None] * (c1 - c0)[None, :]
            out[b, part == j] = v[part == j]
        if not alpha:
            out[b, :, 3] = 255
    return (np.floor(out) / 255.0).astype(np.float32)


def int_to_float(v, signed):
    """INT-domain values (half bits; sign-magnitude for the signed format) -> float32"""
    v = np.asarray(v, np.int64)
    h = np.where(v < 0, 0x8000 | (-v), v).astype(np.uint16) if signed else v.astype(np.uint16)
    return h.view(np.float16).astype(np.float32)


def structured_hdr(T, n, seed, signed, shapes=None):
    """[n, 16, 4] float blocks: per block two regions on a BC6H shape (random or `shapes`), or a random pixel mask, each region two
    flat colours; magnitudes 1e-4 .. 6e4, both signs for the signed format, near-equal colours in a third of the blocks"""
    rng = np.random.default_rng(seed)
    out = np.ones((n, 16, 4), np.float32)
    for b in range(n):
        if shapes is None and rng.random() < 0.2:
            # near-flat in the INT domain: one colour and offsets of a few units per channel, larger in one channel
            base = rng.integers(1, 0x7BFF - 600, 3) * (rng.choice([-1, 1], 3) if signed else 1)
            amp = np.array([1, 1, 1]) * int(rng.choice([2, 8, 40])) * np.where(np.arange(3) == rng.integers(0, 3), int(rng.choice([1, 4, 12])), 1)
            v = base[None, :] + rng.integers(0, 2, (16, 1)) * rng.integers(-1, 2, (1, 3)) * amp[None, :]
            out[b, :, :3] = int_to_float(np.clip(v, -0x7BFF if signed else 0, 0x7BFF), signed)
            continue
        s = int(shapes[b] if shapes is not None else rng.integers(0, 32))
        region = T.part2[s] if (shapes is not None or rng.random() < 0.7) else rng.integers(0, 2, 16)
        scale = 10.0 ** rng.uniform(-4, 4.8)
        for j in range(2):
            a = rng.uniform(-1 if signed else 0, 1, 3) * scale
            spread = 10.0 ** rng.uniform(-4, -2) if rng.random() < 0.33 else 10.0 ** rng.uniform(-2, 0)
            c = a + rng.normal(0, 1, 3) * scale * spread
            pick = rng.integers(0, 2, 16)
            v = np.where(pick[:, None] == 1, c[None, :], a[None, :])
            out[b, region == j, :3] = v[region == j]
    return np.clip(out, -65504, 65504).astype(np.float32)


# ---- forced cells -------------------------------------------------------------------------------------------------------------
def bc7_forced_cells(T, per=2, seed=0):
    """(force [n, 5], opaque-or-alpha content [n, 16, 4], flags) of the forced BC7 cells: every partition of modes 0 (16), 1, 2, 3
    and 7 (64 each); modes 4 and 5 at every rotation, mode 4 at both index selectors; mode 6; on opaque and (modes 4-7) alpha
    content.  Two-subset modes on two-subset content of the forced shape, three-subset modes on three-subset content."""
    force, px = [], []
    for m, n_shapes, ns, alpha in ((1, 64, 2, False), (3, 64, 2, False), (7, 64, 2, True), (0, 16, 3, False), (2, 64, 3, False)):
        shapes = np.repeat(np.arange(n_shapes), per)
        px.append(structured_ldr(T, shapes.size, seed + m, alpha, shapes, ns))
        for s in shapes:
            force.append((m, -1, -1, s, -1) if ns == 2 else (m, -1, -1, -1, s))
    for alpha in (False, True):
        cells = [(4, r, i) for r in range(4) for i in range(2)] + [(5, r, -1) for r in range(4)] + [(6, -1, -1)]
        for m, r, i in cells:
            px.append(structured_ldr(T, 4 * per, seed + 100 * m + 10 * r + i + alpha, alpha, None, 1))
            force += [(m, r, i, -1, -1)] * (4 * per)
    return np.array(force, np.int32), np.concatenate(px)


def bc6h_forced_cells(T, signed, per=2, seed=0):
    """(force [n, 2], content [n, 16, 4]) of the forced BC6H cells: every two-region mode at each of the 32 shapes and every
    one-region mode.  Content: per region two flat colours whose quantised codes, at the forced mode's precision, lie within the
    mode's delta range of the block's first endpoint, decoded to INT values and stored as half floats."""
    rng = np.random.default_rng(seed + signed)
    force, px = [], []
    for m, (code, regions, prec, db) in enumerate(BC6H_MODES):
        shapes = np.repeat(np.arange(32), per) if regions == 2 else np.full(16 * per, -1)
        for s in shapes:
            qhi = (1 << (prec - 1)) - 1 if signed else (1 << prec) - 1
            qlo = -qhi if signed else 0
            d = min(db) if min(db) else prec
            r = max(1, (1 << (d - 1)) // 2)
            base = rng.integers(qlo + r, qhi - r + 1, 3) if qhi - qlo > 2 * r else rng.integers(qlo, qhi + 1, 3)
            q = np.clip(base[None, :] + rng.integers(-r, r + 1, (4, 3)), qlo, qhi)
            q[0] = base
            v = bc6h_finish(bc6h_unquantize(q, prec, signed), signed)
            region = T.part2[s] if regions == 2 else np.zeros(16, np.int64)
            blk = np.ones((16, 4), np.float32)
            for j in range(regions):
                pick = rng.integers(0, 2, 16)
                blk[region == j, :3] = int_to_float(np.where(pick[:, None] == 1, v[2 * j + 1][None], v[2 * j][None]), signed)[region == j]
            px.append(blk)
            force.append((m, s))
    return np.array(force, np.int32), np.stack(px)


def bc6h_requantize(q, prec, signed):
    """the code the encoder's endpoint quantisation (dxb_bc6h_pick_mode) gives the decoded value of code q: q itself for every code
    below 16-bit precision; at 16 bits the smallest code that decodes to the same value"""
    v = bc6h_finish(bc6h_unquantize(q, prec, signed), signed)
    a = np.abs(v)
    if prec >= (16 if signed else 15):
        mag = np.minimum((a * 32 + 30) // 31, 0x7FFF) if signed else np.minimum((a * 64 + 30) // 31, 0xFFFF)
    else:
        mag = ((a << 11) // 0x7C00 if signed else (a << 12) // 0x7C00) >> (12 - prec)
    return np.where(v < 0, -mag, mag)


def bc6h_edge_cells(T, signed, variants=4, seed=0):
    """(force [n, 2], content [n, 16, 4], cells [n]) of the BC6H endpoint-range cells, `variants` blocks each:
      ("delta", mode, channel, d): in every transformed mode and channel an emitted delta of d = -2^(n-1) and d = 2^(n-1) - 1, the
                                   ends of its n-bit field;
      ("base", mode, channel, b):  in every mode and channel the base endpoint A0 at b = the lowest code, 0 and the highest code the
                                   quantisation returns: the highest code of the field, except at 16-bit unsigned precision, where
                                   2^16 - 1 and 2^16 - 2 decode to the same value and the encoder takes the smaller.  At
                                   16-bit signed precision the codes -1, 0 and 1 all decode to 0, and the +-1 code refinement
                                   (dxb_bc6h_refine_region) keeps the lowest of equal-error codes, so a base of value 0 is
                                   emitted as -1: the cell there is b = -1, built from a base of code 0.
    Each block is built from chosen codes: per region two flat colours, the decoded values of its two endpoint codes, the anchor
    pixel on endpoint A; every channel's codes differ inside a region, every delta fits its field, and every code is the one the
    encoder's quantisation returns for its own decoded value.  The shape of two-region blocks is random."""
    rng = np.random.default_rng(seed + 2 * signed)
    force, px, cells = [], [], []
    for m, (code, regions, prec, db) in enumerate(BC6H_MODES):
        qhi = (1 << (prec - 1)) - 1 if signed else (1 << prec) - 1
        qlo = -qhi if signed else 0
        nep = 2 * regions
        transformed = db[0] > 0
        targets = [("delta", m, c, d) for c in range(3) for d in ((-(1 << (db[c] - 1)), (1 << (db[c] - 1)) - 1) if transformed else ())]
        top = int(bc6h_requantize(np.array(qhi), prec, signed))              # qhi, except 2^16 - 2 at 16-bit unsigned precision
        zero = -1 if (signed and prec == 16) else 0                          # the code a base of value 0 is emitted as
        targets += [("base", m, c, b) for c in range(3) for b in sorted({qlo, zero, top})]
        for cell in targets:
            kind, _, ch, val = cell
            made = 0
            for _ in range(20000):
                if made == variants:
                    break
                q = np.zeros((nep, 3), np.int64)
                for c in range(3):
                    span = (1 << (db[c] - 1)) - 1 if transformed else qhi - qlo
                    q[0, c] = rng.integers(qlo, qhi + 1)
                    if kind == "base" and c == ch:
                        q[0, c] = 0 if val == zero else val
                    lo, hi = (max(qlo, q[0, c] - span - (1 if transformed else 0)), min(qhi, q[0, c] + span)) if transformed else (qlo, qhi)
                    q[1:, c] = rng.integers(lo, hi + 1, nep - 1)
                    if kind == "delta" and c == ch:
                        q[rng.integers(1, nep), c] = q[0, c] + val
                if q.min() < qlo or q.max() > qhi or np.any(q[0::2] == q[1::2]):
                    continue
                if not np.array_equal(bc6h_requantize(q, prec, signed), q):
                    continue
                s = int(rng.integers(0, 32)) if regions == 2 else -1
                region = T.part2[s] if regions == 2 else np.zeros(16, np.int64)
                anchors = (0, int(T.anchor2[s, 1])) if regions == 2 else (0,)
                v = bc6h_finish(bc6h_unquantize(q, prec, signed), signed)
                blk = np.ones((16, 4), np.float32)
                for j in range(regions):
                    pix = np.nonzero(region == j)[0]
                    pick = rng.integers(0, 2, pix.size)
                    pick[pix == anchors[j]] = 0
                    pick[rng.choice(np.nonzero(pix != anchors[j])[0])] = 1       # both colours present
                    blk[pix, :3] = int_to_float(v[2 * j + pick], signed)
                px.append(blk)
                force.append((m, s))
                cells.append(cell)
                made += 1
            assert made == variants, ("no code set for", cell)
    return np.array(force, np.int32), np.stack(px), cells


def bc6h_edge_reached(R, cell):
    """the blocks of record R whose emitted endpoints hold `cell` (bc6h_edge_cells)"""
    kind, m, c, val = cell
    wq = R["wq"]
    nep = 2 * BC6H_MODES[m][1]
    if kind == "base":
        return (R["mode"] == m) & (wq[:, 0, c] == val)
    return (R["mode"] == m) & np.any(wq[:, 1:nep, c] - wq[:, :1, c] == val, axis=1)


# ---- stratified decoder streams -----------------------------------------------------------------------------------------------
def _set_bits(blocks, pos, n, value):
    bits = bits_of(blocks)
    for k in range(n):
        bits[:, pos + k] = (value >> k) & 1
    return np.packbits(bits.astype(np.uint8), axis=1, bitorder="little").reshape(-1)


def _pair(rng, n, vmin, vmax, rel):
    """n endpoint pairs (e0, e1) in [vmin, vmax] with e0 > e1, e0 == e1 or e0 < e1 exactly; rel may be one string or one per pair"""
    a = rng.integers(vmin, vmax + 1, n)
    b = rng.integers(vmin, vmax, n)
    b = b + (b >= a)                                            # uniform over the values other than a
    hi, lo = np.maximum(a, b), np.minimum(a, b)
    rel = np.broadcast_to(np.asarray(rel), (n,))
    return np.where(rel == "==", a, np.where(rel == ">", hi, lo)), np.where(rel == "==", a, np.where(rel == ">", lo, hi))


def decoder_streams(bc, nb, seed):
    """[(label, nb random blocks of `bc` with one stratum's selector fields set)]: every BC7 mode and the reserved mode, every BC6H
    mode field and the four reserved ones, BC1 colour endpoints c0 > c1, c0 == c1, c0 < c1, BC3 / BC4 / BC5 alpha (red, green)
    endpoints a0 > a1, a0 == a1, a0 < a1, and BC4S / BC5S endpoints -128 and -127 in both orders"""
    rng = np.random.default_rng(seed)
    size = F.BLOCK_BYTES[bc]
    def rand():
        return rng.integers(0, 256, (nb, size), dtype=np.uint8)
    out = []
    if bc in (98, 99):
        for m in range(8):
            b = rand()
            b[:, 0] = (b[:, 0] & ~np.uint8((2 << m) - 1)) | np.uint8(1 << m)
            out.append(("mode %d" % m, b.reshape(-1)))
        b = rand()
        b[:, 0] = 0
        out.append(("reserved mode", b.reshape(-1)))
    elif bc in (95, 96):
        for code in [m[0] for m in BC6H_MODES] + list(BC6H_RESERVED):
            n = 2 if code < 2 else 5
            out.append(("mode field %#04x" % code, _set_bits(rand(), 0, n, code)))
    elif bc in (71, 72, 74, 75, 77, 78):
        off = 0 if bc in (71, 72) else 8
        for k, rel in enumerate((">", "==", "<")):
            b = rand()
            c0, c1 = _pair(rng, nb, 0, 0xFFFF, rel)
            b[:, off:off + 4] = np.stack([c0, c1], 1).astype(np.uint16).view(np.uint8).reshape(nb, 4)
            if bc in (77, 78):                                  # the alpha endpoints of the same blocks in every order, too
                a0, a1 = _pair(rng, nb, 0, 255, np.array([">", "==", "<"])[(np.arange(nb) + k) % 3])
                b[:, 0], b[:, 1] = a0, a1
            out.append(("c0 %s c1" % rel, b.reshape(-1)))
    else:                                                       # BC4 / BC5, unsigned and signed: every channel block
        signed = bc in (81, 84)
        offs = (0,) if bc in (80, 81) else (0, 8)
        vmin, vmax = (-128, 127) if signed else (0, 255)
        fixed = {"-128 / -127": (-128, -127), "-127 / -128": (-127, -128), "-128 / -128": (-128, -128)}
        for rel in (">", "==", "<") + (tuple(fixed) if signed else ()):
            b = rand()
            for off in offs:
                a0, a1 = (np.full(nb, fixed[rel][0]), np.full(nb, fixed[rel][1])) if rel in fixed else _pair(rng, nb, vmin, vmax, rel)
                b[:, off:off + 2] = np.stack([a0, a1], 1).astype(np.int8 if signed else np.uint8).view(np.uint8)
            out.append((rel if rel in fixed else "a0 %s a1" % rel, b.reshape(-1)))
    return out
