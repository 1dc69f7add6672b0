#!/usr/bin/env python
"""Generate directxtex_b200/csrc/dxb_bc67_tables.h: the BC6H/BC7 format-spec constant tables
(partition shapes, anchor/fix-up indices) in COMPACT bit-mask form.

The numbers are constants of the BC6H/BC7 bit format (any conforming codec has the same ones);
they are read here from the reference's arrays (BC6HBC7.cpp:57-325) so that they are provably
the same values, and re-encoded as bit masks (one 16-bit word per 2-subset shape, one 32-bit
word with 2 bits per pixel per 3-subset shape) — the form the reference's own compute shaders
use (Shaders/BC7Encode.hlsl:18-55).  Run in the build container only (needs /root/reference).
"""
import os
import re
src = open('/root/reference/DirectXTex/BC6HBC7.cpp').read()
def grab(name, dims):
    i = src.index(name)
    j = src.index('};', i)
    body = src[src.index('=', i) + 1:j]
    body = re.sub(r'//[^\n]*', '', body)
    nums = [int(x) for x in re.findall(r'\d+', body)]
    n = 1
    for d in dims: n *= d
    assert len(nums) == n, (name, len(nums), n)
    return nums
pt = grab('g_aPartitionTable[3][64][16]', (3, 64, 16))
fx = grab('g_aFixUp[3][64][3]', (3, 64, 3))
P = lambda r, s, i: pt[(r * 64 + s) * 16 + i]
F = lambda r, s, k: fx[(r * 64 + s) * 3 + k]
p2 = [sum((P(1, s, i) & 1) << i for i in range(16)) for s in range(64)]
p3 = [sum(P(2, s, i) << (2 * i) for i in range(16)) for s in range(64)]
a2 = [F(1, s, 1) for s in range(64)]
a3a = [F(2, s, 1) for s in range(64)]
a3b = [F(2, s, 2) for s in range(64)]
assert all(F(1, s, 0) == 0 and F(2, s, 0) == 0 for s in range(64))
# A-operand fragments (mma.sync m16n8k16, row-major 16x16 bf16) of the 0/1 matrix  S[shape][pixel] = bit `pixel` of
# dxb_part2[shape]: tiles 0..3 = shapes 16t..16t+15, tile 4 = one row of ones (whole-block totals) then zeros.
# Thread (g = lane >> 2, q = lane & 3) holds {S[g][2q],S[g][2q+1]}, {S[g+8][..]}, {S[g][2q+8],..}, {S[g+8][2q+8],..}.
def _pair(mask, k):
    ONE = 0x3F80
    return (ONE if (mask >> k) & 1 else 0) | ((ONE if (mask >> (k + 1)) & 1 else 0) << 16)
afrag = []
for t in range(5):
    for lane in range(32):
        g, q = lane >> 2, lane & 3
        rows = [p2[16 * t + g], p2[16 * t + g + 8]] if t < 4 else [0xFFFF if g == 0 else 0, 0]
        afrag += [_pair(rows[0], 2 * q), _pair(rows[1], 2 * q), _pair(rows[0], 2 * q + 8), _pair(rows[1], 2 * q + 8)]
# per-pixel words of the stage-1 projections (dxb_bc7.cuh, dxb_bc7_shape_h1): bits 0-15 = byte-permute selector of the pixel's axis
# (0x3210: subset 0's register, 0x7654: subset 1's), the whole word = the pixel's projection bias; entry 8s + k = pixels 2k, 2k + 1.
_h1w = lambda s, i: 0x00307654 if (p2[s] >> i) & 1 else 0x00043210
h1sel = [_h1w(s, 2 * k) | (_h1w(s, 2 * k + 1) << 32) for s in range(64) for k in range(8)]
# BC7 block layout per mode (D3DX_BC7 mode table, BC6HBC7.cpp:1106-1124; bit order of D3DX_BC7::Decode, :2566-2780): mode (unary),
# partition, rotation, index selector, then R of every endpoint, G, B, A, p-bits, colour indices, alpha indices.
# (colour bits, alpha bits, p-bit type 0 none / 1 per endpoint / 2 per subset, subsets, partition bits, rotation bits, selector bits,
#  colour index bits, alpha index bits)
BC7_MODES = [(4, 0, 1, 3, 4, 0, 0, 3, 0), (6, 0, 2, 2, 6, 0, 0, 3, 0), (5, 0, 0, 3, 6, 0, 0, 2, 0), (7, 0, 1, 2, 6, 0, 0, 2, 0),
             (5, 6, 0, 1, 0, 2, 1, 2, 3), (7, 8, 0, 1, 0, 2, 0, 2, 2), (7, 7, 1, 1, 0, 0, 0, 4, 0), (5, 5, 1, 2, 6, 0, 0, 2, 0)]
# Stage 4 of the encoder (dxb_bc7.cuh) reads one layout word per (mode, index selector) and one field word per (mode, lane).
# dxb_bc7_lay[m | sel << 3] (sel = the index selector, only ever 1 in mode 4; other modes repeat their sel = 0 word):
#   bits 0-2 colour index bits, 3-5 alpha index bits (0: no alpha index set), 6-7 subsets, 8 alpha searched with the colour set,
#   9-15 first index bit - w (w = 32 in mode 4, whose first index set crosses bit 64, else 64), 16 w == 32, 17 the first index set is
#   the alpha set, 18-20 bits of the first index set, 21-23 bits of the second set (0: none), 24-30 first bit of the second set - 64 (1: none),
#   32-39 the header's constant bits (mode in unary, index selector), 40-43 the shift of the partition or rotation field (mode + 1).
lay = []
for key in range(16):
    mode, sel = key & 7, key >> 3
    sel = sel if mode == 4 else 0
    cb, ab, pt, ns, partb, rotb, imb, ibc, iba = BC7_MODES[mode]
    if mode == 4:
        ibc, iba = (3, 2) if sel else (2, 3)
    hdrb = mode + 1 + partb + rotb + imb
    npb = 2 * ns if pt == 1 else (ns if pt == 2 else 0)
    first = hdrb + ns * 2 * (3 * cb + ab) + npb
    ib1, ib2 = (2, 3) if mode == 4 else (ibc, iba)
    second = first + 16 * ib1 - ns
    w = 32 if mode == 4 else 64
    # every index set but mode 4's first one lies in bits 64..127, mode 4's first one in bits 32..95
    assert w < first and first + 16 * ib1 - ns <= w + 64 and (ib2 == 0 or (second > 64 and second + 16 * ib2 - 1 == 128))
    assert ib2 == 0 or first + 16 * ib1 - ns == second
    hdr = (1 << mode) | (sel << (mode + 1 + partb + rotb))
    lay.append(ibc | (iba << 3) | (ns << 6) | ((1 if mode in (6, 7) else 0) << 8) | ((first - w) << 9) | ((1 if w == 32 else 0) << 16) |
               ((1 if (mode == 4 and sel) else 0) << 17) | (ib1 << 18) | (ib2 << 21) | (((second - 64) if ib2 else 1) << 24) |
               (hdr << 32) | ((mode + 1) << 40))
# dxb_bc7_lay_ep[16 m + l]: the endpoint fields l (bits 0-31) and l + 16 (bits 32-63) of mode m (field f = channel * 2 * subsets +
# endpoint, endpoint = 2 * subset + 0 / 1; every field lies in bits 0..98).  Per field: bits 0-6 position p, 7-8 subset, 12-14 the
# byte of the subset's endpoint pair (endpoint * 4 + channel: a byte-permute selector that moves it to the top byte), 16-22 120 - p,
# 26-31 32 - width (32: no such field).
# dxb_bc7_lay_pb[16 m + l]: position (63..97) of the p-bit that lane l deposits, 0 for none: per endpoint (p-bit type 1) lane l
# holds the R field of endpoint l; per subset (type 2) lane 2 s holds the R field of subset s's first endpoint.  The p-bit is
# the bit of that R byte just below its field.
lay_ep, lay_pb = [], []
for mode, (cb, ab, pt, ns, partb, rotb, imb, ibc, iba) in enumerate(BC7_MODES):
    hdrb = mode + 1 + partb + rotb + imb
    per = 2 * ns
    pbs = hdrb + ns * 2 * (3 * cb + ab)
    for l in range(16):
        words = []
        for fi in (l, l + 16):
            if fi >= 4 * per or (fi >= 3 * per and ab == 0):
                words.append(32 << 26)
                continue
            c, e = fi // per, fi % per
            nb = ab if c == 3 else cb
            pos = hdrb + (3 * per * cb + e * ab if c == 3 else (c * per + e) * cb)
            assert pos + nb <= 99 and 8 - nb <= pos
            words.append(pos | ((e >> 1) << 7) | ((((e & 1) << 2) | c) << 12) | ((120 - pos) << 16) | ((32 - nb) << 26))
        lay_ep.append(words[0] | (words[1] << 32))
        q = 0
        if pt == 1 and l < per:
            q = pbs + l
        elif pt == 2 and l < per and l % 2 == 0:
            q = pbs + l // 2
        assert q == 0 or 63 <= q <= 97
        lay_pb.append(q)
def arr(name, ctype, vals, fmt, per=8):
    out = [f'DXB_TABLE {ctype} {name}[{len(vals)}] = {{']
    for k in range(0, len(vals), per):
        out.append('    ' + ', '.join(fmt % v for v in vals[k:k + per]) + ',')
    out.append('};')
    return '\n'.join(out)
hdr = '''// dxb_bc67_tables.h — GENERATED by tools/gen_bc67_tables.py; do not edit.
// BC6H/BC7 bit-format constants in compact mask form:
//   dxb_part2[s]   bit i = subset (0/1) of pixel i for 2-subset shape s      (BC6HBC7.cpp:127-194)
//   dxb_part3[s]   bits 2i..2i+1 = subset (0/1/2) of pixel i, 3-subset shape (BC6HBC7.cpp:196-261)
//   dxb_anchor2[s] anchor (fix-up) pixel of subset 1, 2-subset shapes        (BC6HBC7.cpp:285-307)
//   dxb_anchor3a/b[s] anchors of subsets 1 and 2, 3-subset shapes            (BC6HBC7.cpp:309-325)
//   dxb_bc7_afrag[t*128 + lane*4 + r]  tensor-core A fragments of the shape/pixel membership matrix (dxb_bc7.cuh stage 1)
//   dxb_bc7_h1sel[8s + k]  words of pixels 2k (bits 0-31) and 2k + 1 (bits 32-63) of shape s: 0x00043210 subset 0, 0x00307654 subset 1
//                          (axis selector + projection bias of the stage-1 shape ranking, dxb_bc7.cuh)
//   dxb_bc7_lay[m | sel << 3]  BC7 mode m, index selector sel: index bits, subsets, index-field windows, header pieces
//   dxb_bc7_lay_ep[16m + l], dxb_bc7_lay_pb[16m + l]  endpoint fields l and l + 16 and the p-bit that lane l of mode m packs
//                          (block packer, dxb_bc7.cuh stage 4; bit layouts in tools/gen_bc67_tables.py)
// Subset 0's anchor is always pixel 0.
#pragma once
#include <stdint.h>
#ifndef DXB_TABLE
#if defined(__CUDACC__)
#define DXB_TABLE static __device__ const
#else
#define DXB_TABLE static const
#endif
#endif
'''
body = '\n\n'.join([
    arr('dxb_part2', 'uint16_t', p2, '0x%04X'),
    arr('dxb_part3', 'uint32_t', p3, '0x%08X', 4),
    arr('dxb_anchor2', 'uint8_t', a2, '%2d', 16),
    arr('dxb_anchor3a', 'uint8_t', a3a, '%2d', 16),
    arr('dxb_anchor3b', 'uint8_t', a3b, '%2d', 16),
    arr('dxb_bc7_afrag', 'uint32_t', afrag, '0x%08X', 4),
    arr('dxb_bc7_h1sel', 'uint64_t', h1sel, '0x%016XULL', 4),
    arr('dxb_bc7_lay', 'uint64_t', lay, '0x%016XULL', 4),
    arr('dxb_bc7_lay_ep', 'uint64_t', lay_ep, '0x%016XULL', 4),
    arr('dxb_bc7_lay_pb', 'uint8_t', lay_pb, '%2d', 16),
])
out = os.path.join(os.path.dirname(__file__), '..', 'directxtex_b200', 'csrc', 'dxb_bc67_tables.h')
open(out, 'w').write(hdr + '\n' + body + '\n')
print('wrote', os.path.normpath(out))

# ---- BC6H header bit layouts (ms_aDesc, BC6HBC7.cpp:879-1048) and mode table (ms_aInfo :1051-1067) -------------------
def gen_bc6h():
    i = src.index('D3DX_BC6H::ms_aDesc[D3DX_BC6H::c_NumModes][82] =')
    j = src.index('// Mode, Partitions, Transformed, IndexPrec, RGBAPrec', i)
    body = re.sub(r'//[^\n]*', '', src[i:j])
    ents = re.findall(r'\{\s*([A-Z]{1,2})\s*,\s*(\d+)\s*\}', body)
    assert len(ents) == 14 * 82, len(ents)
    fields = ['NA', 'M', 'D', 'RW', 'RX', 'RY', 'RZ', 'GW', 'GX', 'GY', 'GZ', 'BW', 'BX', 'BY', 'BZ']
    codes = [(fields.index(f) << 4) | int(b) for f, b in ents]
    k = src.index('D3DX_BC6H::ms_aInfo[D3DX_BC6H::c_NumModes] =')
    l = src.index('};', k)
    rows = re.findall(r'\{\s*(0x[0-9a-f]+)\s*,\s*(\d)\s*,\s*(true|false)\s*,\s*(\d)\s*,\s*\{\s*\{\s*LDRColorA\((\d+),\s*(\d+),\s*(\d+),\s*0\)\s*,\s*LDRColorA\((\d+),\s*(\d+),\s*(\d+)', src[k:l])
    assert len(rows) == 14
    info = []
    for (m, parts, tr, ip, p0r, p0g, p0b, p1r, p1g, p1b) in rows:
        # packed: mode bits(5) | partitions<<5 | transformed<<6 | base prec<<8 (5 bits) | delta r<<16 | delta g<<20 | delta b<<24
        info.append(int(m, 16) | (int(parts) << 5) | ((1 if tr == 'true' else 0) << 6) | (int(p0r) << 8) | (int(p1r) << 16) | (int(p1g) << 20) | (int(p1b) << 24))
    hdr2 = '''// dxb_bc6h_tables.h — GENERATED by tools/gen_bc67_tables.py; do not edit.
// BC6H bit-format constants:
//   dxb_bc6h_desc[mode][bit]  header bit -> (field << 4) | bit-of-field; fields: 0 NA, 1 M (mode), 2 D (shape),
//                             3..6 RW RX RY RZ, 7..10 GW GX GY GZ, 11..14 BW BX BY BZ     (BC6HBC7.cpp:879-1048)
//   dxb_bc6h_info[mode]       mode bits | partitions<<5 | transformed<<6 | base precision<<8 |
//                             delta bits r<<16 g<<20 b<<24                                  (BC6HBC7.cpp:1051-1067)
// mode index 0..13 = "Mode 1".."Mode 14" of the format specification.
#pragma once
#include <stdint.h>
#ifndef DXB_TABLE
#if defined(__CUDACC__)
#define DXB_TABLE static __device__ const
#else
#define DXB_TABLE static const
#endif
#endif
'''
    lines = ['DXB_TABLE uint8_t dxb_bc6h_desc[14][82] = {']
    for m in range(14):
        row = codes[m * 82:(m + 1) * 82]
        lines.append('    { ' + ', '.join('0x%02X' % c for c in row) + ' },')
    lines.append('};')
    lines.append('')
    lines.append('DXB_TABLE uint32_t dxb_bc6h_info[14] = { ' + ', '.join('0x%08X' % v for v in info) + ' };')
    out2 = os.path.join(os.path.dirname(__file__), '..', 'directxtex_b200', 'csrc', 'dxb_bc6h_tables.h')
    open(out2, 'w').write(hdr2 + '\n' + '\n'.join(lines) + '\n')
    print('wrote', os.path.normpath(out2))


gen_bc6h()
