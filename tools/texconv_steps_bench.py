"""Measures texconv's BC3n layout and -alpha steps inside the one-call pipelines against the split sequences a caller needs without
them (development tool; bench.py is the project benchmark).

W1: 32 x 2048^2 BC5_UNORM normal maps -> 12-level chains -> BC3n (texconv -f BC3n).  One call: dxb200_mipmaps_compress_from_channels_ex
    with bc3Layout = 1.  Split: dxb200_mipmaps_convert_from (Decompress to R8G8B8A8_UNORM, mips, every level down), then
    dxb200_apply_channel_steps with the layout's swizzle and masks and dxb200_compress over all levels.
W2: 64 x 1024^2 premultiplied BC3 -> -alpha -> 11-level chains -> BC7_UNORM with -pmalpha and the alpha-opaque answer.  One call:
    dxb200_mipmaps_compress_from_channels_ex with demultiply.  Split: dxb200_decompress, dxb200_premultiply_alpha(REVERSE), then
    dxb200_mipmaps_compress_from_ex with premultiply and the alpha answer.
Every buffer is pinned (dxb200_host_alloc); a host clock runs around calls that end synchronised; the two ways alternate run by run,
medians and ranges are reported, and the outputs and answers must be identical.

Usage: python tools/texconv_steps_bench.py [--reps N] [--out FILE]
Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from directxtex_b200 import capi, formats as F  # noqa: E402
from tools.chain_steps_bench import card, cutout_rgba8, pinned  # noqa: E402
from tools.levels_from_bench import normals_rgba8, run  # noqa: E402

L = capi.lib


def images(fmt, layout, buf, per, items):
    return capi.images([capi.Image(lw, lh, fmt, r, sp, buf.ctypes.data + i * per + off) for i in range(items) for (off, lw, lh, r, sp) in layout])


def bc_bases(content, w, bc, items, uniq):
    """(pinned buffer of `items` w x w images of bc, each image's bytes): `uniq` different ones made by the library's encoder, repeated"""
    blocks = [capi.compress(content(w, w, s), w, w, 28, bc) for s in range(uniq)]
    per = blocks[0].size
    buf, _ = pinned(items * per)
    for i in range(items):
        buf[i * per:(i + 1) * per] = blocks[i % uniq]
    return buf, per


def w1(reps, items=32, w=2048):
    bc, rgba, df = 83, 28, 77
    base, per = bc_bases(normals_rgba8, w, bc, items, 4)
    levels = F.count_mips(w, w)
    rlayout, rtotal = capi.texture_layout(rgba, w, w, 1, levels)
    olayout, ototal = capi.texture_layout(df, w, w, 1, levels)
    chain, _ = pinned(items * rtotal)
    laid, _ = pinned(items * rtotal)
    out_one, _ = pinned(items * ototal)
    out_sep, _ = pinned(items * ototal)
    bases = images(bc, [(0, w, w) + F.compute_pitch(bc, w, w)], base, per, items)
    chains, lays = images(rgba, rlayout, chain, rtotal, items), images(rgba, rlayout, laid, rtotal, items)
    d_one, d_sep = images(df, olayout, out_one, ototal, items), images(df, olayout, out_sep, ototal, items)
    n = items * levels
    to_rgba8 = capi.chain_source(decompress_format=rgba)
    ts = capi.texconv_steps(bc3_layout=1)
    layout = capi.channel_steps(swizzle=(0, 1, 2, 0), zero_mask=0x4, one_mask=0x1)

    def one():
        assert L.dxb200_mipmaps_compress_from_channels_ex(bases, items, C.byref(capi.chain_source()), None, levels, 0, None, df, 0, 0.5, 1.0,
                                                          d_one, None, C.byref(ts)) == 0
        return 1

    def separate():
        assert L.dxb200_mipmaps_convert_from(bases, items, C.byref(to_rgba8), None, rgba, 0, 0.5, levels, 0, None, chains, None) == 0
        assert L.dxb200_apply_channel_steps(chains, n, C.byref(layout), lays) == 0
        assert L.dxb200_compress(lays, n, df, 0, 0.5, 1.0, d_sep) == 0
        return 1

    k = rtotal / (4 * w * w)                                 # texels of a chain per level-0 texel
    traffic = {"one_call": 1 + k, "separate_calls": 1 + (4 + 4 + 4 + 4 + 4 + 1) * k}
    return dict(items=items, size=w, levels=levels, **run(one, separate, out_one, out_sep, reps), host_bytes_per_texel=traffic)


def w2(reps, items=64, w=1024):
    bc, rgba, df = 77, 28, 98
    base, per = bc_bases(cutout_rgba8, w, bc, items, 8)
    levels = F.count_mips(w, w)
    olayout, ototal = capi.texture_layout(df, w, w, 1, levels)
    dec, _ = pinned(items * w * w * 4)
    dm, _ = pinned(items * w * w * 4)
    out_one, _ = pinned(items * ototal)
    out_sep, _ = pinned(items * ototal)
    bases = images(bc, [(0, w, w) + F.compute_pitch(bc, w, w)], base, per, items)
    decs = images(rgba, [(0, w, w) + F.compute_pitch(rgba, w, w)], dec, w * w * 4, items)
    dms = images(rgba, [(0, w, w) + F.compute_pitch(rgba, w, w)], dm, w * w * 4, items)
    d_one, d_sep = images(df, olayout, out_one, ototal, items), images(df, olayout, out_sep, ototal, items)
    steps, ts = capi.chain_steps(0.0, True), capi.texconv_steps(demultiply=True)

    def one():
        op = C.c_int32(-1)
        assert L.dxb200_mipmaps_compress_from_channels_ex(bases, items, C.byref(capi.chain_source()), None, levels, 0, C.byref(steps), df, 0,
                                                          0.5, 1.0, d_one, C.byref(op), C.byref(ts)) == 0
        return op.value

    def separate():
        op = C.c_int32(-1)
        assert L.dxb200_decompress(bases, items, rgba, decs) == 0
        assert L.dxb200_premultiply_alpha(decs, items, 0x2, dms) == 0
        assert L.dxb200_mipmaps_compress_from_ex(dms, items, None, levels, 0, C.byref(steps), df, 0, 0.5, 1.0, d_sep, C.byref(op)) == 0
        return op.value

    k = ototal / (w * w)                                     # output bytes per level-0 texel
    traffic = {"one_call": 1 + k, "separate_calls": 1 + 4 + 4 + 4 + 4 + k}
    return dict(items=items, size=w, levels=levels, **run(one, separate, out_one, out_sep, reps), host_bytes_per_texel=traffic)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert L.dxb200_init(0) == 0
    out = {"card": card(), "W1_bc5_to_bc3n": w1(a.reps), "W2_bc3_demultiply_to_bc7": w2(a.reps)}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
