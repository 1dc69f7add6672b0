"""Measures dxb200_levels_from against the separate host calls it stands for (development tool; bench.py is the project benchmark).

W1: 64 x 1024^2 BC3 chains (11 levels) re-encoded as BC7_UNORM with premultiply and the alpha-opaque answer (texconv -f BC7_UNORM
    -pmalpha on DDS files that keep their mips).  Separate calls over all the levels: dxb200_decompress (-> R8G8B8A8_UNORM),
    dxb200_premultiply_alpha, dxb200_compress, dxb200_is_alpha_all_opaque.
W2: 32 x 2048^2 BC5_UNORM normal-map chains (12 levels) back to BC5_UNORM with invert Y (texconv -inverty).  Separate calls:
    dxb200_decompress (-> R8G8_UNORM), dxb200_apply_channel_steps, dxb200_compress.
Every buffer is pinned (dxb200_host_alloc); a host clock runs around calls that end synchronised; the two ways alternate run by run,
medians and ranges are reported, and the outputs and answers must be identical.  Host traffic per level-0 texel is computed from the
shapes, not measured.

Usage: python tools/levels_from_bench.py [--reps N] [--out FILE]
Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from directxtex_b200 import capi, formats as F  # noqa: E402
from tools.chain_steps_bench import card, cutout_rgba8, pinned, stats  # noqa: E402

L = capi.lib


def images(fmt, layout, buf, per, items):
    return capi.images([capi.Image(lw, lh, fmt, r, sp, buf.ctypes.data + i * per + off) for i in range(items) for (off, lw, lh, r, sp) in layout])


def bc_chains(content, w, bc, items, uniq):
    """(pinned buffer of `items` BC chains as a DDS file holds them, the layout): each level made from RGBA8 content by the library's
    mips and encoder, `uniq` different chains repeated"""
    layout, total = capi.texture_layout(bc, w, w, 1, F.count_mips(w, w))
    chains = []
    for s in range(uniq):
        rgba, rl = capi.generate_mipmaps(content(w, w, s), w, w, 28)
        chains.append(np.concatenate([capi.compress(rgba[o:o + sl], lw, lh, 28, bc) for (o, lw, lh, _, sl) in rl]))
    buf, _ = pinned(items * total)
    for i in range(items):
        buf[i * total:(i + 1) * total] = chains[i % uniq]
    return buf, layout, total


def normals_rgba8(w, h, seed):
    """a tangent-space normal map: x and y of a rolling height field in R and G"""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32) * (0.02 + 0.01 * seed)
    nx, ny = np.cos(xx) * np.sin(1.7 * yy), np.sin(1.3 * xx + seed) * np.cos(yy)
    img = np.zeros((h, w, 4), np.uint8)
    img[..., 0], img[..., 1], img[..., 3] = ((nx * 0.5 + 0.5) * 255 + 0.5).astype(np.uint8), ((ny * 0.5 + 0.5) * 255 + 0.5).astype(np.uint8), 255
    return img


def run(one, separate, out_one, out_sep, reps):
    a, b = one(), separate()                                # warm-up of every shape
    t_one, t_sep = [], []
    for _ in range(reps):
        for fn, ts in ((one, t_one), (separate, t_sep)):
            t0 = time.perf_counter(); r = fn(); ts.append(time.perf_counter() - t0)
            assert r == (a if fn is one else b)
    assert a == b, "alpha-opaque answers differ"
    assert np.array_equal(out_one, out_sep), "one call and the separate calls differ"
    return {"one_call": stats(t_one), "separate_calls": stats(t_sep), "identical": True, "alpha_all_opaque": bool(a)}


def w1(reps, items=64, w=1024):
    bc, rgba, df = 77, 28, 98
    base, blayout, btotal = bc_chains(cutout_rgba8, w, bc, items, 8)
    levels = len(blayout)
    rlayout, rtotal = capi.texture_layout(rgba, w, w, 1, levels)
    olayout, ototal = capi.texture_layout(df, w, w, 1, levels)
    dec, _ = pinned(items * rtotal)
    pm, _ = pinned(items * rtotal)
    out_one, _ = pinned(items * ototal)
    out_sep, _ = pinned(items * ototal)
    bases = images(bc, blayout, base, btotal, items)
    decs, pms = images(rgba, rlayout, dec, rtotal, items), images(rgba, rlayout, pm, rtotal, items)
    d_one, d_sep = images(df, olayout, out_one, ototal, items), images(df, olayout, out_sep, ototal, items)
    n, steps = items * levels, capi.chain_steps(0.0, True)

    def one():
        op = C.c_int32(-1)
        assert L.dxb200_levels_from(bases, items, levels, None, None, df, 0, 0, 0.5, C.byref(steps), d_one, C.byref(op)) == 0
        return op.value

    def separate():
        op = C.c_int32(-1)
        assert L.dxb200_decompress(bases, n, rgba, decs) == 0
        assert L.dxb200_premultiply_alpha(decs, n, 0, pms) == 0
        assert L.dxb200_compress(pms, n, df, 0, 0.5, 1.0, d_sep) == 0
        assert L.dxb200_is_alpha_all_opaque(d_sep, n, C.byref(op)) == 0
        return op.value

    k = rtotal / (4 * w * w)                                 # texels of a chain per level-0 texel
    traffic = {"one_call": 2 * k, "separate_calls": (1 + 4 + 4 + 4 + 4 + 1 + 1) * k}
    return dict(items=items, size=w, levels=levels, **run(one, separate, out_one, out_sep, reps), host_bytes_per_texel=traffic)


def w2(reps, items=32, w=2048):
    bc, rg = 83, 49
    base, blayout, btotal = bc_chains(normals_rgba8, w, bc, items, 4)
    levels = len(blayout)
    glayout, gtotal = capi.texture_layout(rg, w, w, 1, levels)
    dec, _ = pinned(items * gtotal)
    inv, _ = pinned(items * gtotal)
    out_one, _ = pinned(items * btotal)
    out_sep, _ = pinned(items * btotal)
    bases = images(bc, blayout, base, btotal, items)
    decs, invs = images(rg, glayout, dec, gtotal, items), images(rg, glayout, inv, gtotal, items)
    d_one, d_sep = images(bc, blayout, out_one, btotal, items), images(bc, blayout, out_sep, btotal, items)
    n, channels = items * levels, capi.channel_steps(invert_y=True)

    def one():
        assert L.dxb200_levels_from(bases, items, levels, None, C.byref(channels), bc, 0, 0, 0.5, None, d_one, None) == 0
        return 1

    def separate():
        assert L.dxb200_decompress(bases, n, rg, decs) == 0
        assert L.dxb200_apply_channel_steps(decs, n, C.byref(channels), invs) == 0
        assert L.dxb200_compress(invs, n, bc, 0, 0.5, 1.0, d_sep) == 0
        return 1

    k = gtotal / (2 * w * w)
    traffic = {"one_call": 2 * k, "separate_calls": (1 + 2 + 2 + 2 + 2 + 1) * k}
    return dict(items=items, size=w, levels=levels, **run(one, separate, out_one, out_sep, reps), host_bytes_per_texel=traffic)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert L.dxb200_init(0) == 0
    out = {"card": card(), "W1_bc3_to_bc7_pmalpha": w1(a.reps), "W2_bc5_invert_y": w2(a.reps)}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
