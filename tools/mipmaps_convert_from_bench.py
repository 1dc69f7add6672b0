"""Measures dxb200_mipmaps_convert_from against the separate host calls it stands for (development tool; bench.py is the project
benchmark).

W1: 16 x 2048^2 RGBA32F -> R16G16B16A16_FLOAT full CUBIC chains with the alpha-opaque answer.  Separate calls: dxb200_convert into
    level 0 of the chains, dxb200_generate_mipmaps, dxb200_is_alpha_all_opaque of every level.
W2: 64 x 1024^2 BC3 cut-outs -> B8G8R8A8_UNORM full chains with coverage 0.5, premultiply and the alpha-opaque answer.  Separate
    calls: dxb200_decompress (-> R8G8B8A8_UNORM), dxb200_convert into level 0, dxb200_generate_mipmaps,
    dxb200_scale_mipmaps_alpha_for_coverage per item, dxb200_premultiply_alpha, dxb200_is_alpha_all_opaque.
Every buffer is pinned (dxb200_host_alloc); a host clock runs around calls that end synchronised; the two ways alternate run by run,
medians and ranges are reported, and the outputs and answers must be identical.  Host traffic per level-0 texel is computed from the
shapes, not measured.

Usage: python tools/mipmaps_convert_from_bench.py [--reps N] [--out FILE]
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
from directxtex_b200 import capi, formats as F, synth  # noqa: E402
from tools.chain_steps_bench import card, cutout_rgba8, pinned, stats  # noqa: E402

L = capi.lib


def images(fmt, layout, buf, per, items):
    return capi.images([capi.Image(lw, lh, fmt, r, sp, buf.ctypes.data + i * per + off) for i in range(items) for (off, lw, lh, r, sp) in layout])


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


def w1(reps, items=16, w=2048):
    sf, df, filt = 2, 10, F.TEX_FILTER_CUBIC
    levels = F.count_mips(w, w)
    bsl = F.compute_pitch(sf, w, w)[1]
    layout, total = capi.texture_layout(df, w, w, 1, levels)
    base, _ = pinned(items * bsl)
    for i in range(items):
        base[i * bsl:(i + 1) * bsl] = np.ascontiguousarray(synth.photo_rgba32f(w, w, seed=i % 4, alpha=True)).view(np.uint8).reshape(-1)
    out_one, _ = pinned(items * total)
    out_sep, _ = pinned(items * total)
    bases = images(sf, [(0, w, w, w * 16, bsl)], base, bsl, items)
    d_one, d_sep = images(df, layout, out_one, total, items), images(df, layout, out_sep, total, items)
    lvl0 = capi.images([d_sep[i * levels] for i in range(items)])

    def one():
        op = C.c_int32(-1)
        assert L.dxb200_mipmaps_convert_from(bases, items, None, None, df, 0, 0.5, levels, filt, None, d_one, C.byref(op)) == 0
        return op.value

    def separate():
        op = C.c_int32(-1)
        assert L.dxb200_convert(bases, items, df, 0, 0.5, lvl0) == 0
        assert L.dxb200_generate_mipmaps(d_sep, items, levels, filt) == 0
        assert L.dxb200_is_alpha_all_opaque(d_sep, items * levels, C.byref(op)) == 0
        return op.value

    chain = total / (w * w)                                  # bytes of a chain per level-0 texel
    traffic = {"one_call": 16 + chain, "separate_calls": 16 + 8 + 8 + (chain - 8) + chain}
    return dict(items=items, size=w, **run(one, separate, out_one, out_sep, reps), host_bytes_per_texel=traffic)


def w2(reps, items=64, w=1024):
    bc, rgba, df, ref = 77, 28, 87, 0.5
    levels = F.count_mips(w, w)
    brow, bsl = F.compute_pitch(bc, w, w)
    crow, csl = F.compute_pitch(rgba, w, w)
    layout, total = capi.texture_layout(df, w, w, 1, levels)
    uniq = [capi.compress(cutout_rgba8(w, w, s), w, w, rgba, bc) for s in range(8)]
    base, _ = pinned(items * bsl)
    for i in range(items):
        base[i * bsl:(i + 1) * bsl] = uniq[i % len(uniq)]
    dec, _ = pinned(items * csl)
    out_one, _ = pinned(items * total)
    mips, _ = pinned(items * total)
    cov, _ = pinned(items * total)
    out_sep, _ = pinned(items * total)
    bases = images(bc, [(0, w, w, brow, bsl)], base, bsl, items)
    decs = images(rgba, [(0, w, w, crow, csl)], dec, csl, items)
    d_one = images(df, layout, out_one, total, items)
    d_mips, d_cov, d_sep = images(df, layout, mips, total, items), images(df, layout, cov, total, items), images(df, layout, out_sep, total, items)
    lvl0 = capi.images([d_mips[i * levels] for i in range(items)])
    source, steps = capi.chain_source(), capi.chain_steps(ref, True)

    def one():
        op = C.c_int32(-1)
        assert L.dxb200_mipmaps_convert_from(bases, items, C.byref(source), None, df, 0, 0.5, levels, 0, C.byref(steps), d_one, C.byref(op)) == 0
        return op.value

    def separate():
        op = C.c_int32(-1)
        assert L.dxb200_decompress(bases, items, rgba, decs) == 0
        assert L.dxb200_convert(decs, items, df, 0, 0.5, lvl0) == 0
        assert L.dxb200_generate_mipmaps(d_mips, items, levels, 0) == 0
        for i in range(items):
            s = C.cast(C.byref(d_mips, i * levels * C.sizeof(capi.Image)), C.POINTER(capi.Image))
            d = C.cast(C.byref(d_cov, i * levels * C.sizeof(capi.Image)), C.POINTER(capi.Image))
            assert L.dxb200_scale_mipmaps_alpha_for_coverage(s, levels, ref, d) == 0
        assert L.dxb200_premultiply_alpha(d_cov, items * levels, 0, d_sep) == 0
        assert L.dxb200_is_alpha_all_opaque(d_sep, items * levels, C.byref(op)) == 0
        return op.value

    chain = total / (w * w)
    traffic = {"one_call": 1 + chain, "separate_calls": (1 + 4) + (4 + 4) + (4 + chain - 4) + 2 * chain + 2 * chain + chain}
    return dict(items=items, size=w, **run(one, separate, out_one, out_sep, reps), host_bytes_per_texel=traffic)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert L.dxb200_init(0) == 0
    out = {"card": card(), "W1_rgba32f_to_rgba16f_cubic": w1(a.reps), "W2_bc3_to_bgra8_coverage_pmalpha": w2(a.reps)}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
