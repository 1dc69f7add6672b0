"""Measures texconv's Decompress -> GenerateMipMaps -> Compress of a BC asset (development tool; bench.py is the project benchmark).

64 x 1024^2 BC3 items of synth.content_ldr("cutout") -> full chains -> BC7 and -> BC1, as one dxb200_mipmaps_compress_from call and
as dxb200_decompress + dxb200_mipmaps_compress_ex, on pinned buffers, host clock around calls that end synchronised.  The two
ways alternate run by run; medians are reported, and the outputs must be identical.

Usage: python tools/mipmaps_compress_from_bench.py [--reps N] [--items N] [--size N] [--out FILE]
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


def from_against_two(items, w, df, reps):
    bc, rgba = 77, 28
    levels = F.count_mips(w, w)
    brow, bsl = F.compute_pitch(bc, w, w)
    clayout, ctotal = capi.texture_layout(rgba, w, w, 1, 1)
    olayout, ototal = capi.texture_layout(df, w, w, 1, levels)
    uniq = [capi.compress(cutout_rgba8(w, w, s), w, w, rgba, bc) for s in range(8)]
    base, _ = pinned(items * bsl)
    for i in range(items):
        base[i * bsl:(i + 1) * bsl] = uniq[i % len(uniq)]
    dec, _ = pinned(items * ctotal)
    out_from, _ = pinned(items * ototal)
    out_two, _ = pinned(items * ototal)
    addr = lambda a: a.ctypes.data
    bases = capi.images([capi.Image(w, w, bc, brow, bsl, addr(base) + i * bsl) for i in range(items)])
    decs = capi.images([capi.Image(w, w, rgba, clayout[0][3], clayout[0][4], addr(dec) + i * ctotal) for i in range(items)])
    outs = lambda buf: capi.images([capi.Image(lw, lh, df, r, sp, addr(buf) + i * ototal + off) for i in range(items) for (off, lw, lh, r, sp) in olayout])
    d_from, d_two = outs(out_from), outs(out_two)
    source = capi.chain_source()

    def one():
        assert capi.lib.dxb200_mipmaps_compress_from(bases, items, C.byref(source), levels, 0, None, df, 0, 0.5, 1.0, d_from) == 0

    def two():
        assert capi.lib.dxb200_decompress(bases, items, rgba, decs) == 0
        assert capi.lib.dxb200_mipmaps_compress_ex(decs, items, levels, 0, None, df, 0, 0.5, 1.0, d_two) == 0

    one(); two()                                                # warm-up of every shape
    t_one, t_two = [], []
    for _ in range(reps):
        for fn, ts in ((one, t_one), (two, t_two)):
            t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    assert np.array_equal(out_from, out_two), "one call and two calls differ"
    return {"items": items, "size": w, "target": df, "one_call": stats(t_one), "two_calls": stats(t_two), "identical": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--items", type=int, default=64)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert capi.lib.dxb200_init(0) == 0
    out = {"card": card(), "bc3_to": [from_against_two(a.items, a.size, df, a.reps) for df in (98, 71)]}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
