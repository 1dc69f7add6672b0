"""Measures texconv's mips -> alpha coverage -> premultiply -> BC3 chain (development tool; bench.py is the project benchmark).

1. One call against four: 64 x 1024^2 RGBA8 chains of synth.content_ldr("cutout") -> BC3 with coverage 0.5 and premultiply, as one
   dxb200_mipmaps_compress_ex call and as the four host-pointer calls (generate_mipmaps, scale_mipmaps_alpha_for_coverage per item,
   premultiply_alpha, compress), on pinned buffers, host clock around calls that end synchronised.  Outputs must be identical.
2. The coverage step alone on device-resident chains (1 x 4096^2, 64 x 1024^2): dxb200_scale_mipmaps_alpha_for_coverage_device per
   item, in this build and in another build of the library (--other-lib, e.g. the parent commit's), alternating in one process.

Usage: python tools/chain_steps_bench.py [--other-lib PATH] [--reps N] [--out FILE]
Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from directxtex_b200 import capi, formats as F, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(ts):
    ts = sorted(ts)
    return {"median_ms": 1e3 * ts[len(ts) // 2], "min_ms": 1e3 * ts[0], "max_ms": 1e3 * ts[-1], "runs": len(ts)}


def pinned(nbytes):
    p = capi.lib.dxb200_host_alloc(nbytes)
    assert p, "dxb200_host_alloc"
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p)), p


def cutout_rgba8(w, h, seed):
    return np.ascontiguousarray((synth.content_ldr("cutout", w, h, seed) * 255 + 0.5).astype(np.uint8))


def one_against_four(items, w, reps):
    fmt, df, ref = 28, 77, 0.5
    levels = F.count_mips(w, w)
    clayout, ctotal = capi.texture_layout(fmt, w, w, 1, levels)
    blayout, btotal = capi.texture_layout(df, w, w, 1, levels)
    uniq = [cutout_rgba8(w, w, s) for s in range(8)]
    base, _ = pinned(items * clayout[0][4])
    for i in range(items):
        base[i * clayout[0][4]:(i + 1) * clayout[0][4]] = uniq[i % len(uniq)].reshape(-1)
    chain, _ = pinned(items * ctotal)
    scaled, _ = pinned(items * ctotal)
    pm, _ = pinned(items * ctotal)
    blocks_ex, _ = pinned(items * btotal)
    blocks_4, _ = pinned(items * btotal)
    addr = lambda a: a.ctypes.data
    s0 = clayout[0]
    bases = capi.images([capi.Image(w, w, fmt, s0[3], s0[4], addr(base) + i * s0[4]) for i in range(items)])
    imgs = lambda buf: capi.images([capi.Image(lw, lh, fmt, r, sp, addr(buf) + i * ctotal + off) for i in range(items) for (off, lw, lh, r, sp) in clayout])
    bimgs = lambda buf: capi.images([capi.Image(lw, lh, df, r, sp, addr(buf) + i * btotal + off) for i in range(items) for (off, lw, lh, r, sp) in blayout])
    steps = capi.chain_steps(ref, True, 0)
    d_ex, c_all, s_all, p_all, d_4 = bimgs(blocks_ex), imgs(chain), imgs(scaled), imgs(pm), bimgs(blocks_4)
    for i in range(items):
        chain[i * ctotal:i * ctotal + s0[4]] = base[i * s0[4]:(i + 1) * s0[4]]

    def ex():
        assert capi.lib.dxb200_mipmaps_compress_ex(bases, items, levels, 0, C.byref(steps), df, 0, 0.5, 1.0, d_ex) == 0

    def four():
        assert capi.lib.dxb200_generate_mipmaps(c_all, items, levels, 0) == 0
        for i in range(items):
            assert capi.lib.dxb200_scale_mipmaps_alpha_for_coverage(C.byref(c_all[i * levels]), levels, ref, C.byref(s_all[i * levels])) == 0
        assert capi.lib.dxb200_premultiply_alpha(s_all, items * levels, 0, p_all) == 0
        assert capi.lib.dxb200_compress(p_all, items * levels, df, 0, 0.5, 1.0, d_4) == 0

    ex(); four()                                                # warm-up of every shape
    t_ex, t_4 = [], []
    for _ in range(reps):
        for fn, ts in ((ex, t_ex), (four, t_4)):
            t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    assert np.array_equal(blocks_ex, blocks_4), "one call and four calls differ"
    return {"items": items, "size": w, "one_call": stats(t_ex), "four_calls": stats(t_4), "identical": True}


def coverage_alone(libs, items, w, reps):
    import torch
    fmt, ref = 28, 0.5
    levels = F.count_mips(w, w)
    layout, total = capi.texture_layout(fmt, w, w, 1, levels)
    src = torch.empty(items * total, dtype=torch.uint8, device="cuda")
    uniq = [torch.from_numpy(cutout_rgba8(w, w, s).reshape(-1)) for s in range(min(items, 4))]
    for i in range(items):
        src[i * total:i * total + layout[0][4]].copy_(uniq[i % len(uniq)])
    base = src.data_ptr()
    chains = capi.images([capi.Image(lw, lh, fmt, r, sp, base + i * total + off) for i in range(items) for (off, lw, lh, r, sp) in layout])
    assert capi.lib.dxb200_generate_mipmaps_device(chains, items, levels, 0, None) == 0
    torch.cuda.synchronize()
    outs, res = {}, {}
    for name, L in libs.items():
        out = torch.zeros_like(src)
        outs[name] = (out, capi.images([capi.Image(lw, lh, fmt, r, sp, out.data_ptr() + i * total + off) for i in range(items)
                                        for (off, lw, lh, r, sp) in layout]))
        res[name] = []

    def run(L, dst):
        for i in range(items):
            assert L.dxb200_scale_mipmaps_alpha_for_coverage_device(C.byref(chains[i * levels]), levels, ref, C.byref(dst[i * levels]), None) == 0
        torch.cuda.synchronize()

    for name, L in libs.items():
        run(L, outs[name][1])                                  # warm-up
    for _ in range(reps):
        for name, L in libs.items():
            t0 = time.perf_counter(); run(L, outs[name][1]); res[name].append(time.perf_counter() - t0)
    names = list(libs)
    same = all(torch.equal(outs[names[0]][0], outs[n][0]) for n in names[1:])
    return {"items": items, "size": w, **{n: stats(res[n]) for n in names}, "identical": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", default=None)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert capi.lib.dxb200_init(0) == 0
    out = {"card": card(), "one_against_four": one_against_four(64, 1024, a.reps)}
    libs = {"this": capi.lib}
    if a.other_lib:
        other = C.CDLL(a.other_lib)
        other.dxb200_init(0)
        other.dxb200_scale_mipmaps_alpha_for_coverage_device.argtypes = [C.POINTER(capi.Image), C.c_size_t, C.c_float, C.POINTER(capi.Image), C.c_void_p]
        other.dxb200_scale_mipmaps_alpha_for_coverage_device.restype = C.c_int32
        libs["other"] = other
    out["coverage_alone"] = [coverage_alone(libs, n, w, a.reps) for (n, w) in ((1, 4096), (64, 1024))]
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
