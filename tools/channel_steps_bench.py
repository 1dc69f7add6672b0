"""Measures texconv's channel steps (development tool; bench.py is the project benchmark).

1. 64 x 1024^2 BC5_UNORM normal maps with -inverty and -reconstructz -> full BC7 chains, as one dxb200_mipmaps_compress_from_channels
   call and as the separate host calls dxb200_decompress (-> R8G8B8A8_UNORM, the format texconv picks) + dxb200_apply_channel_steps
   + dxb200_mipmaps_compress_from_ex, on pinned buffers, host clock around calls that end synchronised.  The two ways alternate run
   by run; medians are reported, and the outputs must be identical.
2. The steps' kernel alone (the generic k_convert, all four steps) on 64 x 1024^2 RGBA8 images in device memory, in place, timed
   with CUDA events; bytes moved (read + write) over kernel time, against the H100 SXM data sheet's 3.35 TB/s.

Usage: python tools/channel_steps_bench.py [--reps N] [--items N] [--size N] [--out FILE]
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
from tools.chain_steps_bench import card, pinned, stats  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def normal_map(w, seed):
    g = synth.content_ldr("gradient", w, w, seed=seed)
    img = np.full((w, w, 4), 255, np.uint8)
    img[..., :2] = (g[..., :2] * 255).round().astype(np.uint8)
    return img


def one_against_separate(items, w, reps):
    bc, rgba, df = 83, 28, 98
    levels = F.count_mips(w, w)
    brow, bsl = F.compute_pitch(bc, w, w)
    crow, csl = F.compute_pitch(rgba, w, w)
    olayout, ototal = capi.texture_layout(df, w, w, 1, levels)
    uniq = [capi.compress(normal_map(w, s), w, w, rgba, bc) for s in range(8)]
    base, _ = pinned(items * bsl)
    for i in range(items):
        base[i * bsl:(i + 1) * bsl] = uniq[i % len(uniq)]
    dec, _ = pinned(items * csl)
    stepped, _ = pinned(items * csl)
    out_one, _ = pinned(items * ototal)
    out_sep, _ = pinned(items * ototal)
    addr = lambda a: a.ctypes.data
    bases = capi.images([capi.Image(w, w, bc, brow, bsl, addr(base) + i * bsl) for i in range(items)])
    decs = capi.images([capi.Image(w, w, rgba, crow, csl, addr(dec) + i * csl) for i in range(items)])
    steps = capi.images([capi.Image(w, w, rgba, crow, csl, addr(stepped) + i * csl) for i in range(items)])
    outs = lambda buf: capi.images([capi.Image(lw, lh, df, r, sp, addr(buf) + i * ototal + off) for i in range(items) for (off, lw, lh, r, sp) in olayout])
    d_one, d_sep = outs(out_one), outs(out_sep)
    source = capi.chain_source()
    ch = capi.channel_steps(invert_y=True, reconstruct_z=True)

    def one():
        assert capi.lib.dxb200_mipmaps_compress_from_channels(bases, items, C.byref(source), C.byref(ch), levels, 0, None, df, 0, 0.5, 1.0,
                                                              d_one, None) == 0

    def separate():
        assert capi.lib.dxb200_decompress(bases, items, rgba, decs) == 0
        assert capi.lib.dxb200_apply_channel_steps(decs, items, C.byref(ch), steps) == 0
        assert capi.lib.dxb200_mipmaps_compress_from_ex(steps, items, None, levels, 0, None, df, 0, 0.5, 1.0, d_sep, None) == 0

    one(); separate()                                           # warm-up of every shape
    t_one, t_sep = [], []
    for _ in range(reps):
        for fn, ts in ((one, t_one), (separate, t_sep)):
            t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    assert np.array_equal(out_one, out_sep), "one call and the separate calls differ"
    return {"items": items, "size": w, "one_call": stats(t_one), "separate_calls": stats(t_sep), "identical": True}


def kernel_alone(items, w, reps):
    import torch
    rgba = 28
    row, sl = F.compute_pitch(rgba, w, w)
    buf = torch.randint(0, 256, (items * sl,), dtype=torch.uint8, device="cuda")
    imgs = capi.images([capi.Image(w, w, rgba, row, sl, buf.data_ptr() + i * sl) for i in range(items)])
    ch = capi.channel_steps(swizzle=(1, 0, 2, 3), color_key=0x4080C0, invert_y=True, reconstruct_z=True)
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    call = lambda: capi.lib.dxb200_apply_channel_steps_device(imgs, items, C.byref(ch), imgs, sp)
    for _ in range(3):
        assert call() == 0
    k0 = capi.kernel_launch_count("k_convert")
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); assert call() == 0; e1.record(stream)
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    assert capi.kernel_launch_count("k_convert") - k0 == reps
    t = float(np.median(times))
    moved = 2.0 * items * sl
    return {"items": items, "size": w, "format": rgba, "steps": "swizzle, colour key, invert Y, reconstruct Z", "kernel_ms": t * 1e3,
            "GB_per_s": moved / t / 1e9, "share_of_3.35_TB_per_s": moved / t / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--items", type=int, default=64)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert capi.lib.dxb200_init(0) == 0
    out = {"card": card(), "bc5_normals_to_bc7": one_against_separate(a.items, a.size, a.reps),
           "kernel": kernel_alone(a.items, a.size, 20)}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
