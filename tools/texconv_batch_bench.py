"""Measures dxb200_texconv_batch against a loop of the single calls it stands for (development tool; bench.py is the project benchmark).

W1: 96 BC3 textures that keep their own mips, sizes drawn from {256^2, 512^2, 1024^2, 2048^2, 1024 x 512, 512 x 256}, re-encoded as
    BC7_UNORM with the alpha-opaque answer (kind 2, dxb200_levels_from_ex; texconv -f BC7_UNORM over a folder of DDS files).
W2: 256 RGBA8 textures, sizes drawn from the powers of two 128-2048 per axis, 15 % of them any size from 100 to 2000, made into full
    BC3_UNORM chains with the alpha-opaque answer (kind 0, dxb200_mipmaps_compress_from_channels_ex; texconv -m 0 -f BC3_UNORM).
Each workload runs three ways: the loop of single calls on one thread (device 0), the batch on device 0 and the batch on every visible
device.  Inputs are seeded, every buffer is pinned (dxb200_host_alloc), a host clock runs around calls that end synchronised, the ways
alternate run by run after one warm-up run each, medians and ranges are reported with the launches per texture, and the outputs and
answers of the three ways must be identical.

Usage: python tools/texconv_batch_bench.py [--reps N] [--out FILE]
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
from tools.chain_steps_bench import card, pinned, stats  # noqa: E402

L = capi.lib
POOL = np.random.default_rng(1).integers(0, 256, 64 << 20, dtype=np.uint8)      # seeded texel bytes every input is cut from


def _sizes(w, h, levels):
    out = []
    for _ in range(levels):
        out.append((w, h))
        w, h = max(1, w // 2), max(1, h // 2)
    return out


class Workload:
    """the jobs of one workload: pinned bases cut from POOL, and one pinned set of dst images per way"""

    def __init__(self, kind, bf, df, sizes, ways):
        self.kind, self.df, self.n = kind, df, len(sizes)
        self.base, self.levels, self.out_sizes = [], [], []
        for (w, h) in sizes:
            levels = F.count_mips(w, h)
            bsizes = _sizes(w, h, levels) if kind == 2 else [(w, h)]
            self.levels.append(levels)
            self.base.append([(bw, bh) for (bw, bh) in bsizes])
            self.out_sizes.append(_sizes(w, h, levels))
        nbytes = sum(F.compute_pitch(bf, w, h)[1] for b in self.base for (w, h) in b)
        self.hbase, _ = pinned(nbytes)
        at, self.bimg = 0, []
        for k, b in enumerate(self.base):
            ims = []
            for (w, h) in b:
                row, sl = F.compute_pitch(bf, w, h)
                src = (k * 7919 * 4096) % (len(POOL) - sl)
                self.hbase[at:at + sl] = POOL[src:src + sl]
                ims.append(capi.Image(w, h, bf, row, sl, self.hbase.ctypes.data + at))
                at += sl
            self.bimg.append(capi.images(ims))
        obytes = sum(F.compute_pitch(df, w, h)[1] for o in self.out_sizes for (w, h) in o)
        self.out = {}
        for way in ways:
            buf, _ = pinned(obytes)
            at, dims = 0, []
            for o in self.out_sizes:
                ims = []
                for (w, h) in o:
                    row, sl = F.compute_pitch(df, w, h)
                    ims.append(capi.Image(w, h, df, row, sl, buf.ctypes.data + at))
                    at += sl
                dims.append(capi.images(ims))
            self.out[way] = (buf, dims, [C.c_int32(-1) for _ in sizes])
        self.texels = sum(w * h for (w, h) in sizes)

    def jobs(self, way):
        _, dims, opaque = self.out[way]
        return [capi.TexconvJob(self.kind, self.bimg[k], 1, self.levels[k], None, None, 0, None, None, self.df, 0, 0, 0.5, dims[k],
                                C.pointer(opaque[k])) for k in range(self.n)]


def single(j):
    if j.kind == 0:
        return L.dxb200_mipmaps_compress_from_channels_ex(j.base, j.items, j.source, j.channels, j.levels, j.filter, j.steps, j.dstFormat,
                                                          j.compressFlags, j.threshold, 1.0, j.dst, j.alphaAllOpaque, j.ts)
    return L.dxb200_levels_from_ex(j.base, j.items, j.levels, j.source, j.channels, j.dstFormat, j.convertFilter, j.compressFlags, j.threshold,
                                   j.steps, j.dst, j.alphaAllOpaque, j.ts)


_current = []


def run(wl, way, devices):
    """one timed run of `way`; the initialised devices change (untimed, with one warm-up run) only when `devices` differ"""
    if _current != devices:
        L.dxb200_shutdown()
        capi.init_devices(devices)
        _current[:] = devices
        run(wl, way, devices)
    jobs = wl.jobs(way)
    n0 = L.dxb200_launch_count()
    t0 = time.perf_counter()
    if way == "loop":
        for j in jobs:
            hr = single(j)
            assert hr == 0, (hex(F.hr_u32(hr)), capi.last_error())
    else:
        table = (capi.TexconvJob * len(jobs))(*jobs)
        hr = L.dxb200_texconv_batch(table, len(jobs), None)
        assert hr == 0, (hex(F.hr_u32(hr)), capi.last_error())
    t = time.perf_counter() - t0
    return t, (L.dxb200_launch_count() - n0) / len(jobs)


def measure(name, wl, reps, ndev):
    ways = {"loop": [0], "batch_device0": [0], "batch_all_devices": list(range(ndev))}
    times = {w: [] for w in ways}
    launches = {}
    for w, devs in ways.items():
        run(wl, w, devs)                                 # warm-up: module loads, slot buffers, the memory pool
    for _ in range(reps):
        for w, devs in ways.items():
            t, per = run(wl, w, devs)
            times[w].append(t)
            launches[w] = per
    ref_buf, _, ref_op = wl.out["loop"]
    for w in ways:
        buf, _, op = wl.out[w]
        assert np.array_equal(buf, ref_buf), (name, w)
        assert [o.value for o in op] == [o.value for o in ref_op], (name, w)
    return {"textures": wl.n, "level0_texels": wl.texels, "devices": ndev,
            "ways": {w: dict(stats(times[w]), launches_per_texture=launches[w]) for w in ways}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ndev = L.dxb200_device_count()
    assert ndev >= 1, "no CUDA device: nothing to measure"
    rng = np.random.default_rng(2024)
    ways = ("loop", "batch_device0", "batch_all_devices")
    w1_sizes = [(256, 256), (512, 512), (1024, 1024), (2048, 2048), (1024, 512), (512, 256)]
    w1 = Workload(2, 77, 98, [w1_sizes[k] for k in rng.integers(0, len(w1_sizes), 96)], ways)
    pow2 = [128, 256, 512, 1024, 2048]
    w2_sizes = [(int(rng.integers(100, 2001)), int(rng.integers(100, 2001))) if rng.random() < 0.15 else
                (pow2[rng.integers(0, 5)], pow2[rng.integers(0, 5)]) for _ in range(256)]
    w2 = Workload(0, 28, 77, w2_sizes, ways)
    res = {"card": card(), "W1_bc3_levels_to_bc7": measure("W1", w1, a.reps, ndev), "W2_rgba8_to_bc3_chains": measure("W2", w2, a.reps, ndev)}
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt)


if __name__ == "__main__":
    main()
