"""Measures dxb200_texconv_batch_device, texconv over textures already in device memory (development tool; bench.py is the project
benchmark).

W2 (of tools/texconv_batch_bench.py): 256 RGBA8 textures of mixed sizes made into full BC3_UNORM chains with the alpha-opaque answer.
   The device batch on torch CUDA buffers against dxb200_texconv_batch on pinned host buffers holding the same bytes.
C: 64 1024^2 RGBA8 cut-outs made into BC3_UNORM chains with alpha coverage at 0.5, premultiplied alpha and the alpha-opaque answer.
   The device batch against the composed _device calls a caller writes without it: generate_mipmaps over every chain, coverage per
   texture, premultiply, compress, and is_alpha_all_opaque per texture, into caller-allocated chains.
Copy-in: the device-to-device copies the device batch makes of W2's bases (each level 0 into scratch at the next 256-byte boundary),
   timed alone with CUDA events, as a share of the device batch's event time.
Each call ends synchronised (every job asks for the alpha answer); a host clock runs around it.  The ways alternate run by run after
one warm-up run each; medians and ranges of --reps runs are reported, and the outputs and answers of the ways compared must be
identical.

Usage: python tools/texconv_batch_device_bench.py [--reps N] [--out FILE]
Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from directxtex_b200 import capi, formats as F  # noqa: E402
from tools.chain_steps_bench import card, cutout_rgba8, stats  # noqa: E402
from tools.texconv_batch_bench import Workload  # noqa: E402

L = capi.lib
IMG = C.POINTER(capi.Image)


def at(images, k):
    """images k, k + 1, ... of a ctypes array of capi.Image"""
    return C.cast(C.addressof(images) + k * C.sizeof(capi.Image), IMG)


def on_device(images, host_base, dev_base):
    """images whose pixels lie in the host buffer at host_base moved to the same offsets of the device buffer at dev_base"""
    out = []
    for im in images:
        c = capi.Image.from_buffer_copy(im)
        c.pixels = dev_base + (im.pixels - host_base)
        out.append(c)
    return capi.images(out)


class DeviceW2:
    """W2's bases and one set of dst chains in CUDA memory, laid out as the pinned host buffers are"""

    def __init__(self, wl):
        self.wl = wl
        self.base = torch.from_numpy(np.array(wl.hbase)).cuda()
        hb = wl.hbase.ctypes.data
        self.bimg = [on_device(b, hb, self.base.data_ptr()) for b in wl.bimg]
        hbuf, dims, _ = wl.out["host"]
        self.dst = torch.zeros(len(hbuf), dtype=torch.uint8, device="cuda")
        self.dimg = [on_device(d, hbuf.ctypes.data, self.dst.data_ptr()) for d in dims]
        self.opaque = [C.c_int32(-1) for _ in range(wl.n)]

    def jobs(self):
        wl = self.wl
        return [capi.TexconvJob(wl.kind, self.bimg[k], 1, wl.levels[k], None, None, 0, None, None, wl.df, 0, 0, 0.5, self.dimg[k],
                                C.pointer(self.opaque[k])) for k in range(wl.n)]


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def batch_host(jobs):
    table = (capi.TexconvJob * len(jobs))(*jobs)
    hr = L.dxb200_texconv_batch(table, len(jobs), None)
    assert hr == 0, (hex(F.hr_u32(hr)), capi.last_error())


def batch_device(jobs, stream):
    hr, _ = capi.texconv_batch_device(jobs, stream)
    assert hr == 0, (hex(hr), capi.last_error())


def w2(reps, stream):
    rng = np.random.default_rng(2024)
    rng.integers(0, 6, 96)                               # W1's draws, so that W2's sizes are texconv_batch_bench's
    pow2 = [128, 256, 512, 1024, 2048]
    sizes = [(int(rng.integers(100, 2001)), int(rng.integers(100, 2001))) if rng.random() < 0.15 else
             (pow2[rng.integers(0, 5)], pow2[rng.integers(0, 5)]) for _ in range(256)]
    wl = Workload(0, 28, 77, sizes, ("host",))
    dev = DeviceW2(wl)
    ways = {"host_batch_pinned": lambda: batch_host(wl.jobs("host")), "device_batch": lambda: batch_device(dev.jobs(), stream)}
    times = {w: [] for w in ways}
    for fn in ways.values():
        fn()
    for _ in range(reps):
        for w, fn in ways.items():
            times[w].append(timed(fn))
    hbuf, _, hop = wl.out["host"]
    assert np.array_equal(dev.dst.cpu().numpy(), hbuf), "W2 bytes"
    assert [o.value for o in dev.opaque] == [o.value for o in hop], "W2 answers"
    # the copy-in: level 0 of every texture into scratch at the next 256-byte boundary, device to device, against the batch's time
    scratch = torch.empty(sum((im[0].slicePitch + 255) // 256 * 256 for im in wl.bimg), dtype=torch.uint8, device="cuda")
    spans = [(im[0].pixels - wl.hbase.ctypes.data, im[0].slicePitch) for im in wl.bimg]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    share = []
    for _ in range(reps):
        with torch.cuda.stream(stream):
            ev[0].record()
            at = 0
            for off, n in spans:
                scratch[at:at + n].copy_(dev.base[off:off + n])
                at += (n + 255) // 256 * 256
            ev[1].record()
            ev[2].record()
        batch_device(dev.jobs(), stream)
        with torch.cuda.stream(stream):
            ev[3].record()
        stream.synchronize()
        share.append((ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3])))
    copy_ms = sorted(c for c, _ in share)[len(share) // 2]
    batch_ms = sorted(b for _, b in share)[len(share) // 2]
    return {"textures": wl.n, "level0_texels": wl.texels, "ways": {w: stats(t) for w, t in times.items()},
            "copy_in": {"bytes": int(sum(n for _, n in spans)), "median_ms": copy_ms, "device_batch_event_median_ms": batch_ms,
                        "share": copy_ms / batch_ms}}


def composed(n, w, base, chain, opaque, stream):
    """what a caller composes from the _device calls: level 0 of each chain copied from its base, GenerateMipMaps over every chain,
    coverage per texture into a second set of chains, premultiply in place there, Compress, IsAlphaAllOpaque per texture"""
    levels = F.count_mips(w, w)
    handle = stream.cuda_stream
    tch, ch_img, cov_img, bc_img, copies = chain
    with torch.cuda.stream(stream):
        for d, s, nbytes in copies:
            tch[d:d + nbytes].copy_(base[s:s + nbytes])
    hr = L.dxb200_generate_mipmaps_device(ch_img, n, levels, 0, handle)
    assert hr == 0, hex(F.hr_u32(hr))
    for i in range(n):
        hr = L.dxb200_scale_mipmaps_alpha_for_coverage_device(at(ch_img, i * levels), levels, 0.5,
                                                              at(cov_img, i * levels), handle)
        assert hr == 0, hex(F.hr_u32(hr))
    hr = L.dxb200_premultiply_alpha_device(cov_img, n * levels, 0, cov_img, handle)
    assert hr == 0, hex(F.hr_u32(hr))
    hr = L.dxb200_compress_device(cov_img, n * levels, 77, 0, 0.5, 1.0, bc_img, handle)
    assert hr == 0, hex(F.hr_u32(hr))
    for i in range(n):
        hr = L.dxb200_is_alpha_all_opaque_device(at(bc_img, i * levels), levels, C.byref(opaque[i]), handle)
        assert hr == 0, hex(F.hr_u32(hr))


def _chains(fmt, w, n, levels, dev):
    """n chains of fmt in one CUDA tensor, every image on a 256-byte boundary: (tensor, images)"""
    layout = []
    at = 0
    for _ in range(n):
        for (lw, lh) in [(max(1, w >> l), max(1, w >> l)) for l in range(levels)]:
            row, sl = F.compute_pitch(fmt, lw, lh)
            layout.append((lw, lh, row, sl, at))
            at += (sl + 255) // 256 * 256
    t = torch.zeros(at, dtype=torch.uint8, device=dev)
    return t, capi.images([capi.Image(lw, lh, fmt, row, sl, t.data_ptr() + o) for (lw, lh, row, sl, o) in layout])


def cutouts(reps, stream):
    n, w = 64, 1024
    levels = F.count_mips(w, w)
    seeds = [cutout_rgba8(w, w, s) for s in range(8)]
    base = torch.from_numpy(np.concatenate([seeds[i % 8].reshape(-1) for i in range(n)])).cuda()
    row, sl = F.compute_pitch(28, w, w)
    bimg = capi.images([capi.Image(w, w, 28, row, sl, base.data_ptr() + i * sl) for i in range(n)])
    steps = capi.chain_steps(0.5, True)
    tdst, dimg = _chains(77, w, n, levels, "cuda")
    opaque = [C.c_int32(-1) for _ in range(n)]
    jobs = [capi.TexconvJob(0, at(bimg, i), 1, levels, None, None, 0, C.pointer(steps), None, 77, 0, 0, 0.5,
                            at(dimg, i * levels), C.pointer(opaque[i])) for i in range(n)]
    tch, ch_img = _chains(28, w, n, levels, "cuda")
    tcov, cov_img = _chains(28, w, n, levels, "cuda")
    tbc, bc_img = _chains(77, w, n, levels, "cuda")
    copies = [(ch_img[i * levels].pixels - tch.data_ptr(), i * sl, sl) for i in range(n)]
    copts = [C.c_int32(-1) for _ in range(n)]
    ways = {"device_batch": lambda: batch_device(jobs, stream),
            "composed_device_calls": lambda: composed(n, w, base, (tch, ch_img, cov_img, bc_img, copies), copts, stream)}
    times = {k: [] for k in ways}
    for fn in ways.values():
        fn()
    for _ in range(reps):
        for k, fn in ways.items():
            times[k].append(timed(lambda: (fn(), stream.synchronize())))
    assert torch.equal(tdst, tbc), "cut-out bytes"
    assert [o.value for o in opaque] == [o.value for o in copts], "cut-out answers"
    return {"textures": n, "size": w, "ways": {k: stats(t) for k, t in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert L.dxb200_device_count() >= 1 and torch.cuda.is_available(), "no CUDA device: nothing to measure"
    assert L.dxb200_init(0) == 0
    stream = torch.cuda.Stream()
    res = {"card": card(), "W2_rgba8_to_bc3_chains": w2(a.reps, stream), "C_cutouts_coverage_premultiply_bc3": cutouts(a.reps, stream)}
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt)


if __name__ == "__main__":
    main()
