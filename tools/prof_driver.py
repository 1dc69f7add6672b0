#!/usr/bin/env python
"""Times each hot-path kernel with CUDA events on device-resident data (two warm-up calls, then `reps` calls).  Usage: python tools/prof_driver.py [bc7|bc6h|bc15|bc3|dec|rows|rowscubic|rowslinear|rowshalf|all] [reps]"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from directxtex_b200 import capi, formats as F, synth  # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "all"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
assert capi.lib.dxb200_init(0) == 0
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).cuda()


def mip_chains(fmt, w, h, items, base, levels=0):
    """`items` chains of `levels` levels (0 = full) in one device buffer, level 0 of each a copy of the device bytes `base`;
    the item stride is padded to 256 bytes so that every item is vector-aligned (as the host-staged path does)"""
    layout, total = F.mip_chain_layout(fmt, w, h, levels)
    total = (total + 255) & ~255
    chain = torch.zeros(total * items, dtype=torch.uint8, device="cuda")
    imgs = []
    for it in range(items):
        chain[it * total: it * total + base.numel()] = base
        for (off, lw, lh, row, sl) in layout:
            imgs.append(capi.Image(lw, lh, fmt, row, sl, chain.data_ptr() + it * total + off))
    return chain, capi.images(imgs), len(layout)


def timed(name, fn, units):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print("%-28s %8.3f ms  %10.1f Munits/s" % (name, ms, units / ms / 1e3))


if what in ("bc7", "all"):
    w = h = 4096
    d_in = dev(synth.c2_rgba32f(w, h))
    d_out = torch.zeros(F.compute_pitch(98, w, h)[1], dtype=torch.uint8, device="cuda")
    s = capi.images([capi.Image(w, h, 2, *F.compute_pitch(2, w, h), d_in.data_ptr())])
    d = capi.images([capi.Image(w, h, 98, *F.compute_pitch(98, w, h), d_out.data_ptr())])
    timed("bc7 4096^2 rgba32f", lambda: capi.lib.dxb200_compress_device(s, 1, 98, 0, 0.5, 1.0, d, st), w * h)

if what in ("bc6h", "all"):
    w = h = 2048
    d_in = dev(synth.c3_rgba16f(w, h))
    d_out = torch.zeros(F.compute_pitch(95, w, h)[1], dtype=torch.uint8, device="cuda")
    s = capi.images([capi.Image(w, h, 10, *F.compute_pitch(10, w, h), d_in.data_ptr())])
    d = capi.images([capi.Image(w, h, 95, *F.compute_pitch(95, w, h), d_out.data_ptr())])
    timed("bc6h 2048^2 rgba16f (C3)", lambda: capi.lib.dxb200_compress_device(s, 1, 95, 0, 0.5, 1.0, d, st), w * h)

if what in ("bc15", "all"):
    w = h = 8192
    d_in = dev(synth.c5_r8(w, h))
    d_out = torch.zeros(F.compute_pitch(80, w, h)[1], dtype=torch.uint8, device="cuda")
    s = capi.images([capi.Image(w, h, 61, *F.compute_pitch(61, w, h), d_in.data_ptr())])
    d = capi.images([capi.Image(w, h, 80, *F.compute_pitch(80, w, h), d_out.data_ptr())])
    timed("bc4 8192^2 r8 (C5)", lambda: capi.lib.dxb200_compress_device(s, 1, 80, 0, 0.5, 1.0, d, st), w * h)
    w = h = 4096
    img = np.tile(synth.c1_rgba8(1024, 1024), (4, 4, 1))
    d_in = dev(img)
    for fmt, nm in ((71, "bc1"), (77, "bc3")):
        d_out = torch.zeros(F.compute_pitch(fmt, w, h)[1], dtype=torch.uint8, device="cuda")
        s = capi.images([capi.Image(w, h, 28, *F.compute_pitch(28, w, h), d_in.data_ptr())])
        d = capi.images([capi.Image(w, h, fmt, *F.compute_pitch(fmt, w, h), d_out.data_ptr())])
        timed("%s 4096^2 rgba8" % nm, lambda: capi.lib.dxb200_compress_device(s, 1, fmt, 0, 0.5, 1.0, d, st), w * h)

if what == "bc3":
    w = h = 4096
    d_in = dev(np.tile(synth.c1_rgba8(1024, 1024), (4, 4, 1)))
    d_out = torch.zeros(F.compute_pitch(77, w, h)[1], dtype=torch.uint8, device="cuda")
    s = capi.images([capi.Image(w, h, 28, *F.compute_pitch(28, w, h), d_in.data_ptr())])
    d = capi.images([capi.Image(w, h, 77, *F.compute_pitch(77, w, h), d_out.data_ptr())])
    timed("bc3 4096^2 rgba8", lambda: capi.lib.dxb200_compress_device(s, 1, 77, 0, 0.5, 1.0, d, st), w * h)

if what in ("dec", "all"):
    w = h = 4096
    for bc, dfmt, nm in ((98, 28, "bc7"), (71, 28, "bc1"), (80, 61, "bc4")):
        nb = F.compute_pitch(bc, w, h)[1]
        d_in = torch.randint(0, 256, (nb,), dtype=torch.uint8, device="cuda")
        if bc == 98:
            d_in.view(-1, 16)[:, 0] = 0x40       # valid mode-6 blocks
        d_out = torch.zeros(F.compute_pitch(dfmt, w, h)[1], dtype=torch.uint8, device="cuda")
        s = capi.images([capi.Image(w, h, bc, *F.compute_pitch(bc, w, h), d_in.data_ptr())])
        d = capi.images([capi.Image(w, h, dfmt, *F.compute_pitch(dfmt, w, h), d_out.data_ptr())])
        timed("decompress %s 4096^2" % nm, lambda: capi.lib.dxb200_decompress_device(s, 1, dfmt, d, st), w * h)

if what in ("rows", "all", "rowscubic", "rowslinear"):
    w = h = 8192
    d_in = dev(synth.c5_r8(w, h))
    d_f = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda")
    d_b = torch.zeros(w * h, dtype=torch.uint8, device="cuda")
    s = capi.images([capi.Image(w, h, 61, w, w * h, d_in.data_ptr())])
    f = capi.images([capi.Image(w, h, 41, w * 4, w * h * 4, d_f.data_ptr())])
    b = capi.images([capi.Image(w, h, 61, w, w * h, d_b.data_ptr())])
    timed("convert r8->r32f 8192^2", lambda: capi.lib.dxb200_convert_device(s, 1, 41, 0, 0.5, f, st), w * h)
    timed("convert r32f->r8 8192^2", lambda: capi.lib.dxb200_convert_device(f, 1, 61, 0, 0.5, b, st), w * h)
    # C4-like: 64 x (1024^2 RGBA8) box mip chains
    items, w, h = 64, 1024, 1024
    chain, arr, nl = mip_chains(28, w, h, items, dev(synth.c1_rgba8(w, h)))
    for fl, nm in ((F.TEX_FILTER_BOX, "box"), (F.TEX_FILTER_CUBIC, "cubic"), (F.TEX_FILTER_LINEAR, "linear")):
        if what.startswith("rows") and what != "rows" and what != "rows" + nm:
            continue
        timed("mips %s 64x1024^2 rgba8" % nm, lambda: capi.lib.dxb200_generate_mipmaps_device(arr, items, nl, fl, st), items * w * h * 4 // 3)
    if what in ("rows", "all"):
        del chain
        # k_mip_tile: BOX on its vector path takes both levels of a 3-level chain (the fused kernel needs 4 levels and the
        # tail kernel a source of at most 64x64) ...
        chain, arr, nl = mip_chains(28, w, h, items, dev(synth.c1_rgba8(w, h)), levels=3)
        timed("mips box 3 levels 64x1024^2", lambda: capi.lib.dxb200_generate_mipmaps_device(arr, items, nl, F.TEX_FILTER_BOX, st), items * w * h * 5 // 16)
        del chain
        # ... and LINEAR at sizes that are not multiples of 8 (no fused kernel) runs every level above 64x64
        w, h = 1023, 767
        chain, arr, nl = mip_chains(28, w, h, items, dev(synth.c1_rgba8(w, h)))
        timed("mips linear 64x1023x767 rgba8", lambda: capi.lib.dxb200_generate_mipmaps_device(arr, items, nl, F.TEX_FILTER_LINEAR, st), items * w * h * 4 // 3)
    del chain

if what in ("rowshalf", "all"):
    # the half-float store: k_convert_vec<2,10>, k_convert_vec<28,10> and the fused BOX kernel k_mip_box3<10>
    w = h = 4096
    d_h = torch.zeros(w * h * 8, dtype=torch.uint8, device="cuda")
    hh = capi.images([capi.Image(w, h, 10, w * 8, w * h * 8, d_h.data_ptr())])
    for sf, bpp, img in ((2, 16, synth.c2_rgba32f(w, h)), (28, 4, np.tile(synth.c1_rgba8(1024, 1024), (4, 4, 1)))):
        d_in = dev(img)
        s = capi.images([capi.Image(w, h, sf, w * bpp, w * h * bpp, d_in.data_ptr())])
        timed("convert %d->rgba16f 4096^2" % sf, lambda: capi.lib.dxb200_convert_device(s, 1, 10, 0, 0.5, hh, st), w * h)
        del d_in
    items, w, h = 16, 1024, 1024
    chain, arr, nl = mip_chains(10, w, h, items, dev(synth.c3_rgba16f(w, h)))
    timed("mips box 16x1024^2 rgba16f", lambda: capi.lib.dxb200_generate_mipmaps_device(arr, items, nl, F.TEX_FILTER_BOX, st), items * w * h * 4 // 3)
