"""Measures texconv's "set alpha mode" test of a compressed output, IsAlphaAllOpaque (development tool; bench.py is the project
benchmark).

64 x 1024^2 BC3 items of synth.content_ldr("cutout") -> full chains -> BC7 and -> BC1 (the chains of DESIGN.md section 4), as they are
(the answer is found in the first blocks) and with their alpha made opaque (every block is decoded), timed three ways:
  * the reference's ScratchImage::IsAlphaAllOpaque of the output on the host (tests/cpp/alpha_opaque_probe.cpp linked with the
    reference build, when oracle/_ref/libdxtex_ref.so exists), single thread;
  * dxb200_mipmaps_compress_from_ex against dxb200_mipmaps_compress_from on pinned buffers, alternating run by run, medians of
    --reps runs; the blocks must be identical;
  * dxb200_is_alpha_all_opaque of the downloaded chains (pinned).
Host clock around calls that end synchronised.

Usage: python tools/alpha_opaque_bench.py [--reps N] [--items N] [--size N] [--out FILE]
Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from directxtex_b200 import capi, formats as F  # noqa: E402
from tools.chain_steps_bench import card, cutout_rgba8, pinned, stats  # noqa: E402


def reference_probe():
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libdxtex_ref.so")):
        return None
    from tests import alpha_opaque_lib as A
    return A.Probe(tempfile.mkdtemp(prefix="alpha_opaque_bench"), reference=True)


def cutout(w, seed, opaque):
    img = cutout_rgba8(w, w, seed)
    if opaque:
        img[..., 3] = 255
    return img


def run(items, w, df, reps, probe, opaque_alpha):
    bc, rgba = 77, 28
    levels = F.count_mips(w, w)
    brow, bsl = F.compute_pitch(bc, w, w)
    olayout, ototal = capi.texture_layout(df, w, w, 1, levels)
    uniq = [capi.compress(cutout(w, s, opaque_alpha), w, w, rgba, bc) for s in range(8)]
    base, _ = pinned(items * bsl)
    for i in range(items):
        base[i * bsl:(i + 1) * bsl] = uniq[i % len(uniq)]
    out_from, _ = pinned(items * ototal)
    out_ex, _ = pinned(items * ototal)
    addr = lambda a: a.ctypes.data
    bases = capi.images([capi.Image(w, w, bc, brow, bsl, addr(base) + i * bsl) for i in range(items)])
    outs = lambda buf: capi.images([capi.Image(lw, lh, df, r, sp, addr(buf) + i * ototal + off) for i in range(items) for (off, lw, lh, r, sp) in olayout])
    d_from, d_ex = outs(out_from), outs(out_ex)
    source = capi.chain_source()
    opaque = C.c_int32(-1)

    def plain():
        assert capi.lib.dxb200_mipmaps_compress_from(bases, items, C.byref(source), levels, 0, None, df, 0, 0.5, 1.0, d_from) == 0

    def with_answer():
        assert capi.lib.dxb200_mipmaps_compress_from_ex(bases, items, C.byref(source), levels, 0, None, df, 0, 0.5, 1.0, d_ex, C.byref(opaque)) == 0

    def scan():
        a = C.c_int32(-1)
        assert capi.lib.dxb200_is_alpha_all_opaque(d_ex, items * levels, C.byref(a)) == 0
        return a.value

    plain(); with_answer(); scan()                              # warm-up of every shape
    t_plain, t_ex, t_scan = [], [], []
    for _ in range(reps):
        for fn, ts in ((plain, t_plain), (with_answer, t_ex), (scan, t_scan)):
            t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    assert np.array_equal(out_from, out_ex), "_from_ex's blocks differ from _from's"
    assert scan() == opaque.value
    out = {"items": items, "size": w, "target": df, "alpha": "opaque" if opaque_alpha else "cutout", "from": stats(t_plain), "from_ex": stats(t_ex), "host_scan": stats(t_scan),
           "identical": True, "opaque": opaque.value}
    if probe is not None:
        t0 = time.perf_counter()
        want = probe.opaque(df, w, w, out_ex, items=items, levels=levels)
        out["reference_s"] = time.perf_counter() - t0
        assert want == (opaque.value == 1), "the answer differs from the reference's"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--items", type=int, default=64)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    assert capi.lib.dxb200_init(0) == 0
    probe = reference_probe()
    out = {"card": card(), "bc3_to": [run(a.items, a.size, df, a.reps, probe, op) for op in (False, True) for df in (98, 71)]}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
