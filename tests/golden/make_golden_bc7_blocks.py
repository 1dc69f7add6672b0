#!/usr/bin/env python
"""Generates tests/golden/golden_bc7_blocks_v1.npz: the SHA-1 of the BC7 blocks the host emulator (tests/emul) emits for a fixed
set of inputs, so that a change to the encoder that must keep its blocks bit for bit is checked on the CPU before it runs anywhere.

Cases (bc7_block_cases):
    every LDR content class of directxtex_b200.synth at 256 x 256 to BC7_UNORM with flags 0, TEX_COMPRESS_BC7_USE_3SUBSETS and
    TEX_COMPRESS_BC7_QUICK, and to BC7_UNORM_SRGB with flags 0;
    the centre 1024 x 1024 crop of the 4096 x 4096 C2 image (the benchmark's input) to BC7_UNORM;
    a 250 x 130 photo with alpha (partial blocks on both edges) to BC7_UNORM.
Stored per case: <key>_in = SHA-1 of the RGBA32F input bytes (so that a change of the generators is told apart from a change of
the encoder), <key>_out = SHA-1 of the emitted blocks.

    python tests/golden/make_golden_bc7_blocks.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from directxtex_b200 import formats as F, synth  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_bc7_blocks_v1.npz")
SIZE, SEED = 256, 5
BC7, BC7_SRGB = F.DXGI_FORMAT["BC7_UNORM"], F.DXGI_FORMAT["BC7_UNORM_SRGB"]
THREE, QUICK = F.TEX_COMPRESS_BC7_USE_3SUBSETS, F.TEX_COMPRESS_BC7_QUICK


def bc7_block_cases():
    """[(key, (w, h), make_image, dst_format, flags)]; make_image() returns the RGBA32F source"""
    cases = []
    for kind in synth.LDR_CLASSES:
        make = (lambda k: lambda: synth.content_ldr(k, SIZE, SIZE, SEED))(kind)
        for dst, flags in ((BC7, 0), (BC7, THREE), (BC7, QUICK), (BC7_SRGB, 0)):
            cases.append(("%s_%d_%x" % (kind, dst, flags), (SIZE, SIZE), make, dst, flags))
    cases.append(("c2crop1024_98_0", (1024, 1024), c2_crop, BC7, 0))
    cases.append(("partial250x130_98_0", (250, 130), lambda: synth.photo_rgba32f(250, 130, SEED, alpha=True), BC7, 0))
    return cases


def c2_crop(side=1024):
    img = synth.c2_rgba32f(4096, 4096)
    y0 = (4096 - side) // 2
    return np.ascontiguousarray(img[y0:y0 + side, y0:y0 + side])


def sha1(a):
    return np.frombuffer(hashlib.sha1(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    from tests import oracle_lib
    emul = oracle_lib.load_emul()
    data = {}
    for key, (w, h), make, dst, flags in bc7_block_cases():
        img = make()
        hr, blocks = emul.compress(img, w, h, 2, dst, flags)
        assert hr == 0, key
        data[key + "_in"], data[key + "_out"] = sha1(img), sha1(blocks)
        print(key, flush=True)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
