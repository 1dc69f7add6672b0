"""The device's BC7 blocks equal the pinned ones (tests/golden/golden_bc7_blocks_v1.npz; see test_cpu_bc7_pinned.py) on both
kernels: batches of equal-size RGBA32F images through k_compress_bc7_tma, and single images, the benchmark's crop and partial
blocks through k_compress_bc7.  BC7_UNORM only: to BC7_UNORM_SRGB the device converts with its own powf, which differs from the
host's in the last bit for a few inputs (one block of the cluster2 class), so those blocks are pinned on the host alone."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests.kernel_routes import launched

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_bc7_blocks as G  # noqa: E402

BC7_KERNELS = ("k_compress_bc7_tma", "k_compress_bc7")
CASES = [c for c in G.bc7_block_cases() if c[3] == G.BC7]


@pytest.fixture(scope="module")
def golden():
    return np.load(G.OUT)


@pytest.mark.gpu
@pytest.mark.parametrize("dst,flags", [(G.BC7, 0), (G.BC7, G.THREE), (G.BC7, G.QUICK)])
def test_tma_batch_equals_pinned(golden, dst, flags):
    """every 256 x 256 content class of (dst, flags) as one batch at a constant image stride on the device API"""
    torch = pytest.importorskip("torch")
    batch = [c for c in CASES if c[1] == (G.SIZE, G.SIZE) and c[3] == dst and c[4] == flags]
    assert len(batch) > 1
    w = h = G.SIZE
    n = len(batch)
    d_in = torch.from_numpy(np.stack([c[2]() for c in batch]).reshape(-1).view(np.uint8)).cuda()
    row, sl = F.compute_pitch(dst, w, h)
    d_out = torch.zeros(n * sl, dtype=torch.uint8, device="cuda")
    s = capi.images([capi.Image(w, h, 2, w * 16, w * h * 16, d_in.data_ptr() + i * w * h * 16) for i in range(n)])
    d = capi.images([capi.Image(w, h, dst, row, sl, d_out.data_ptr() + i * sl) for i in range(n)])
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    hr, ran = launched(BC7_KERNELS, capi.lib.dxb200_compress_device, s, n, dst, flags, 0.5, 1.0, d, st)
    assert hr == 0 and ran == {"k_compress_bc7_tma"}, (hr, ran)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy().reshape(n, sl)
    bad = [c[0] for i, c in enumerate(batch) if not np.array_equal(G.sha1(out[i]), golden[c[0] + "_out"])]
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_direct_kernel_equals_pinned(golden, case):
    """one image per call: the direct kernel, partial blocks included"""
    key, (w, h), make, dst, flags = case
    blocks, ran = launched(BC7_KERNELS, capi.compress, make(), w, h, 2, dst, flags)
    assert ran == {"k_compress_bc7"}, ran
    assert np.array_equal(G.sha1(blocks), golden[key + "_out"]), key
