"""The device branches of the shared arithmetic headers against exact references, on their whole input domains (tests/probe/probe.cu,
built for sm_90a with the library's flags).  tests/test_cpu_primitives.py checks the host branches against the same references; the
two together give device == host emulator on these domains, which is what lets the CPU quality measurements describe the GPU.

Why the kernels' arguments lie inside each domain (call sites in directxtex_b200/csrc):
  i2f_small, byte_to_float   pixel loads of 8/10/16-bit channels (dxb_pixel.cuh): integers below 2^16, bytes of a loaded word.
  f2u_trunc_small            dxb_unorm8_trunc / dxb_unorm8_scalar / the 10:10:10:2 store: the argument is clamped to [0, 1] (NaN
                             to 0) and scaled by 255 / 1023 / 3 first, so it lies in [+0, 1023].  In (-1, 0) the device returns
                             mantissa bits of 2^23 - |f| where the host truncates to 0: recorded only, no caller gets there.
  f2i_rn_small               dxb_bc7_eval: dequantised endpoints, integers in [0, 255]; the 8/16-bit UNORM / SNORM stores
                             (dxb_pixel.cuh): clamp(v, 0 or -1, 1) (dxb_clamp maps NaN to the lower bound) times 127, 255, 32767
                             or 65535, so |argument| <= 65535.
  f2i, f2u, f2i_rn, round_even   C-cast / RNE semantics inside int32 / uint32.  Outside (and NaN) the device saturates (NaN to 0)
                             and x86 gives 0x80000000: recorded only; the callers clamp before converting.
  half_to_float, float_to_half   every half, every non-NaN float (a NaN stays a NaN; its payload is not compared).
  unorm8                     dxb_pack_unorm8x4 (device: FADD.RZ onto 2^23 and PRMT) == dxb_unorm8_trunc == floor(clamp(v + 0.5/255,
                             0, 1) * 255) for every float in every channel position.
  rcp_int                    integers only: dxb_bc7_subset_axes passes |a|^2 <= 4 * 128^2 (s8 axis components) and
                             dxb_bc7_shape_h1 a projection extent <= 2 * 4 * 255 * 128 < 2^18.  The sweep covers every integer
                             1 .. 2^24 - 1, so a caller with a larger integer operand stays covered.
  quant2f                    endpoints are clamped to [0, 255] before quantisation (dxb_bc7_eval); -0 included.
  bc7_weights, pal4, nearest, deq4, put_bits4   the whole field / weight / byte domains of BC7.
  simd                       random words with extreme bytes (0, 1, 127, 128, 254, 255) and accumulators INT_MIN / INT_MAX / 0 / -1.
  warp                       dxb_warp.cuh collectives (lane exchange, broadcast, warp and half-warp min / OR, half-warp gather) on
                             2^15 warps of random lane values, a quarter of them with ties, halves differing.
  udiv                       every divisor below 2^16 (tiles per row / image) and random ones below 2^31, numerators over the whole
                             32-bit range (the kernel passes tile indices below 2^31)."""
import os
import time

import pytest

from tests import probe_lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def probe():
    if not os.path.exists(probe_lib.DEVICE_SO):
        pytest.fail("tests/probe/_build/libdxb_probe.so missing: run __graft_entry__.build()")
    p = probe_lib.Probe(probe_lib.DEVICE_SO)
    assert p.on_device
    return p


@pytest.mark.parametrize("name,arg,begin,count", probe_lib.domains(), ids=lambda v: str(v))
def test_device_primitive_equals_reference(probe, name, arg, begin, count):
    t = time.perf_counter()
    n, recs = probe.run(name, arg, begin, count)
    print("%s arg=%#x: %d inputs, %.3f s" % (name, arg, count, time.perf_counter() - t))
    assert n == 0, probe_lib.describe(name, arg, n, recs)


def test_device_outside_preconditions(probe):
    """Where device and host part ways outside the preconditions (dxb_f2u_trunc_small on (-1, 0), float -> int32 outside int32):
    recorded (printed), not required to match."""
    for (name, arg, begin, count) in probe_lib.RECORDED:
        n, recs = probe.run(name, arg, begin, count)
        print(probe_lib.describe(name, arg, n, recs[:4]) + "  (of %d inputs)" % count)
