"""TEST INFRASTRUCTURE: ctypes access to the primitive probe (tests/probe/probe.cu) and the input domains of its checks.

The probe is built twice: libdxb_probe.so by nvcc for sm_90a with the library's flags (the device branches of the shared headers)
and libdxb_probe_host.so by g++ with the emulator's flags (the host branches).  A check maps a 64-bit index to one input; a run
evaluates the indices begin + j * step, j < count, and returns the mismatch count and up to 16 (input, got, want) records."""
import ctypes as C
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVICE_SO = os.path.join(ROOT, "tests", "probe", "_build", "libdxb_probe.so")
HOST_SO = os.path.join(ROOT, "tests", "probe", "_build", "libdxb_probe_host.so")

# (bits, p-bit) of the eight BC7 endpoint field layouts, in the probe's order (ref_layout_bits / ref_layout_p)
LAYOUT_HAS_P = (1, 1, 0, 1, 0, 0, 0, 1)
# per BC7 mode: colour field bits, alpha field bits (0: none), p-bits present (ref_mode_cb / ref_mode_ab / ref_mode_p)
MODE_CB = (4, 6, 5, 7, 5, 7, 7, 5)
MODE_AB = (0, 0, 0, 0, 6, 8, 7, 5)
MODE_P = (1, 1, 0, 1, 0, 0, 1, 1)

# float-pattern domains: index i < npos is the bit pattern i, index npos + k the pattern 0x80000000 + k
FLOAT_NPOS = {"f2u_trunc_small": 0x4B000000, "f2i_rn_small": 0x4A800000, "f2i": 0x4F000000, "f2u": 0x4F800000,
              "f2i_rn": 0x4F000000, "round_even": 1 << 32, "float_to_half": 1 << 32, "quant2f": 0x437F0001}


def domains():
    """[(check, arg, begin, count)]: the full input domain of every check whose mismatches must be zero (the preconditions the
    callers keep; see the test modules' docstrings)"""
    d = [("i2f_small", 0, 0, (1 << 23) - 1),                        # every |n| < 2^22
         ("byte_to_float", 0, 0, 4 * 256 * 1024),                   # byte value x position x (0x00 / 0xFF / 1022 random) others
         ("f2u_trunc_small", 0, 0, 0x4B000001),                     # [+0, 2^23) and -0
         ("f2i_rn_small", 0, 0, 2 * 0x4A800000),                    # (-2^22, 2^22)
         ("f2i", 0, 0, 0x4F000000 + 0x4F000001),                    # [-2^31, 2^31)
         ("f2u", 0, 0, 0x4F800000 + 0x3F800000),                    # (-1, 2^32)
         ("f2i_rn", 0, 0, 0x4F000000 + 0x4F000001),
         ("round_even", 0, 0, 1 << 32),                             # every float
         ("half_to_float", 0, 0, 1 << 16),
         ("float_to_half", 0, 0, 1 << 32),                          # every non-NaN float
         ("unorm8", 0, 0, 1 << 34),                                 # every float at each of the 4 channel positions
         ("rcp_int", 0, 1, (1 << 24) - 1),                          # 1 .. 2^24 - 1 (the encoder passes integers below 2^18)
         ("bc7_weights", 0, 0, 28),
         ("pal4", 0, 0, 3 << 29),
         ("put_bits4", 0, 0, 1 << 23),
         ("udiv", 0, 0, 65535 * 64), ("udiv", 1, 0, 1 << 26)]
    for lay, has_p in enumerate(LAYOUT_HAS_P):
        for p in ((0, 1) if has_p else (0,)):                       # p = 1 results are only selected for layouts with a p-bit
            d.append(("quant2f", lay | (p << 3), 0, 0x437F0002))    # every float in [+0, 255] and -0
    for v in range(5):                                              # <16> with 2/3/4 index bits, <8> with 2/3
        d.append(("nearest1", v, 0, 1 << 26))
        d.append(("nearest4", v, 0, 1 << 26))
    for m in range(8):
        for p in ((0, 1) if MODE_P[m] else (0,)):
            d.append(("deq4", m | (p << 3), 0, 1 << (3 * MODE_CB[m] + MODE_AB[m])))
    for v in range(8):                                              # dp4a u8s8 / u8u8, dp2a lo / hi, prmt, vabsdiff4, min3, max3
        d.append(("simd", v, 0, 1 << 26))
    for v in range(10):                                             # dxb_warp.cuh collectives: 2^15 warps of 32 lanes each
        d.append(("warp", v, 0, 32 << 15))
    return d


# Outside the preconditions: device and host may part ways here, the counts are recorded, not required to be zero.
RECORDED = [("f2u_trunc_small_neg", 0, 0, 0x3F7FFFFF),               # (-1, -0): every caller clamps to >= 0 first
            ("f2i_out_of_range", 0, 0, 0x31000000 + 0x30FFFFFF)]     # |f| >= 2^31, infinities, NaN: saturation vs 0x80000000


class Probe:
    def __init__(self, path):
        L = self.L = C.CDLL(path)
        L.probe_name.argtypes = [C.c_int]
        L.probe_name.restype = C.c_char_p
        L.probe_run.argtypes = [C.c_int, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p]
        L.probe_run.restype = C.c_int
        self.ids = {}
        i = 0
        while L.probe_name(i):
            self.ids[L.probe_name(i).decode()] = i
            i += 1
        self.on_device = bool(L.probe_on_device())

    def run(self, name, arg, begin, count, step=1):
        """(mismatch count, [(input, got, want)] of up to 16 mismatches)"""
        out = (C.c_ulonglong * 49)()
        rc = self.L.probe_run(self.ids[name], arg, begin, count, step, C.cast(out, C.c_void_p))
        if rc != 0:
            raise RuntimeError("probe_run(%s, %d) failed: %d" % (name, arg, rc))
        n = int(out[0])
        return n, [(int(out[1 + 3 * r]), int(out[2 + 3 * r]), int(out[3 + 3 * r])) for r in range(min(n, 16))]


def describe(name, arg, n, recs):
    lines = ["%s arg=%#x: %d mismatches; first (input, got, want):" % (name, arg, n)]
    lines += ["  in=%#018x got=%#010x want=%#010x" % r for r in recs]
    return "\n".join(lines)
