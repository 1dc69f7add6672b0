"""TEST INFRASTRUCTURE: builds the encoder test harnesses (tests/bc7_ranking/, tests/bc67_blocks/) into a temporary directory.

host_lib: g++ with the host emulator's flags (tests/emul/build.sh), so it runs the host branches the emulator runs.
device_lib: nvcc for sm_90a with the library's own flags (directxtex_b200/build.py), so it runs the device branches the kernels run."""
import ctypes as C
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "directxtex_b200", "csrc")
HERE = os.path.join(ROOT, "tests", "bc7_ranking")
HOST_FLAGS = ["-std=c++17", "-O2", "-msse2", "-mfpmath=sse", "-mfma", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared", "-x", "c++"]


def host_lib(src, out_dir, src_dir=HERE):
    """src (a file of src_dir, by default tests/bc7_ranking/) built with the emulator's flags into out_dir"""
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    out = os.path.join(str(out_dir), os.path.splitext(src)[0] + "_host.so")
    r = subprocess.run([cxx] + HOST_FLAGS + ["-I", CSRC, "-I", os.path.join(ROOT, "include"), os.path.join(src_dir, src), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return C.CDLL(out)


def device_lib(src, out_dir, src_dir=HERE):
    from directxtex_b200 import build as b
    out = os.path.join(str(out_dir), os.path.splitext(src)[0] + "_device.so")
    r = subprocess.run([b._nvcc()] + b._flags() + ["-shared", "-cudart", "static", os.path.join(src_dir, src), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return C.CDLL(out)


def run_collective(L, arg, count):
    """(mismatch count, (input, got, want) of one mismatch)"""
    L.coll_run.argtypes = [C.c_uint32, C.c_uint64, C.c_void_p]
    L.coll_run.restype = C.c_int
    out = (C.c_ulonglong * 4)()
    rc = L.coll_run(arg, count, C.cast(out, C.c_void_p))
    assert rc == 0, "coll_run(%d) failed: %d" % (arg, rc)
    return int(out[0]), (int(out[1]), int(out[2]), int(out[3]))


# (arg, count): 2^15 warps of 32 lanes for the collectives, 2^24 words for the dot product
COLLECTIVE_DOMAINS = [(0, 32 << 15), (1, 32 << 15), (2, 32 << 15), (3, 1 << 24)]
COLLECTIVE_NAMES = {0: "half_ballot4_u64", 1: "nth_set_bit_u64", 2: "warp_max_u32", 3: "dp4a_s8s8"}
