"""directxtex_b200 — H100 (sm_90a) backend for the DirectXTex hot path.

The product is ``_lib/libdxtex_b200.so`` (CUDA kernels behind the C ABI declared in
``include/dxtex_b200.h``) plus the C++ ``namespace DirectX`` mirror in ``host/``.  This Python
package is only the thin ctypes binding that the tests and ``bench.py`` use to reach the C ABI;
it contains no codec logic and no fallback: if the shared library is missing, importing
``directxtex_b200.capi`` raises.
"""
from .formats import *          # noqa: F401,F403


def __getattr__(name):
    # `capi` loads the shared library at import time; keep it lazy so that `directxtex_b200.build` can be imported
    # (and run) when the library does not exist yet or is stale
    if name == "capi":
        import importlib
        return importlib.import_module(".capi", __name__)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
