"""Which kernels the library compiled and which ones a call launched.

kernel_entries() reads the kernel entry points of libdxtex_b200.so from its device code with the toolkit's cuobjdump, so that
the route tests compare their lists with what the library contains rather than with the CUDA sources.  launched() runs a call
and reports which of the named kernels it launched (dxb200_kernel_launch_count)."""
import functools
import os
import re
import subprocess

from directxtex_b200 import build, capi


def _arg(text):
    """one demangled template argument: "(unsigned int)84" -> 84, "(bool)1" -> True"""
    m = re.fullmatch(r"\((unsigned int|bool)\)(\d+)", text)
    assert m, text
    return bool(int(m.group(2))) if m.group(1) == "bool" else int(m.group(2))


@functools.lru_cache(maxsize=None)
def kernel_entries(lib=capi.LIB_PATH):
    """{kernel name: set of template-argument tuples} of every kernel entry point (STO_ENTRY symbol) of `lib`; a kernel that is
    not a template has the single tuple ()"""
    bindir = os.path.dirname(build._nvcc())
    syms = subprocess.run([os.path.join(bindir, "cuobjdump"), "-symbols", lib], capture_output=True, text=True, check=True).stdout
    mangled = [line.split()[-1] for line in syms.splitlines() if "STO_ENTRY" in line]
    assert mangled, lib
    names = subprocess.run([os.path.join(bindir, "cu++filt")], input="\n".join(mangled) + "\n", capture_output=True, text=True,
                           check=True).stdout.splitlines()
    assert len(names) == len(mangled)
    out = {}
    for name in names:
        m = re.fullmatch(r"(?:void )?(\w+)(?:<(.*)>)?\(.*\)", name.strip())
        assert m, name
        out.setdefault(m.group(1), set()).add(tuple(_arg(a) for a in m.group(2).split(", ")) if m.group(2) else ())
    return out


def launched(kernels, fn, *args, **kwargs):
    """(fn(*args, **kwargs), the set of names in `kernels` whose launch count it moved)"""
    before = {k: capi.kernel_launch_count(k) for k in kernels}
    out = fn(*args, **kwargs)
    return out, {k for k in kernels if capi.kernel_launch_count(k) != before[k]}
