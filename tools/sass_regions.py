#!/usr/bin/env python
"""Static SASS instruction count of one kernel, per encoder stage (runs on the CPU, needs nvdisasm / cuobjdump).

    python tools/sass_regions.py directxtex_b200/_lib/dxb_k_bc7.o k_compress_bc7_tmaILb0ELb1 [--pipes]

The object (or cubin) must be built with -lineinfo (directxtex_b200/build.py does), and --src must hold the sources
it was built from (line numbers).  `nvdisasm -gi` annotates each instruction with its source line followed by the
chain of call sites it was inlined through.  A region is a span of source lines (REGIONS: file, first line
containing `start`, up to the line before the first line containing `end` after it, or to the end of the brace block
opened at `start` when `end` is None).  An instruction counts under the innermost line of its chain that lies in a
region, so an inlined helper that belongs to no region (a fp32-pair wrapper, dxb_rne, dxb_convert_pixel, ...) is
counted under the stage that calls it.  An instruction without line information takes the region of the one before
it.  Instruction scheduling mixes neighbouring lines, so the split is good to a few instructions per region.

--pipes splits each region's count by the execution pipe the opcode issues to (PIPES).  An H100 SM sub-partition has 32
FP32 lanes but 16 lanes for each integer half: a warp instruction on the ALU pipe (logic, shifts, compares, selects,
min/max, integer adds, byte permutes) or on the FMA-heavy integer pipe (IMAD, IDP, the tensor-core MMAs) occupies its
pipe for two cycles, so a region whose ALU share is well above 50 % is bound by that pipe rather than by the issue slot.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "directxtex_b200", "csrc")

# (region, file, start anchor, end anchor or None = end of the brace block opened at the start line)
REGIONS = [
    ("tma loop + convert", "dxb_k_bc7.cu", "k_compress_bc7_tma(const", None),
    ("direct loop + convert", "dxb_k_bc7.cu", "k_compress_bc7(const", None),
    ("s1 moments (mma)", "dxb_bc7.cuh", "DXB_DEV void dxb_bc7_build_moments", None),
    ("s1 h1 part A (axes)", "dxb_bc7.cuh", "DXB_DEV void dxb_bc7_subset_axes", None),
    ("s1 h1 part A (axes)", "dxb_bc7.cuh", "DXB_DEV void dxb_bc7_shape_axes", None),
    ("s1 h1 part B (quantisation)", "dxb_bc7.cuh", "DXB_DEV float dxb_bc7_shape_qerr", None),
    ("s1 h1 part B (quantisation)", "dxb_bc7.cuh", "DXB_DEV float dxb_bc7_shape_h1", None),
    ("s1 select", "dxb_bc7.cuh", "// ---- stage 1: moment table", "// ---- stage 2:"),
    ("s2 tasks + rotation", "dxb_bc7.cuh", "// ---- stage 2:", "// ---- stage 3:"),
    ("s2 rotation", "dxb_bc7.cuh", "DXB_DEV float dxb_bc7_rotation_estimate1", "// -----"),
    ("s2 moments/PCA/extents", "dxb_bc7.cuh", "DXB_DEV dxb_bc7_res dxb_bc7_eval", "// ---- evaluation rounds"),
    ("s2 quantisation", "dxb_bc7.cuh", "DXB_DEV dxb_bc7_qconst dxb_bc7_make_qconst", "struct dxb_bc7_modecfg"),
    ("s2 quantisation", "dxb_bc7.cuh", "// ---- evaluation rounds", "// p-bit choice"),
    ("s2 rounds (pixel loops, refit)", "dxb_bc7.cuh", "// p-bit choice", "// natural channel order"),
    ("s3 winner (+ 3-subset pass)", "dxb_bc7.cuh", "// ---- stage 3:", "// ---- stage 4:"),
    ("s4 nearest + packer", "dxb_bc7.cuh", "// ---- stage 4:", "#if !DXB_ON_DEVICE\n// emulator entry"),
    ("s4 nearest + packer", "dxb_bc7.cuh", "// stage 4 helpers", "// The encoder proper"),
]


def _line_of(text, anchor, start=0):
    i = text.find(anchor, start)
    if i < 0:
        raise SystemExit("anchor not found: %r" % anchor)
    return text.count("\n", 0, i) + 1, i


def region_spans(src_dir):
    """{basename: [(first, last, region)]}"""
    spans = {}
    for name, fname, start, end in REGIONS:
        text = open(os.path.join(src_dir, fname)).read()
        first, pos = _line_of(text, start)
        if end is None:
            depth, i = 0, text.index("{", pos)
            while True:
                depth += {"{": 1, "}": -1}.get(text[i], 0)
                if depth == 0:
                    break
                i += 1
            last = text.count("\n", 0, i) + 1
        else:
            last = _line_of(text, end, pos + len(start))[0] - 1
        spans.setdefault(fname, []).append((first, last, name))
    return spans


def disassemble(path, kernel):
    with tempfile.TemporaryDirectory() as tmp:
        cubin = path
        if not path.endswith(".cubin"):
            subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(path)], cwd=tmp, check=True, capture_output=True)
            cubins = [f for f in os.listdir(tmp) if f.endswith(".cubin")]
            if len(cubins) != 1:
                raise SystemExit("expected one cubin in %s, found %s" % (path, cubins))
            cubin = os.path.join(tmp, cubins[0])
        out = subprocess.run(["nvdisasm", "-gi", cubin], check=True, capture_output=True, text=True).stdout
    sections = re.split(r"^//-+ (\.text\.\S+) -+$", out, flags=re.M)
    hits = [(sections[k], sections[k + 1]) for k in range(1, len(sections) - 1, 2) if kernel in sections[k]]
    if len(hits) != 1:
        raise SystemExit("kernel %r matches %d functions: %s" % (kernel, len(hits), [h[0] for h in hits]))
    return hits[0]


LINE = re.compile(r'//## File "([^"]+)", line (\d+)')
INSN = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+(.*?);?\s*$")
OPCODE = re.compile(r"^(?:@!?U?P[T0-9]+\s+)?([A-Z0-9_]+)")

# opcode (without modifiers) -> pipe class on sm_90; the uniform datapath (U*) and moves fall under "other"
PIPES = {
    "FP32": "FFMA FADD FMUL FFMA32I FADD32I FMUL32I FSWZADD HFMA2 HADD2 HMUL2",
    "FMA-int": "IMAD IMAD32I IDP IMUL HMMA IMMA",
    "ALU": "LOP3 LOP SHF SHL SHR ISETP SEL FSEL FSETP FSET FMNMX IADD3 IADD VIADD PRMT VABSDIFF4 VABSDIFF VIMNMX VIMNMX3 "
           "VIADDMNMX IMNMX LEA ISCADD IABS PLOP3 P2R R2P I2FP",
    "XU": "MUFU F2I I2F F2F FRND FCHK POPC FLO BREV",
    "MIO": "LDS STS LDG STG LD ST LDC LDL STL SHFL REDUX ATOMS ATOMG ATOM RED LDSM LDGSTS UTMALDG SYNCS MATCH",
    "control": "BRA BRX BSSY BSYNC EXIT CALL RET BAR WARPSYNC NOP YIELD BPT DEPBAR ENDCOLLECTIVE ELECT FENCE MEMBAR",
}
PIPE_OF = {op: pipe for pipe, ops in PIPES.items() for op in ops.split()}
PIPE_ORDER = list(PIPES) + ["other"]


def pipe_of(insn):
    m = OPCODE.match(insn)
    return PIPE_OF.get(m.group(1), "other") if m else "other"


def count(sass, spans):
    def region(f, ln):
        for a, b, name in spans.get(os.path.basename(f), ()):
            if a <= ln <= b:
                return name
        return None
    counts, pipes, chain, fresh, last = {}, {}, [], False, "(unattributed)"
    for line in sass.splitlines():
        m = LINE.search(line)
        if m:
            if not fresh:
                chain, fresh = [], True
            chain.append((m.group(1), int(m.group(2))))
            continue
        i = INSN.match(line)
        if not i:
            continue
        fresh = False
        r = next((x for x in (region(f, ln) for f, ln in chain) if x), None) or last
        last = r
        counts[r] = counts.get(r, 0) + 1
        per = pipes.setdefault(r, {})
        p = pipe_of(i.group(1))
        per[p] = per.get(p, 0) + 1
    return counts, pipes


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("binary", help="object file or cubin built with -lineinfo")
    ap.add_argument("kernel", help="substring of the kernel's mangled name, e.g. k_compress_bc7_tmaILb0ELb1")
    ap.add_argument("--src", default=CSRC, help="directory of the sources the binary was built from")
    ap.add_argument("--pipes", action="store_true", help="split each region's count by execution pipe (PIPES)")
    args = ap.parse_args()
    name, sass = disassemble(args.binary, args.kernel)
    counts, pipes = count(sass, region_spans(args.src))
    order = [r[0] for r in REGIONS] + ["(unattributed)"]
    print(name[len(".text."):])
    if args.pipes:
        print("%-34s %6s" % ("region", "SASS") + "".join("%9s" % p for p in PIPE_ORDER) + "   ALU share")
    total = {}
    for r in sorted(counts, key=order.index) + ["total"]:
        per = pipes.get(r, total)
        n = counts.get(r, sum(counts.values()))
        line = "%-34s %6d" % (r, n)
        if args.pipes:
            line += "".join("%9d" % per.get(p, 0) for p in PIPE_ORDER) + "   %5.0f %%" % (100.0 * per.get("ALU", 0) / max(n, 1))
            if r != "total":
                for p, v in per.items():
                    total[p] = total.get(p, 0) + v
        print(line)


if __name__ == "__main__":
    sys.exit(main())
