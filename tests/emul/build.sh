#!/bin/sh
# tests/emul/build.sh — builds the host lock-step emulator (test infrastructure only).
set -e
cd "$(dirname "$0")"
mkdir -p _build
CXX=/usr/bin/g++; [ -x "$CXX" ] || CXX=g++
DEFS=""
[ -f ../../directxtex_b200/csrc/dxb_bc7.cuh ] && DEFS="-DDXB_EMUL_BC7"
FLAGS="-std=c++17 -O2 -msse2 -mfpmath=sse -mfma -ffp-contract=off -fopenmp -fPIC -shared -x c++"
$CXX $FLAGS $DEFS -I../../directxtex_b200/csrc emul.cpp -o _build/libdxb_emul.so
echo built tests/emul/_build/libdxb_emul.so
# the primitive probe's host build (tests/probe/probe.cu): the emulator's compiler and flags, so it runs the host branches the
# emulator runs
mkdir -p ../probe/_build
$CXX $FLAGS -I../../directxtex_b200/csrc -I../../include ../probe/probe.cu -o ../probe/_build/libdxb_probe_host.so
echo built tests/probe/_build/libdxb_probe_host.so
