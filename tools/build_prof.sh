#!/bin/bash
# The library with phase clocks (-DB2INS_PHASE_CLOCKS) in one translation unit, for spec2_phase.py and
# phase_probe.py.  Runs anywhere with nvcc.
#   bash tools/build_prof.sh [OUT]          (default tools/libb2ins_prof.so)
set -e
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
OUT="$(realpath -m "${1:-$ROOT/tools/libb2ins_prof.so}")"
cd "$ROOT/gnss_ins_sim_b200/csrc"
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC \
  -DB2INS_PHASE_CLOCKS -DB2INS_SINGLE_TU -shared -o "$OUT" b2ins_api.cu
