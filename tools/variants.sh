#!/bin/bash
# Compile-time variants of the single-warp G = 1 kernel (register cap: B2INS_G1_MINBLOCKS CTAs per SM) and
# time 10^6 runs with each.  Build part runs anywhere with nvcc; timing part needs the GPU box.
#   bash tools/variants.sh build          -> tools/libb2ins_mb{3,4,5}.so
#   bash tools/variants.sh time > gpurun_out/variants_r02.jsonl
cd "$(dirname "$0")/../gnss_ins_sim_b200/csrc" || exit 1
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC"
if [ "$1" = "build" ]; then
  for mb in 3 4 5; do
    mkdir -p _obj/mb$mb
    for u in b2ins_api mc_plain_rf0 mc_plain_rf1 mc_spec_rf0 mc_spec_rf1; do
      nvcc $FLAGS -DB2INS_G1_MINBLOCKS=$mb -c -o _obj/mb$mb/$u.o $u.cu &
    done
    wait
    nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../tools/libb2ins_mb$mb.so _obj/mb$mb/*.o || exit 1
  done
  exit 0
fi
cd ../..
for mb in 3 4 5; do
  for rf in 1 0; do
    echo -n "{\"minblocks\": $mb, \"result\": "
    B2INS_MC_SHAPE=0 B2INS_LIB=$PWD/tools/libb2ins_mb$mb.so python tools/probe_mc.py 1000000 1 $rf 2 | tr -d '\n'
    echo "}"
  done
done
