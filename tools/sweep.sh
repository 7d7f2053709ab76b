#!/bin/bash
# Build the library with alternative compile-time parameters into tools/sweep/ (development sweeps; see tools/sweep_run.sh).
# each config: "WARPS K MINB LOOK [PLOOK ULOOK]"   (PLOOK/ULOOK: lookback windows of the pairs and u64 kernels, default 8 and
# 32).  WARPS K MINB set the u32 keys geometry; the pairs and u64 geometries take EXTRA_DEFS (-DOSB_PAIRS_WIDE_WARPS=..
# -DOSB_PAIRS_WIDE_K=.. -DOSB_PAIRS_WIDE_MINB=.., -DOSB_U64_WARPS=.. -DOSB_U64_K=.. -DOSB_U64_MINB=..), which apply to every
# config of a run.  A phase-probe build for tools/phase_probe.py: EXTRA_DEFS=-DOSB_PHASE_PROBE=1.
set -e
cd "$(dirname "$0")/../gpusorting_b200/csrc"
mkdir -p ../../tools/sweep
rm -f ../../tools/sweep/*.so
CONFIGS=${CONFIGS:-"16 32 2 16;16 32 2 32"}
IFS=';' read -ra CFGS <<< "$CONFIGS"
for cfg in "${CFGS[@]}"; do
  set -- $cfg
  plook=${5:-8}
  ulook=${6:-32}
  tag=W$1_K$2_B$3_L$4_P${plook}_U${ulook}
  nvcc -std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -Xcompiler -fvisibility=hidden \
       -DOSB200_BUILDING -DOSB_WIDE_WARPS=$1 -DOSB_WIDE_K=$2 -DOSB_WIDE_MINB=$3 -DOSB_LOOK=$4 \
       -DOSB_PAIRS_LOOK=$plook -DOSB_U64_LOOK=$ulook $EXTRA_DEFS -Xptxas -v \
       -shared -o ../../tools/sweep/libosb_$tag.so osb_kernels.cu osb_host.cu osb_sharded.cu -lnccl 2> ../../tools/sweep/build_$tag.log &
done
wait
ls -la ../../tools/sweep/*.so
