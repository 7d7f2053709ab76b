#!/bin/bash
# run sweep_check (bit-exactness) and quick_bench (keys u32, default variant) with every sweep library;
# OSB_SKIP_PAIRS=0 times the pairs and u64 sorts as well.
for lib in tools/sweep/*.so; do
  echo "== $lib"
  OSB200_LIB=$PWD/$lib timeout 120 python tools/sweep_check.py 2>&1 | tail -1
  OSB200_LIB=$PWD/$lib OSB_SKIP_PAIRS=${OSB_SKIP_PAIRS-1} OSB_VARIANTS=2 timeout 180 python tools/quick_bench.py ${1:-30} 2>&1 | grep -E "variant=2|pairs|u64|Error|error|assert" | grep -v REFERENCE
done
