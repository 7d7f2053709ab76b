"""Development probe: per-phase wall clocks of the wide DigitBinningPass (library built with -DOSB_PHASE_PROBE=1, e.g.
EXTRA_DEFS=-DOSB_PHASE_PROBE=1 tools/sweep.sh; OSB200_LIB names the library)."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402

lib = ctypes.CDLL(os.environ["OSB200_LIB"])
n = 1 << int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 30
src = torch.empty(n, dtype=torch.int32, device="cuda")
g.init_random(src, 0, 10)
work = src.clone()
s = g.OneSweepSorter(n, 4, 0)
s.sort_keys(work)
torch.cuda.synchronize()
out = (ctypes.c_ulonglong * 11)()
lib.osb200_debug_phases(out, 1)
work.copy_(src)
s.sort_keys(work)
torch.cuda.synchronize()
lib.osb200_debug_phases(out, 0)
# a persistent CTA runs many tiles: every figure is per tile.  "tile start" holds each CTA's start-up (plan, histogram clear)
# once; "wait for keys" is how long the tile's keys, loaded during the previous tile, still take to land
names = ["tile start", "wait for keys", "count", "reduce/scan/bases", "rank + next loads", "lookback", "scatter", None,
         "barrier after lookback"]
tiles = out[7]
tot = sum(out[i] for i in range(9) if i != 7)
print(f"tiles {tiles}; mean clocks per tile: total {tot / tiles:.0f}")
for i, nm in enumerate(names):
    if nm is None:
        continue
    print(f"  {nm:22s} {out[i] / tiles:9.0f} clk  {100.0 * out[i] / tot:5.1f}%")
print(f"lookback windows per tile (digit 0): {out[9] / tiles:.2f}; stalled polls per tile: {out[10] / tiles:.2f}")
