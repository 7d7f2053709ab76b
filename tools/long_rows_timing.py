"""Long-row sort (sort_long_rows) against the routes a caller has without it: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  long       gpusorting_b200.sort_long_rows(x): values and int32 positions within the row
  torch      torch.sort(x, dim=-1, stable=True)
  composite  (16- and 32-bit keys) an int64 key per element, the row id above the key's radix image, argsorted as "u64" on
             the stream's cached (8, 4) sorter, then the values gathered and the positions made row-relative
  argsort    (one row) gpusorting_b200.argsort(x) on the same keys: the device-wide sort of one row
Workloads: float32 randn * 3 and bfloat16 over [B, V] for V in {32,000, 128,256, 151,936} and B in {1, 8, 64, 256, 1,024};
[16, 2^20] float32 and int64 (uniform over [-2^40, 2^40)); one row of 2^26 float32.  The boundary: sort_rows on
[B, 16,384] against sort_long_rows on [B, 16,385] float32, per key.  The inputs have no NaN and no -0.0 (torch orders -0.0
equal to +0.0).  Every arm's values and positions are compared with the long arm's on the timed inputs, bit for bit.  The
card's name, power limit and SM clocks are read with nvidia-smi (a read-only query) in the same call and printed with the
times.

  python tools/long_rows_timing.py [--warmup 3] [--runs 10] [--quick]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402
from tests import bigcheck  # noqa: E402
from tools.keys16_timing import card, timed  # noqa: E402

VOCABS = (32000, 128256, 151936)
BATCHES = (1, 8, 64, 256, 1024)


def make(shape, dtype, gen):
    if dtype.is_floating_point:
        x = (torch.randn(shape, generator=gen, device="cuda") * 3).to(dtype)
        x[x == 0] = 1
        return x
    return torch.randint(-(1 << 40), 1 << 40, shape, generator=gen, device="cuda", dtype=dtype)


def bits(t):
    return bigcheck.bits_of(t)


def composite(x):
    """the row id above each key's radix image, argsorted on the (8, 4) sorter, split back into values and positions"""
    rows, row_len = x.shape
    kb = x.element_size()
    img = bigcheck.radix16(x.reshape(-1), "bf16" if x.dtype == torch.bfloat16 else "f16").long() if kb == 2 else \
        bigcheck.to_radix32(x.reshape(-1), "f")
    rid = torch.arange(rows, device="cuda").repeat_interleave(row_len)
    key = (rid << (8 * kb)) | img
    _, idx = g.argsort(key, "u64")
    i = idx.long()
    return x.reshape(-1)[i].view(rows, row_len), (i - (i // row_len) * row_len).int().view(rows, row_len)


def agree(a, b):
    return bool(torch.equal(bits(a[0]).reshape(-1), bits(b[0]).reshape(-1)) and
                torch.equal(a[1].int().reshape(-1), b[1].int().reshape(-1)))


def run(arms, warmup, runs):
    outs = {a: fn() for a, fn in arms.items()}
    torch.cuda.synchronize()
    ok = {a: agree(outs["long"], o) for a, o in outs.items() if a != "long"}
    del outs
    torch.cuda.empty_cache()
    times = {a: [] for a in arms}
    for rep in range(warmup + runs):
        for a, fn in arms.items():
            ms, r = timed(fn)
            del r
            if rep >= warmup:
                times[a].append(ms)
    med = {a: statistics.median(t) for a, t in times.items()}
    return {"agrees_with_long": ok, "median_ms": {a: round(v, 4) for a, v in med.items()},
            "min_ms": {a: round(min(t), 4) for a, t in times.items()},
            "max_ms": {a: round(max(t), 4) for a, t in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--quick", action="store_true", help="the smallest workloads only (a rehearsal)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_rows_timing needs a CUDA device")
    result = {"metric": "long_rows_ms", "runs": args.runs, **card(), "workloads": {}}
    gen = torch.Generator(device="cuda").manual_seed(71)
    work = [(name, dtype, (b, v)) for name, dtype in (("f32", torch.float32), ("bf16", torch.bfloat16))
            for v in VOCABS for b in BATCHES]
    work += [("f32", torch.float32, (16, 1 << 20)), ("i64", torch.int64, (16, 1 << 20)), ("f32", torch.float32, (1, 1 << 26))]
    if args.quick:
        work = work[:2]
    for name, dtype, shape in work:
        x = make(shape, dtype, gen)
        arms = {"long": lambda: g.sort_long_rows(x), "torch": lambda: torch.sort(x, dim=-1, stable=True)}
        if x.element_size() <= 4:
            arms["composite"] = lambda: composite(x)
        if shape == (1, 1 << 26):
            arms["argsort"] = lambda: g.argsort(x.view(-1), "f32")
        entry = run(arms, args.warmup, args.runs)
        n = shape[0] * shape[1]
        med = entry["median_ms"]
        entry["keys"] = n
        entry["long_gkeys_per_s"] = round(n / med["long"] / 1e6, 3)
        entry["speedup_over_torch"] = round(med["torch"] / med["long"], 3)
        if "composite" in med:
            entry["speedup_over_composite"] = round(med["composite"] / med["long"], 3)
        result["workloads"][f"{name}/{shape[0]}x{shape[1]}"] = entry
        del x
        torch.cuda.empty_cache()
    if not args.quick:
        for b in (64, 1024):
            xs = make((b, 16384), torch.float32, gen)
            xl = make((b, 16385), torch.float32, gen)
            arms = {"sort_rows_C": lambda: g.sort_rows(xs), "long_C+1": lambda: g.sort_long_rows(xl)}
            times = {a: [] for a in arms}
            for rep in range(args.warmup + args.runs):
                for a, fn in arms.items():
                    ms, r = timed(fn)
                    del r
                    if rep >= args.warmup:
                        times[a].append(ms)
            result["workloads"][f"boundary/{b}"] = {
                "ns_per_key": {a: round(statistics.median(t) * 1e6 / (b * (16384 if a == "sort_rows_C" else 16385)), 4)
                               for a, t in times.items()}}
            del xs, xl
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
