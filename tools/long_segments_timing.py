"""Long-segment sort (sort_long_segments) against the routes a caller has without it: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  long       gpusorting_b200.sort_long_segments(x, off, max_segment_len=...): values and int32 positions within the segment
  long_keys  the same with return_indices=False
  torch      the composite PyTorch offers: torch.sort(x, stable=True), gather the segment ids, stable torch.sort of those,
             gather again (values and global int64 positions; the per-element segment ids are built untimed)
  segments   (every segment within sort_segments' limit) gpusorting_b200.sort_segments with the same bound
  rows       (equal lengths) gpusorting_b200.sort_long_rows of the same keys viewed as rows
Workloads: float32 and bfloat16 randn * 3 and int64 uniform over [-2^62, 2^62), about 2^--log2n keys in segments whose
lengths are uniform over 1,000-20,000, log-uniform over 1-2^17, all 32,000 or all 151,936; segments within the limit C
(16,384 keys, 8,192 for int64; lengths log-uniform over 1-C) with max_segment_len = C and with a loose bound of 2^20, which
sends the call down the long path with no long segment (the cost of its histogram and plan); and one segment of 2^--log2n
keys.  The inputs have no NaN and no -0.0, where torch's order differs from the bit-pattern order; with those excluded
every arm's output is compared with the long arm's bit for bit (positions made global with the segment's offset).  The
card's name, power limit and SM clocks are read with nvidia-smi (a read-only query) in the same call and printed with the
times.

  python tools/long_segments_timing.py [--log2n 26] [--warmup 3] [--runs 10] [--quick]"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402
from tools.keys16_timing import card, timed  # noqa: E402

INT_OF = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def make(dtype, n, gen):
    if dtype == torch.int64:
        return torch.randint(-(1 << 62), 1 << 62, (n,), generator=gen, device="cuda", dtype=torch.int64)
    x = (torch.randn(n, generator=gen, device="cuda") * 3).to(dtype)
    return torch.where(x == 0, torch.ones_like(x), x)


def lengths(kind, n, cap, gen):
    """segment lengths summing to at most n"""
    if kind.startswith("equal"):
        L = int(kind[5:])
        return torch.full((n // L,), L, dtype=torch.int64, device="cuda")
    if kind == "single":
        return torch.full((1,), n, dtype=torch.int64, device="cuda")
    if kind == "uniform1000-20000":
        ls = torch.randint(1000, 20001, (n // 1000,), generator=gen, device="cuda")
    else:
        top = (1 << 17) if kind == "log1-2^17" else cap
        ls = torch.exp(torch.rand(n, generator=gen, device="cuda") * math.log(top + 1)).long().clamp(1, top)
    return ls[: int((ls.cumsum(0) <= n).sum())]


def run(arms, ref, check, warmup, runs):
    outs = {a: fn() for a, fn in arms.items()}
    torch.cuda.synchronize()
    ok = {a: check(outs[ref], o, a) for a, o in outs.items() if a != ref}
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
    ap.add_argument("--log2n", type=int, default=26)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--quick", action="store_true", help="the first two workloads of float32 only (a rehearsal)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_segments_timing needs a CUDA device")
    n = 1 << args.log2n
    result = {"metric": "long_segments_ms", "n": n, "runs": args.runs, **card(), "workloads": {}}
    gen = torch.Generator(device="cuda").manual_seed(83)
    kinds = ("uniform1000-20000", "log1-2^17", "equal32000", "equal151936", "within_cap", "within_cap_loose", "single")
    for name, dtype in (("f32", torch.float32), ("bf16", torch.bfloat16), ("i64", torch.int64)):
        cap = 8192 if dtype == torch.int64 else 16384
        for kind in kinds[:2] if args.quick else kinds:
            if args.quick and name != "f32":
                break
            L = lengths("log1-cap" if kind.startswith("within_cap") else kind, n, cap, gen)
            off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), L.cumsum(0)])
            m = int(off[-1])
            x = make(dtype, m, gen)
            seg = torch.repeat_interleave(torch.arange(L.numel(), device="cuda"), L)
            start = off[:-1].repeat_interleave(L)
            max_len = (1 << 20) if kind == "within_cap_loose" else int(L.max())
            ib = INT_OF[x.element_size()]

            def torch_composite():
                o1 = torch.sort(x, stable=True)[1]
                o2 = torch.sort(seg[o1], stable=True)[1]
                perm = o1[o2]
                return x[perm], perm

            def check(ref, o, arm):
                keys = o if not isinstance(o, tuple) else o[0]
                good = bool(torch.equal(ref[0].view(ib), keys.view(ib).reshape(-1)))
                if isinstance(o, tuple):
                    pos = o[1].reshape(-1).long()
                    good = good and bool(torch.equal(ref[1].long() + start, pos if arm == "torch" else pos + start))
                return good

            arms = {"long": lambda: g.sort_long_segments(x, off, max_segment_len=max_len),
                    "long_keys": lambda: g.sort_long_segments(x, off, return_indices=False, max_segment_len=max_len),
                    "torch": torch_composite}
            if max_len <= cap:
                arms["segments"] = lambda: g.sort_segments(x, off, max_segment_len=max_len)
            if kind.startswith("equal") or kind == "single":
                xr = x.view(-1, int(L[0]))
                arms["rows"] = lambda: g.sort_long_rows(xr)
            entry = run(arms, "long", check, args.warmup, args.runs)
            med = entry["median_ms"]
            entry.update({"keys": m, "segments": int(L.numel()), "max_segment_len": max_len,
                          "long_gkeys_per_s": round(m / med["long"] / 1e6, 3),
                          "speedup_over_torch": round(med["torch"] / med["long"], 3)})
            for other in ("segments", "rows"):
                if other in med:
                    entry[f"speedup_over_{other}"] = round(med[other] / med["long"], 3)
            result["workloads"][f"{name}/{kind}"] = entry
            del x, seg, start, arms
            torch.cuda.empty_cache()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
