"""Segment top-k (topk_segments) against the routes a caller has without it: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  segments           gpusorting_b200.topk_segments(x, off, k): [S, k] values and int32 positions, sorted
  segments_unsorted  the same with sorted=False
  dense              the composite PyTorch offers: torch.full padding of [S, longest], a scatter of the keys, torch.topk,
                     then the columns past each segment's length masked (the per-element segment ids and positions are
                     built untimed)
  sort_gather        (every segment within the cap: 16,384 keys, 8,192 for int64) sort_segments, then a gather of the first
                     m = min(length, k) keys and positions of each segment
  rows               (equal lengths) topk_rows of the same keys viewed as rows
Workloads: float32 and bfloat16 from torch.randn * 3 and int64 uniform over [-2^62, 2^62), about 2^--log2n keys in segments
whose lengths are log-uniform over 1-64 (k = 8, per-graph selection), uniform over 1,000-20,000 (k = 100, retrieval),
log-uniform over 1-2^17 (k = 50), or all 64 (k = 8) or all 32,000 (k = 50).  The inputs have no NaN and no -0.0.  Every
arm's output is compared on the timed inputs: the dense composite's values (torch's tie order differs, so its indices are
not), sort_gather's and rows' values and indices bit for bit, and the unsorted arm's positions as a set per row.  The card's
name, power limit and SM clocks are read with nvidia-smi (a read-only query) in the same call and printed with the times.

  python tools/topk_segments_timing.py [--log2n 26] [--warmup 3] [--runs 10]"""
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
from tools.rows_timing import inputs  # noqa: E402

WORKLOADS = (("log1-64", 8), ("1000-20000", 100), ("log1-131072", 50), ("equal64", 8), ("equal32000", 50))


def lengths(kind, n, gen):
    """segment lengths summing to at most n"""
    if kind.startswith("equal"):
        L = int(kind[5:])
        return torch.full((n // L,), L, dtype=torch.int64, device="cuda")
    if kind.startswith("log"):
        hi = int(kind.split("-")[1])
        ls = torch.exp(torch.rand(n, generator=gen, device="cuda") * math.log(hi + 1)).long().clamp(1, hi)
    else:
        lo, hi = (int(v) for v in kind.split("-"))
        ls = torch.randint(lo, hi + 1, (n // lo,), generator=gen, device="cuda")
    return ls[: int((ls.cumsum(0) <= n).sum())]


def lowest(dtype):
    return torch.finfo(dtype).min if dtype.is_floating_point else torch.iinfo(dtype).min


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=26)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("topk_segments_timing needs a CUDA device")
    n = 1 << args.log2n
    result = {"metric": "topk_segments_ms", "n": n, "runs": args.runs, **card(), "workloads": {}}
    gen = torch.Generator(device="cuda").manual_seed(29)
    for name, dtype in (("f32", torch.float32), ("bf16", torch.bfloat16), ("i64", torch.int64)):
        cap = 8192 if dtype == torch.int64 else 16384
        for kind, k in WORKLOADS:
            L = lengths(kind, n, gen)
            S = L.numel()
            off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), L.cumsum(0)])
            m_keys = int(off[-1])
            x = inputs(dtype, m_keys, 26)
            if dtype.is_floating_point:
                x = x * 3
            seg = torch.repeat_interleave(torch.arange(S, device="cuda"), L)
            pos = torch.arange(m_keys, device="cuda") - off[:-1][seg]
            max_len = int(L.max())
            kk = min(k, max_len)
            cols = torch.arange(k, device="cuda")
            mask = cols[None, :] < L.clamp(max=k)[:, None]

            def segments():
                return g.topk_segments(x, off, k)

            def segments_unsorted():
                return g.topk_segments(x, off, k, sorted=False)

            def dense():
                d = torch.full((S, max_len), lowest(dtype), dtype=dtype, device="cuda")
                d[seg, pos] = x
                v, i = torch.topk(d, kk, dim=-1)
                return torch.where(mask[:, :kk], v, torch.zeros_like(v)), torch.where(mask[:, :kk], i, -1)

            def sort_gather():
                v, i = g.sort_segments(x, off, descending=True, max_segment_len=max_len)
                src = (off[:-1, None] + cols[None, :]).clamp(max=max(m_keys - 1, 0))
                return v[src], torch.where(mask, i[src], -1)

            arms = {"segments": segments, "segments_unsorted": segments_unsorted, "dense": dense}
            if max_len <= cap:
                arms["sort_gather"] = sort_gather
            if kind.startswith("equal"):
                xr = x.view(S, max_len)
                arms["rows"] = lambda: g.topk(xr, k)
            outs = {a: fn() for a, fn in arms.items()}
            torch.cuda.synchronize()
            sv, si = outs["segments"]
            agree = {}
            dv = outs["dense"][0]
            agree["dense"] = bool(torch.equal(sv[:, :kk][mask[:, :kk]], dv[mask[:, :kk]]))
            uv, ui = outs["segments_unsorted"]
            agree["segments_unsorted"] = bool(torch.equal(torch.sort(ui, dim=1).values, torch.sort(si, dim=1).values))
            if "sort_gather" in outs:
                gv, gi = outs["sort_gather"]
                agree["sort_gather"] = bool(torch.equal(sv[mask], gv[mask]) and torch.equal(si, gi))
            if "rows" in outs:
                rv, ri = outs["rows"]
                agree["rows"] = bool(torch.equal(sv, rv) and torch.equal(si, ri))
            del outs, sv, si, uv, ui, dv
            torch.cuda.empty_cache()
            times = {a: [] for a in arms}
            for rep in range(args.warmup + args.runs):
                for a, fn in arms.items():
                    ms, r = timed(fn)
                    del r
                    if rep >= args.warmup:
                        times[a].append(ms)
            med = {a: statistics.median(t) for a, t in times.items()}
            entry = {
                "keys": m_keys,
                "segments": S,
                "k": k,
                "agrees_with_segments": agree,
                "median_ms": {a: round(v, 3) for a, v in med.items()},
                "min_ms": {a: round(min(t), 3) for a, t in times.items()},
                "max_ms": {a: round(max(t), 3) for a, t in times.items()},
                "speedup_over_dense": round(med["dense"] / med["segments"], 3),
            }
            if "sort_gather" in med:
                entry["speedup_over_sort_gather"] = round(med["sort_gather"] / med["segments"], 3)
            if "rows" in med:
                entry["segments_over_rows"] = round(med["segments"] / med["rows"], 3)
            result["workloads"][f"{name}/{kind}/k{k}"] = entry
            del x, seg, pos, L, off, mask
            torch.cuda.empty_cache()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
