"""Segment sort (sort_segments) against the routes a caller has without it: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  segments       gpusorting_b200.sort_segments(x, off): values and int32 indices within the segment, new tensors
  segments_keys  sort_segments(x, off, return_indices=False)
  torch          the composite PyTorch offers: torch.sort(x, stable=True), gather the segment ids, stable torch.sort of
                 those, gather again (values and global int64 positions; the per-element segment ids are built untimed)
  segmented_u32_keys  (4-byte dtypes) osb200_segmented_sort_u32 of the uint32 view, in place on a copy (the copy untimed);
                 compared with sort_segments of the same uint32 view
  rows, rows_keys     (equal lengths) sort_rows of the same keys viewed as rows
Workloads: float32 and bfloat16 from torch.randn and int64 uniform over [-2^62, 2^62), about 2^--log2n keys in segments
whose lengths are uniform over 1-8, 1-64, 1-256, 257-2,048 and 2,049 to the cap (16,384 keys, 8,192 for int64),
log-uniform over 1 to the cap, or all 256 or 2,048.  The inputs have no NaN and no -0.0, where torch's order differs from
the bit-pattern order; with those excluded every arm's output is compared bit for bit (our indices plus the segment's
offset against torch's positions).  The card's name, power limit and SM clocks are read with nvidia-smi (a read-only
query) in the same call and printed with the times.

  python tools/segments_timing.py [--log2n 26] [--warmup 3] [--runs 10]"""
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


def lengths(kind, n, cap, gen):
    """segment lengths summing to at most n"""
    k = n  # enough draws for any workload: every length is at least 1
    if kind.startswith("equal"):
        L = int(kind[5:])
        return torch.full((n // L,), L, dtype=torch.int64, device="cuda")
    if kind == "log":
        ls = torch.exp(torch.rand(k, generator=gen, device="cuda") * math.log(cap + 1)).long().clamp(1, cap)
    else:
        lo, hi = {"1-8": (1, 8), "1-64": (1, 64), "1-256": (1, 256), "257-2048": (257, 2048), "2049-cap": (2049, cap)}[kind]
        ls = torch.randint(lo, hi + 1, (k // lo,), generator=gen, device="cuda")
    return ls[: int((ls.cumsum(0) <= n).sum())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=26)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("segments_timing needs a CUDA device")
    n = 1 << args.log2n
    result = {"metric": "segments_ms", "n": n, "runs": args.runs, **card(), "workloads": {}}
    s = g.onesweep._cached_sorter(torch.cuda.current_device(), 4, 4, n, int(torch.cuda.current_stream().cuda_stream))
    gen = torch.Generator(device="cuda").manual_seed(27)
    for name, dtype in (("f32", torch.float32), ("bf16", torch.bfloat16), ("i64", torch.int64)):
        cap = 8192 if dtype == torch.int64 else 16384
        for kind in ("1-8", "1-64", "1-256", "257-2048", "2049-cap", "log", "equal256", "equal2048"):
            L = lengths(kind, n, cap, gen)
            off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), L.cumsum(0)])
            m = int(off[-1])
            x = inputs(dtype, m, 26)
            seg = torch.repeat_interleave(torch.arange(L.numel(), device="cuda"), L)
            max_len = int(L.max())

            def segments():
                return g.sort_segments(x, off, max_segment_len=max_len)

            def segments_keys():
                return g.sort_segments(x, off, return_indices=False, max_segment_len=max_len)

            def torch_composite():
                o1 = torch.sort(x, stable=True)[1]
                o2 = torch.sort(seg[o1], stable=True)[1]
                perm = o1[o2]
                return x[perm], perm

            arms = {"segments": segments, "segments_keys": segments_keys, "torch": torch_composite}
            preps = {}
            if x.element_size() == 4:
                xu = x.view(torch.uint32)
                seg_buf = torch.empty_like(xu)
                arms["segmented_u32_keys"] = lambda: s.segmented_sort(seg_buf, off, max_segment_len=max_len)
                preps["segmented_u32_keys"] = lambda: seg_buf.copy_(xu)
            if kind.startswith("equal"):
                xr = x.view(-1, max_len)
                arms["rows"] = lambda: g.sort_rows(xr)
                arms["rows_keys"] = lambda: g.sort_rows(xr, return_indices=False)
            outs = {}
            for a, fn in arms.items():
                if a in preps:
                    preps[a]()
                outs[a] = fn()
            torch.cuda.synchronize()
            ref_v, ref_p = outs["torch"]
            start = off[:-1].repeat_interleave(L)
            identical = {}
            for a, o in outs.items():
                if a == "torch":
                    continue
                if a == "segmented_u32_keys":  # unsigned order: compared with the segment sort of the uint32 view
                    identical[a] = bool(torch.equal(seg_buf, g.sort_segments(xu, off, return_indices=False, max_segment_len=max_len)))
                    continue
                v, i = o if isinstance(o, tuple) else (o, None)
                v = v.reshape(-1)
                same_v = torch.equal(v.view(torch.int16), ref_v.view(torch.int16)) if dtype == torch.bfloat16 else torch.equal(v, ref_v)
                identical[a] = bool(same_v and (i is None or torch.equal(i.reshape(-1).long() + start, ref_p)))
            del outs, ref_v, ref_p, start
            torch.cuda.empty_cache()
            times = {a: [] for a in arms}
            for rep in range(args.warmup + args.runs):
                for a, fn in arms.items():
                    ms, r = timed(fn, preps.get(a))
                    del r
                    if rep >= args.warmup:
                        times[a].append(ms)
            med = {a: statistics.median(t) for a, t in times.items()}
            entry = {
                "keys": m,
                "segments": L.numel(),
                "identical_to_torch": identical,
                "median_ms": {a: round(v, 3) for a, v in med.items()},
                "min_ms": {a: round(min(t), 3) for a, t in times.items()},
                "max_ms": {a: round(max(t), 3) for a, t in times.items()},
                "speedup_over_torch": round(med["torch"] / med["segments"], 3),
            }
            if "rows" in med:
                entry["segments_over_rows"] = round(med["segments"] / med["rows"], 3)
                entry["segments_keys_over_rows_keys"] = round(med["segments_keys"] / med["rows_keys"], 3)
            if "segmented_u32_keys" in med:
                entry["speedup_over_segmented_u32_keys"] = round(med["segmented_u32_keys"] / med["segments_keys"], 3)
            result["workloads"][f"{name}/{kind}"] = entry
            del x, seg, L, off
            torch.cuda.empty_cache()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
