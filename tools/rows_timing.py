"""Row sort (sort_rows) against torch.sort(x, dim=-1, stable=True), and its warp path against its block path: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  rows          gpusorting_b200.sort_rows(x): values and int32 indices, new tensors
  torch         torch.sort(x, dim=-1, stable=True): values and int64 indices
  rows_keys     sort_rows(x, return_indices=False)
  rows_block, rows_block_keys   (rows of at most 256 keys) the same two calls with option "debug_rows_block" = 1, which sends
                the short rows through the block path (one 256-thread CTA and a 2,048-key tile per row) instead of one warp per row
  segmented_u32_keys  (float32 rows of at most 256 keys) segmented_sort of the uint32 view, in place on a copy (the copy
                untimed): the existing segmented sort in its 256-key geometry; compared with sort_rows of the uint32 view
Workloads: float32 and bfloat16 from torch.randn and int64 uniform over [-2^62, 2^62), 2^--log2n keys in rows of 32, 64,
256, 1,024, 4,096 and 16,384 keys (8,192 for int64: the longest row a 64-bit sort takes).  The inputs have no NaN and no -0.0,
where torch's order differs from the bit-pattern order; with those excluded the outputs of every arm are compared bit for
bit (torch's int64 indices with .long() of ours).  The card's name, power limit and SM clocks are read with nvidia-smi (a
read-only query) in the same call and printed with the times.

  python tools/rows_timing.py [--log2n 26] [--warmup 3] [--runs 10]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402
from tools.keys16_timing import card, timed  # noqa: E402


def inputs(dtype, n, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if dtype == torch.int64:
        return torch.randint(-(1 << 62), 1 << 62, (n,), generator=gen, device="cuda", dtype=torch.int64)
    x = torch.randn(n, generator=gen, device="cuda").to(dtype)
    return torch.where(x == 0, torch.ones_like(x), x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=26)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rows_timing needs a CUDA device")
    n = 1 << args.log2n
    result = {"metric": "rows_ms", "n": n, "runs": args.runs, **card(), "workloads": {}}
    # the sorter module-level sort_rows uses on the current stream: the hook is set on it for the block arms
    s = g.onesweep._cached_sorter(torch.cuda.current_device(), 4, 4, 1, int(torch.cuda.current_stream().cuda_stream))
    for name, dtype in (("f32", torch.float32), ("bf16", torch.bfloat16), ("i64", torch.int64)):
        x = inputs(dtype, n, 26)
        for row_len in (32, 64, 256, 1024, 4096, 8192 if dtype == torch.int64 else 16384):
            xr = x.view(-1, row_len)

            def rows():
                return g.sort_rows(xr)

            def rows_keys():
                return g.sort_rows(xr, return_indices=False)

            def torch_sort():
                return torch.sort(xr, dim=-1, stable=True)

            def block(fn):
                def run():
                    s.set_option("debug_rows_block", 1)
                    try:
                        return fn()
                    finally:
                        s.set_option("debug_rows_block", 0)
                return run

            arms = {"rows": rows, "torch": torch_sort, "rows_keys": rows_keys}
            preps = {}
            if row_len <= 256:
                arms["rows_block"] = block(rows)
                arms["rows_block_keys"] = block(rows_keys)
            if row_len <= 256 and dtype == torch.float32:
                # the segmented sort (uint32 keys, in place) over the same rows: its 256-key geometry
                xu = xr.view(torch.uint32)
                seg_buf = torch.empty_like(xu)
                offsets = torch.arange(0, n + 1, row_len, dtype=torch.int64, device="cuda")
                arms["segmented_u32_keys"] = lambda: s.segmented_sort(seg_buf.view(-1), offsets, max_segment_len=row_len)
                preps["segmented_u32_keys"] = lambda: seg_buf.copy_(xu)
            outs = {}
            for a, fn in arms.items():
                if a in preps:
                    preps[a]()
                outs[a] = fn()
            torch.cuda.synchronize()
            ref_v, ref_i = outs["torch"]
            identical = {}
            for a, o in outs.items():
                if a == "torch":
                    continue
                if a == "segmented_u32_keys":  # unsigned order: compared with the row sort of the uint32 view
                    identical[a] = bool(torch.equal(seg_buf, g.sort_rows(xu, return_indices=False)))
                    continue
                v, i = o if isinstance(o, tuple) else (o, None)
                identical[a] = bool(torch.equal(v, ref_v) and (i is None or torch.equal(i.long(), ref_i)))
            del outs, ref_v, ref_i
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
                "rows": n // row_len,
                "identical_to_torch": identical,
                "median_ms": {a: round(v, 3) for a, v in med.items()},
                "min_ms": {a: round(min(t), 3) for a, t in times.items()},
                "max_ms": {a: round(max(t), 3) for a, t in times.items()},
                "rows_speedup_over_torch": round(med["torch"] / med["rows"], 3),
                "gkeys_per_s": {a: round(n / (v * 1e6), 2) for a, v in med.items()},
            }
            if row_len <= 256:
                entry["warp_speedup_over_block"] = round(med["rows_block"] / med["rows"], 3)
                entry["warp_speedup_over_block_keys"] = round(med["rows_block_keys"] / med["rows_keys"], 3)
            if "segmented_u32_keys" in med:
                entry["warp_speedup_over_segmented_keys"] = round(med["segmented_u32_keys"] / med["rows_keys"], 3)
            result["workloads"][f"{name}/{row_len}"] = entry
            torch.cuda.empty_cache()
        del x
        torch.cuda.empty_cache()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
