"""Row top-k (gpusorting_b200.topk) against torch.topk, torch.sort + slice and sort_rows + slice: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  topk            gpusorting_b200.topk(x, k): values and int32 indices in stable-sort order
  topk_unsorted   gpusorting_b200.topk(x, k, sorted=False)
  torch_topk      torch.topk(x, k, dim=-1)
  torch_sort      torch.sort(x, dim=-1, descending=True, stable=True), then [..., :k]
  rows            (rows of at most 16,384 keys) gpusorting_b200.sort_rows(x, descending=True), then [..., :k]
Workloads (k largest):
  MoE routing     float32 randn*3, [2^20, 64] with k = 2 and 8, [2^18, 256] with k = 8
  retrieval       float32 randn*3, [2^14, 1,024] and [2^12, 4,096] with k = 64
  sampling        batch 1, 8, 64, 256 and 1,024 over vocabularies of 32,000, 128,256 and 151,936 keys, k = 50 and 1,024, float32
                  and bfloat16, randn*3 (logits: few distinct top digits) and uniform in [0, 1)
Before any time is used, every arm's output is compared: topk's values and indices bit for bit with torch.sort's first k
columns (and with sort_rows'), its values with torch.topk's, and topk_unsorted's (value, position) pairs with topk's.  The
inputs have no NaN and no -0.0, where torch's order differs from the bit-pattern order.  The card's name, power limit and SM
clocks are read with nvidia-smi (a read-only query) in the same call and printed with the times.

  python tools/topk_timing.py [--warmup 3] [--runs 10] [--only moe,retrieval,sampling]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402
from tools.keys16_timing import card, timed  # noqa: E402


def inputs(shape, dtype, dist, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if dist == "uniform":
        return torch.rand(shape, generator=gen, device="cuda").to(dtype)
    x = (torch.randn(shape, generator=gen, device="cuda") * 3).to(dtype)
    return torch.where(x == 0, torch.ones_like(x), x)


def workloads(only):
    out = []
    if "moe" in only:
        out += [("moe", torch.float32, "randn3", (1 << 20, 64), 2), ("moe", torch.float32, "randn3", (1 << 20, 64), 8),
                ("moe", torch.float32, "randn3", (1 << 18, 256), 8)]
    if "retrieval" in only:
        out += [("retrieval", torch.float32, "randn3", (1 << 14, 1024), 64),
                ("retrieval", torch.float32, "randn3", (1 << 12, 4096), 64)]
    if "sampling" in only:
        for dtype in (torch.float32, torch.bfloat16):
            for dist in ("randn3", "uniform"):
                for vocab in (32000, 128256, 151936):
                    for batch in (1, 8, 64, 256, 1024):
                        for k in (50, 1024):
                            out.append(("sampling", dtype, dist, (batch, vocab), k))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--only", default="moe,retrieval,sampling")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("topk_timing needs a CUDA device")
    result = {"metric": "topk_ms", "runs": args.runs, **card(), "workloads": {}}
    for i, (kind, dtype, dist, shape, k) in enumerate(workloads(args.only.split(","))):
        x = inputs(shape, dtype, dist, 100 + i)
        arms = {
            "topk": lambda: g.topk(x, k),
            "topk_unsorted": lambda: g.topk(x, k, sorted=False),
            "torch_topk": lambda: torch.topk(x, k, dim=-1),
            "torch_sort": lambda: [t[..., :k] for t in torch.sort(x, dim=-1, descending=True, stable=True)],
        }
        if shape[-1] <= 16384:
            arms["rows"] = lambda: [t[..., :k] for t in g.sort_rows(x, descending=True)]
        outs = {a: fn() for a, fn in arms.items()}
        torch.cuda.synchronize()
        v, i_ = outs["topk"]
        sv, si = outs["torch_sort"]
        uv, ui = outs["topk_unsorted"]
        by_pos, u_by_pos = torch.argsort(i_, dim=-1), torch.argsort(ui, dim=-1)
        agree = {
            "topk_vs_torch_sort": bool(torch.equal(v, sv) and torch.equal(i_.long(), si)),
            "topk_vs_torch_topk_values": bool(torch.equal(v, outs["torch_topk"].values)),
            "unsorted_vs_topk": bool(torch.equal(torch.gather(ui, -1, u_by_pos), torch.gather(i_, -1, by_pos))
                                     and torch.equal(torch.gather(uv, -1, u_by_pos), torch.gather(v, -1, by_pos))),
        }
        if "rows" in outs:
            rv, ri = outs["rows"]
            agree["topk_vs_rows"] = bool(torch.equal(v, rv) and torch.equal(i_, ri))
        del outs, v, i_, sv, si, uv, ui, by_pos, u_by_pos
        torch.cuda.empty_cache()
        times = {a: [] for a in arms}
        for rep in range(args.warmup + args.runs):
            for a, fn in arms.items():
                ms, r = timed(fn)
                del r
                if rep >= args.warmup:
                    times[a].append(ms)
        med = {a: statistics.median(t) for a, t in times.items()}
        name = f"{kind}/{str(dtype).replace('torch.', '')}/{dist}/{shape[0]}x{shape[1]}/k{k}"
        result["workloads"][name] = {
            "agree": agree,
            "median_ms": {a: round(m, 4) for a, m in med.items()},
            "min_ms": {a: round(min(t), 4) for a, t in times.items()},
            "max_ms": {a: round(max(t), 4) for a, t in times.items()},
            "speedup_over_torch_topk": round(med["torch_topk"] / med["topk"], 3),
            "speedup_over_torch_sort": round(med["torch_sort"] / med["topk"], 3),
            "unsorted_speedup_over_torch_topk": round(med["torch_topk"] / med["topk_unsorted"], 3),
        }
        if "rows" in med:
            result["workloads"][name]["speedup_over_rows"] = round(med["rows"] / med["topk"], 3)
        del x
        torch.cuda.empty_cache()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
