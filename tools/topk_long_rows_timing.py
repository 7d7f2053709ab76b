"""Row top-k of long rows (gpusorting_b200.topk_long_rows) against topk, torch.topk and torch.sort + slice: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  long            gpusorting_b200.topk_long_rows(x, k): values and int32 indices in stable-sort order
  long_unsorted   gpusorting_b200.topk_long_rows(x, k, sorted=False)
  topk            (k <= 16,384, 8,192 for 8-byte keys) gpusorting_b200.topk(x, k): one CTA per row
  torch_topk      torch.topk(x, k, dim=-1)
  torch_sort      torch.sort(x, dim=-1, descending=True, stable=True), then [..., :k]
Workloads (k largest):
  sampling        float32 and bfloat16, randn*3 and uniform in [0, 1), batch 1, 8 and 64 over 32,000, 128,256 and 151,936
                  keys with k = 50 and 1,024 -- below the path rule's threshold (the SM count), the split path
  batch           batch 256 and 1,024 over 128,256 float32 keys, k = 50 -- at or above it, topk_rows' launch
  flat            one row of 2^26 and 2^28 float32 keys (randn*3), k = 1,000, 2^16 and 2^20
  int64           [16, 2^20] int64 (uniform over the full range), k = 50 and 2^14
Before any time is used, every arm's output is compared: long's values and indices bit for bit with torch.sort's first k
columns and with topk's, its values with torch.topk's, and long_unsorted's (value, position) pairs with long's.  The inputs
have no NaN and no -0.0, where torch's order differs from the bit-pattern order.  The card's name, power limit and SM clocks
are read with nvidia-smi (a read-only query) in the same call and printed with the times.

  python tools/topk_long_rows_timing.py [--warmup 3] [--runs 10] [--only sampling,batch,flat,int64]"""
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
    if dtype == torch.int64:
        return torch.randint(-(1 << 62), 1 << 62, shape, generator=gen, device="cuda", dtype=torch.int64)
    if dist == "uniform":
        return torch.rand(shape, generator=gen, device="cuda").to(dtype)
    x = (torch.randn(shape, generator=gen, device="cuda") * 3).to(dtype)
    return torch.where(x == 0, torch.ones_like(x), x)


def workloads(only):
    out = []
    if "sampling" in only:
        for dtype in (torch.float32, torch.bfloat16):
            for dist in ("randn3", "uniform"):
                for vocab in (32000, 128256, 151936):
                    for batch in (1, 8, 64):
                        for k in (50, 1024):
                            out.append(("sampling", dtype, dist, (batch, vocab), k))
    if "batch" in only:
        out += [("batch", torch.float32, "randn3", (b, 128256), 50) for b in (256, 1024)]
    if "flat" in only:
        out += [("flat", torch.float32, "randn3", (1, n), k) for n in (1 << 26, 1 << 28) for k in (1000, 1 << 16, 1 << 20)]
    if "int64" in only:
        out += [("int64", torch.int64, "full", (16, 1 << 20), k) for k in (50, 1 << 14)]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--only", default="sampling,batch,flat,int64")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("topk_long_rows_timing needs a CUDA device")
    result = {"metric": "topk_long_rows_ms", "runs": args.runs, **card(), "workloads": {}}
    for i, (kind, dtype, dist, shape, k) in enumerate(workloads(args.only.split(","))):
        x = inputs(shape, dtype, dist, 100 + i)
        arms = {
            "long": lambda: g.topk_long_rows(x, k),
            "long_unsorted": lambda: g.topk_long_rows(x, k, sorted=False),
            "torch_topk": lambda: torch.topk(x, k, dim=-1),
            "torch_sort": lambda: [t[..., :k] for t in torch.sort(x, dim=-1, descending=True, stable=True)],
        }
        if k <= (8192 if x.element_size() == 8 else 16384):
            arms["topk"] = lambda: g.topk(x, k)
        outs = {a: fn() for a, fn in arms.items()}
        torch.cuda.synchronize()
        v, i_ = outs["long"]
        sv, si = outs["torch_sort"]
        uv, ui = outs["long_unsorted"]
        by_pos, u_by_pos = torch.argsort(i_, dim=-1), torch.argsort(ui, dim=-1)
        agree = {
            "long_vs_torch_sort": bool(torch.equal(v, sv) and torch.equal(i_.long(), si)),
            "long_vs_torch_topk_values": bool(torch.equal(v, outs["torch_topk"].values)),
            "unsorted_vs_long": bool(torch.equal(torch.gather(ui, -1, u_by_pos), torch.gather(i_, -1, by_pos))
                                     and torch.equal(torch.gather(uv, -1, u_by_pos), torch.gather(v, -1, by_pos))),
        }
        if "topk" in outs:
            tv, ti = outs["topk"]
            agree["long_vs_topk"] = bool(torch.equal(v, tv) and torch.equal(i_, ti))
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
        entry = {
            "agree": agree,
            "median_ms": {a: round(m, 4) for a, m in med.items()},
            "min_ms": {a: round(min(t), 4) for a, t in times.items()},
            "max_ms": {a: round(max(t), 4) for a, t in times.items()},
            "speedup_over_torch_topk": round(med["torch_topk"] / med["long"], 3),
            "speedup_over_torch_sort": round(med["torch_sort"] / med["long"], 3),
            "unsorted_speedup_over_torch_topk": round(med["torch_topk"] / med["long_unsorted"], 3),
        }
        if "topk" in med:
            entry["speedup_over_topk"] = round(med["topk"] / med["long"], 3)
        result["workloads"][name] = entry
        del x
        torch.cuda.empty_cache()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
