"""Row select (gpusorting_b200.kthvalue / median / quantile, osb200_select_rows) against torch and against sorting: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  select          the library's kthvalue / median / quantile (values and int32 positions; quantile: values)
  lib_sort        gpusorting_b200.sort_long_rows, then the columns (and ATen's quantile formula)
  torch_sort      torch.sort(stable=True), then the columns (and ATen's quantile formula)
  torch_kth       torch.kthvalue / torch.median (dim=-1), where torch has them
  torch_topk      (threshold workloads) torch.topk(x, 50).values[..., -1]
  split           (paths workloads) select_rows on a sorter with the "debug_long_rows" hook: the split path on rows the
                  row sort's kernels would take
Workloads:
  median, quantile  [1, 2^26] float32 randn*3: median, and quantile(q = [0.01, 0.5, 0.99]) (torch.quantile refuses it)
  q999             quantile(0.999) of [1, 2^28] float32
  int64            kthvalue(k = 2^19) of [16, 2^20] int64
  bf16             median of [1, 2^26] bfloat16
  threshold        kthvalue(x, L - 50 + 1), the top-k filtering threshold, of [1, 8, 64, 256] x 128,256 float32 and bfloat16
  short            median of [2^20, 64], [2^14, 1024] and [2^12, 16384] float32
  skewed           median of [1, 2^26] float32, all keys equal, and with a constant top byte
  paths            median of [64, 16384] and [2^12, 16384] float32: the row sort's kernels against the split path
Before any time is used, every arm's output is compared: values bit for bit, and positions where an arm has them (torch's
kthvalue / median only where the key is unique in its row).  The inputs have no NaN and no -0.0, where torch's order differs
from the bit-pattern order.  The card's name, power limit and SM clocks are read with nvidia-smi (a read-only query) in the
same call and printed with the times.

  python tools/select_rows_timing.py [--warmup 2] [--runs 9] [--only median,quantile,q999,int64,bf16,threshold,short,skewed,paths]"""
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
    if dist == "equal":
        return torch.full(shape, 1.5, device="cuda", dtype=dtype)
    if dist == "top_byte":  # positive floats in [2, 4): one top byte
        return (2 + 2 * torch.rand(shape, generator=gen, device="cuda")).to(dtype)
    x = (torch.randn(shape, generator=gen, device="cuda") * 3).to(dtype)
    return torch.where(x == 0, torch.ones_like(x), x)


def aten_quantile(srt, q, L):
    """ATen's quantile on sorted rows: ranks q * (L - 1) in the keys' dtype, linear interpolation"""
    pos = torch.tensor(q, dtype=srt.dtype) * (L - 1)
    below = pos.long().clamp(0, L - 1)
    above = pos.ceil().long().clamp(0, L - 1)
    w = (pos - below.to(srt.dtype)).to(srt.device)
    return torch.lerp(srt[..., below.to(srt.device)], srt[..., above.to(srt.device)], w.expand(*srt.shape[:-1], len(q)))


def workloads(only):
    out = []
    if "median" in only:
        out.append(("median", torch.float32, "randn3", (1, 1 << 26), "median"))
    if "quantile" in only:
        out.append(("quantile", torch.float32, "randn3", (1, 1 << 26), [0.01, 0.5, 0.99]))
    if "q999" in only:
        out.append(("q999", torch.float32, "randn3", (1, 1 << 28), [0.999]))
    if "int64" in only:
        out.append(("int64", torch.int64, "full", (16, 1 << 20), 1 << 19))
    if "bf16" in only:
        out.append(("bf16", torch.bfloat16, "randn3", (1, 1 << 26), "median"))
    if "threshold" in only:
        out += [("threshold", dt, "randn3", (b, 128256), 128256 - 50 + 1) for dt in (torch.float32, torch.bfloat16)
                for b in (1, 8, 64, 256)]
    if "short" in only:
        out += [("short", torch.float32, "randn3", s, "median") for s in ((1 << 20, 64), (1 << 14, 1024), (1 << 12, 16384))]
    if "skewed" in only:
        out += [("skewed", torch.float32, d, (1, 1 << 26), "median") for d in ("equal", "top_byte")]
    if "paths" in only:
        out += [("paths", torch.float32, "randn3", s, "median") for s in ((64, 16384), (1 << 12, 16384))]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--only", default="median,quantile,q999,int64,bf16,threshold,short,skewed,paths")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("select_rows_timing needs a CUDA device")
    result = {"metric": "select_rows_ms", "runs": args.runs, **card(), "workloads": {}}
    for i, (kind, dtype, dist, shape, what) in enumerate(workloads(args.only.split(","))):
        x = inputs(shape, dtype, dist, 300 + i)
        L = shape[-1]
        split = None
        if isinstance(what, list):  # quantiles: values only
            arms = {
                "select": lambda: g.quantile(x, what, dim=-1),
                "lib_sort": lambda: aten_quantile(g.sort_long_rows(x, return_indices=False), what, L),
                "torch_sort": lambda: aten_quantile(torch.sort(x, dim=-1, stable=True).values, what, L),
            }
        else:
            k = (L - 1) // 2 + 1 if what == "median" else what
            arms = {
                "select": lambda: g.kthvalue(x, k),
                "lib_sort": lambda: [t[..., k - 1] for t in g.sort_long_rows(x)],
                "torch_sort": lambda: [t[..., k - 1] for t in torch.sort(x, dim=-1, stable=True)],
                "torch_kth": (lambda: torch.median(x, dim=-1)) if what == "median" else (lambda: torch.kthvalue(x, k, dim=-1)),
            }
            if kind == "threshold":
                arms["torch_topk"] = lambda: (torch.topk(x, 50, dim=-1).values[..., -1], None)
            if kind == "paths":
                split = g.OneSweepSorter(g.select_workspace_words(shape[0], L, 1), 4, 0)
                split.set_option("debug_long_rows", 1)
                arms["split"] = lambda: split.select_rows(x, [k - 1], "f32")
        outs = {a: fn() for a, fn in arms.items()}
        torch.cuda.synchronize()
        if isinstance(what, list):
            agree = {a: bool(torch.equal(outs[a].reshape(-1), outs["select"].reshape(-1))) for a in arms if a != "select"}  # one row
        else:
            v, idx = outs["select"]
            agree = {}
            for a in ("lib_sort", "torch_sort", "split"):
                if a in outs:
                    ov, oi = outs[a]
                    ov, oi = ov.reshape(v.shape), oi.reshape(v.shape)
                    agree[a] = bool(torch.equal(ov, v) and torch.equal(oi.long(), idx.long()))
            tv, ti = outs["torch_kth"]
            unique = (x == v.unsqueeze(-1)).sum(-1) == 1
            agree["torch_kth"] = bool(torch.equal(tv, v) and torch.equal(ti[unique], idx.long()[unique]))
            if "torch_topk" in outs:
                agree["torch_topk"] = bool(torch.equal(outs["torch_topk"][0], v))
        del outs
        torch.cuda.empty_cache()
        times = {a: [] for a in arms}
        for rep in range(args.warmup + args.runs):
            for a, fn in arms.items():
                ms, r = timed(fn)
                del r
                if rep >= args.warmup:
                    times[a].append(ms)
        med = {a: statistics.median(t) for a, t in times.items()}
        name = f"{kind}/{str(dtype).replace('torch.', '')}/{dist}/{shape[0]}x{shape[1]}/" + (
            "q" + ",".join(str(q) for q in what) if isinstance(what, list) else str(what))
        result["workloads"][name] = {
            "agree": agree,
            "median_ms": {a: round(m, 4) for a, m in med.items()},
            "min_ms": {a: round(min(t), 4) for a, t in times.items()},
            "max_ms": {a: round(max(t), 4) for a, t in times.items()},
            "speedup": {a: round(m / med["select"], 3) for a, m in med.items() if a != "select"},
        }
        if split is not None:
            split.close()
        del x
        torch.cuda.empty_cache()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
