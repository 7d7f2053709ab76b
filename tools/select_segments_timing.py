"""Segment select (gpusorting_b200.select_segments / median_segments / quantile_segments, osb200_select_segments) against
sorting every segment: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  select     select_segments at the query's ranks per segment (values and int32 positions), ranks built on the device
  lib_sort   gpusorting_b200.sort_long_segments (values and positions), then a gather at offsets[s] + rank
  torch      the composite PyTorch offers: torch.sort(x, stable=True), gather the segment ids, a stable torch.sort of those,
             then the gather
  torch_q    (quantile, float32 only, where the segments are few) torch.quantile of every segment in a Python loop
Workloads, about 2^26 keys each, for float32 randn*3, bfloat16 and int64: log-uniform lengths 1-64, uniform 1,000-20,000,
log-uniform 1-2^17, all 151,936, and one segment of 2^26.  Queries: median (rank (L - 1) // 2), and the ranks of quantile
q = [0.01, 0.5, 0.99] (lower and upper rank of each, plus 0 and L - 1: 8 ranks).  max_segment_len is passed, so no arm
waits on the host.  Before any time is used the arms' values and positions are compared bit for bit.  The card's name,
power limit and SM clocks are read with nvidia-smi (a read-only query) in the same call.

  python tools/select_segments_timing.py [--warmup 2] [--runs 9] [--only logu64,uni20k,logu17,vocab,one]"""
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

N = 1 << 26
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "i64": torch.int64}
QS = [0.01, 0.5, 0.99]


def lengths_for(name, gen):
    if name == "logu64":
        L = torch.exp(torch.rand(N // 20, generator=gen) * math.log(64)).long().clamp(1, 64)
    elif name == "uni20k":
        L = torch.randint(1000, 20001, (N // 10500,), generator=gen)
    elif name == "logu17":
        L = torch.exp(torch.rand(N // 9000, generator=gen) * math.log(1 << 17)).long().clamp(1, 1 << 17)
    elif name == "vocab":
        L = torch.full((N // 151_936,), 151_936)
    else:
        L = torch.tensor([N])
    c = torch.cumsum(L, 0)
    L = L[: int((c <= N).sum())]
    return L


def keys(dtype, n, gen):
    if dtype == torch.int64:
        return torch.randint(-(1 << 62), 1 << 62, (n,), generator=gen, device="cuda", dtype=torch.int64)
    x = (torch.randn(n, generator=gen, device="cuda") * 3).to(dtype)
    return torch.where(x == 0, torch.ones_like(x), x)


def query_ranks(lengths, query):
    last = (lengths - 1).clamp(min=0)
    if query == "median":
        return (last // 2)[:, None]
    q = torch.tensor(QS, dtype=torch.float32, device=lengths.device)
    pos = q[None, :] * last.float()[:, None]
    r = torch.cat([pos.long(), pos.ceil().long(), torch.zeros_like(last)[:, None], last[:, None]], 1)
    return torch.sort(r, dim=1)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--only", default="logu64,uni20k,logu17,vocab,one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("select_segments_timing.py needs a CUDA device: there is nothing to time on the CPU")
    out = {"tool": "select_segments_timing", **card(), "runs": args.runs, "results": []}
    for wname in args.only.split(","):
        gen = torch.Generator().manual_seed(len(wname))
        lengths = lengths_for(wname, gen).cuda()
        off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), torch.cumsum(lengths, 0)])
        n, S, max_len = int(off[-1]), lengths.numel(), int(lengths.max())
        seg = torch.repeat_interleave(torch.arange(S, device="cuda"), lengths)
        for tname, dtype in DTYPES.items():
            x = keys(dtype, n, torch.Generator(device="cuda").manual_seed(7))
            for query in ("median", "quantile"):
                rk = query_ranks(lengths, query)
                rk32 = rk.to(torch.int32)
                flat = (off[:-1, None] + rk).clamp(max=max(n - 1, 0))

                def select():
                    return g.select_segments(x, off, rk32, True, max_len)

                def lib_sort():
                    v, i = g.sort_long_segments(x, off, max_segment_len=max_len)
                    return v[flat], i[flat]

                def torch_composite():
                    o1 = torch.sort(x, stable=True)[1]
                    o2 = torch.sort(seg[o1], stable=True)[1]
                    perm = o1[o2]
                    return x[perm][flat], (perm[flat] - off[:-1, None]).to(torch.int32)

                arms = {"select": select, "lib_sort": lib_sort, "torch": torch_composite}
                if query == "quantile" and tname == "f32" and S <= 512:
                    xs = [x[int(off[s]):int(off[s + 1])] for s in range(S)]
                    qt = torch.tensor(QS, device="cuda")
                    arms["quantile_segments"] = lambda: g.quantile_segments(x, off, QS, max_segment_len=max_len)
                    arms["torch_q"] = lambda: torch.stack([torch.quantile(s_, qt) if s_.numel() <= 1 << 24 else qt for s_ in xs], 1)
                ib = {2: torch.int16, 4: torch.int32, 8: torch.int64}[x.element_size()]
                ref = arms["select"]()
                agree = {}
                for a in ("lib_sort", "torch"):
                    o = arms[a]()
                    agree[a] = bool(torch.equal(ref[0].view(ib), o[0].view(ib)) and torch.equal(ref[1], o[1]))
                if "torch_q" in arms and max_len <= 1 << 24:
                    qa, qb = arms["quantile_segments"](), arms["torch_q"]()
                    agree["torch_q"] = bool(torch.equal(qa, qb))
                times = {a: [] for a in arms if a != "torch_q" or max_len <= 1 << 24}
                for _ in range(args.warmup):
                    for a in times:
                        arms[a]()
                for _ in range(args.runs):
                    for a in times:
                        times[a].append(timed(arms[a])[0])
                med = {a: statistics.median(v) for a, v in times.items()}
                out["results"].append({"workload": wname, "dtype": tname, "query": query, "n": n, "segments": S,
                                       "max_len": max_len, "ms": {a: round(v, 4) for a, v in med.items()},
                                       "vs_lib_sort": round(med["lib_sort"] / med["select"], 3),
                                       "vs_torch": round(med["torch"] / med["select"], 3), "agree": agree})
                del rk, rk32, flat
            del x
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
