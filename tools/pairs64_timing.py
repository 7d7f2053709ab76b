"""64-bit keys with uint32 payloads (a (8, 4) sorter, osb200_create_pairs64) at 2^30 keys: one JSON line.

Arms, timed alternately with CUDA events, one call per sample:
  argsort    OneSweepSorter.argsort(keys): input untouched, sorted keys and int32 indices out
  torch      torch.sort(keys, stable=True): sorted keys and int64 indices
  pairs      sort_pairs_typed on keys and payloads already in place (the copy and iota untimed)
  keys       sort_keys_typed on a copy of the same keys (the u64 keys-only path, the floor; the copy untimed)
Workloads: uniform int64 keys, int64 keys below 2^20 (the passes of the upper five bytes are skipped: 3 of 8 execute) and
normal float64 keys (torch.randn).  The keys and indices of argsort and torch are compared element by element (the inputs
hold no NaN and no -0.0, so the two orders agree).  The card's name, power limit and maximum SM clock are read with
nvidia-smi (a read-only query) and printed with the times.

  python tools/pairs64_timing.py [--log2n 30] [--warmup 3] [--runs 10] [--arms argsort,torch,pairs,keys]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

# at 2^30 int64 keys the torch arm's scratch (~40 GB) and the other arms' buffers share the 80 GB: segments that grow
# in place keep the caching allocator from fragmenting between the arms
os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402

WORKLOADS = (("uniform_i64", "i64"), ("small_i64_lt_2p20", "i64"), ("normal_f64", "f64"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 and q.stdout.strip() else ""
    name, power, clock = ([x.strip() for x in line.split(",")] + ["", "", ""])[:3]
    return {"gpu": name or torch.cuda.get_device_name(), "power_limit": power or "unknown", "max_sm_clock": clock or "unknown"}


def timed(fn, prep=None):
    if prep is not None:
        prep()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), r


def make_keys(wl, n):
    gen = torch.Generator(device="cuda").manual_seed(64)
    if wl == "uniform_i64":
        return torch.randint(-(1 << 63), (1 << 63) - 1, (n,), dtype=torch.int64, device="cuda", generator=gen)
    if wl == "small_i64_lt_2p20":
        return torch.randint(0, 1 << 20, (n,), dtype=torch.int64, device="cuda", generator=gen)
    return torch.randn(n, dtype=torch.float64, device="cuda", generator=gen)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--arms", default="argsort,torch,pairs,keys")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pairs64_timing needs a CUDA device")
    want = args.arms.split(",")
    n = 1 << args.log2n
    s = g.OneSweepSorter(n, 8, 4)
    result = {"metric": "pairs64_ms", "n": n, "runs": args.runs, **card(), "tile_keys": s.info("tile_keys"), "workloads": {}}
    try:
        for wl, key_type in WORKLOADS:
            src = make_keys(wl, n)
            entry = {}
            # the cross-check holds both results; torch.sort's scratch is released before the argsort runs
            if "argsort" in want and "torch" in want:
                kt, it = torch.sort(src, stable=True)
                torch.cuda.empty_cache()
                ka, ia = s.argsort(src, key_type)
                entry["executed_passes"] = s.info("last_executed_passes")
                entry["outputs_identical"] = bool(torch.equal(ka, kt) and torch.equal(ia.long() & 0xFFFFFFFF, it))
                del kt, it, ka, ia
                torch.cuda.empty_cache()
            k2 = torch.empty_like(src)
            v2 = torch.empty(n, dtype=torch.int32, device="cuda")

            def prep_pairs():
                k2.copy_(src)
                torch.arange(n, dtype=torch.int32, device="cuda", out=v2)

            arms = {
                "argsort": (lambda: s.argsort(src, key_type), None),
                "torch": (lambda: torch.sort(src, stable=True), None),
                "pairs": (lambda: s.sort_pairs_typed(k2, v2, key_type), prep_pairs),
                "keys": (lambda: s.sort_keys_typed(k2, key_type), lambda: k2.copy_(src)),
            }
            arms = {a: arms[a] for a in want}
            if "argsort" in arms and "executed_passes" not in entry:
                s.argsort(src, key_type)
                entry["executed_passes"] = s.info("last_executed_passes")
            times = {a: [] for a in arms}
            for rep in range(args.warmup + args.runs):
                for a, (fn, prep) in arms.items():
                    ms, r = timed(fn, prep)
                    del r
                    if rep >= args.warmup:
                        times[a].append(ms)
            med = {a: statistics.median(t) for a, t in times.items()}
            entry["median_ms"] = {a: round(v, 3) for a, v in med.items()}
            entry["min_ms"] = {a: round(min(t), 3) for a, t in times.items()}
            entry["max_ms"] = {a: round(max(t), 3) for a, t in times.items()}
            if "argsort" in med and "torch" in med:
                entry["argsort_speedup_over_torch"] = round(med["torch"] / med["argsort"], 3)
            result["workloads"][wl] = entry
            del src, k2, v2
            torch.cuda.empty_cache()
    finally:
        s.close()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
