"""argsort against what a caller composes without it, at 2^30 keys: one JSON line.

Arms, timed alternately with CUDA events, one call per sample:
  argsort   OneSweepSorter.argsort(keys): input untouched, sorted keys and int32 indices out
  composed  keys.clone() + torch.arange(n) + sort_pairs_typed on the copy (what a caller needs for the same result)
  pairs     sort_pairs / sort_pairs_typed on keys and payloads already in place (the copy and iota untimed)
Workloads: uniform uint32 keys (the reference generator, entropy preset 1) and normal float32 keys (torch.randn).
The outputs of the first two arms are compared bit for bit.  The card's name, power limit and maximum SM clock are read
with nvidia-smi (a read-only query) and printed with the times.

  python tools/argsort_timing.py [--log2n 30] [--warmup 3] [--runs 20]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("argsort_timing needs a CUDA device")
    n = 1 << args.log2n
    result = {"metric": "argsort_ms", "n": n, "runs": args.runs, **card(), "workloads": {}}
    s = g.OneSweepSorter(n, 4, 4)
    try:
        for wl, key_type in (("uniform_u32", "u32"), ("normal_f32", "f32")):
            if key_type == "u32":
                src = torch.empty(n, dtype=torch.int32, device="cuda")
                g.init_random(src, 0, 30)
            else:
                gen = torch.Generator(device="cuda").manual_seed(30)
                src = torch.randn(n, dtype=torch.float32, device="cuda", generator=gen)
            k2 = torch.empty_like(src)
            v2 = torch.empty(n, dtype=torch.int32, device="cuda")

            def arm_argsort():
                return s.argsort(src, key_type)

            def arm_composed():
                k = src.clone()
                v = torch.arange(n, dtype=torch.int32, device="cuda")
                s.sort_pairs_typed(k, v, key_type)
                return k, v

            def prep_pairs():
                k2.copy_(src)
                torch.arange(n, dtype=torch.int32, device="cuda", out=v2)

            def arm_pairs():
                if key_type == "u32":
                    s.sort_pairs(k2, v2)
                else:
                    s.sort_pairs_typed(k2, v2, key_type)

            arms = {"argsort": (arm_argsort, None), "composed": (arm_composed, None), "pairs": (arm_pairs, prep_pairs)}
            # outputs of the two ways to the same result, compared bit for bit
            (ka, ia), (kc, ic) = arm_argsort(), arm_composed()
            torch.cuda.synchronize()
            identical = bool(torch.equal(ka.view(torch.int32), kc.view(torch.int32)) and torch.equal(ia, ic))
            del ka, ia, kc, ic
            times = {a: [] for a in arms}
            for rep in range(args.warmup + args.runs):
                for a, (fn, prep) in arms.items():
                    ms, r = timed(fn, prep)
                    del r
                    if rep >= args.warmup:
                        times[a].append(ms)
            med = {a: statistics.median(t) for a, t in times.items()}
            result["workloads"][wl] = {
                "outputs_identical": identical,
                "median_ms": {a: round(v, 3) for a, v in med.items()},
                "min_ms": {a: round(min(t), 3) for a, t in times.items()},
                "max_ms": {a: round(max(t), 3) for a, t in times.items()},
                "argsort_over_composed": round(med["argsort"] / med["composed"], 3),
                "argsort_over_pairs": round(med["argsort"] / med["pairs"], 3),
            }
            del src, k2, v2
            torch.cuda.empty_cache()
    finally:
        s.close()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
