"""16-bit key sorts against the routes a caller has without them, at 2^30 keys: one JSON line.

Arms, timed alternately with CUDA events, one call per sample (the median of --runs samples after --warmup):
  keys16        sort_keys16(keys) in place (the copy of the input into the buffer untimed)
  keys_f32      x.float() -> sort_keys_typed("f32") -> .to(dtype): the conversion route through the 32-bit sort
  keys_torch    torch.sort(x, stable=True) values
  argsort16     argsort16(x): sorted keys and int32 indices, input untouched
  argsort_f32   argsort(x.float(), "f32"), keys converted back with .to(dtype)
  argsort_torch torch.sort(x, stable=True) values and indices
Workloads: normal-distributed bfloat16 and float16 (torch.randn) and uniform int16.  The outputs of keys16 and keys_f32,
and of argsort16 and argsort_f32, are compared bit for bit.  Per-kernel milliseconds of one profiled call of each 16-bit
and 32-bit sort follow ([hist, scan, pass0, pass1, ...], option "profile").  The card's name, power limit and SM clocks are
read with nvidia-smi (a read-only query) in the same call and printed with the times.

  python tools/keys16_timing.py [--log2n 30] [--warmup 3] [--runs 10]"""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 and q.stdout.strip() else ""
    name, power, clock, cur = ([x.strip() for x in line.split(",")] + ["", "", "", ""])[:4]
    return {"gpu": name or torch.cuda.get_device_name(), "power_limit": power or "unknown",
            "max_sm_clock": clock or "unknown", "sm_clock_at_start": cur or "unknown"}


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


def bits(t):
    return t.view(torch.int16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("keys16_timing needs a CUDA device")
    n = 1 << args.log2n
    result = {"metric": "keys16_ms", "n": n, "runs": args.runs, **card(), "workloads": {}}
    s = g.OneSweepSorter(n, 4, 4)
    try:
        for wl, key_type, dtype in (("normal_bf16", "bf16", torch.bfloat16), ("normal_f16", "f16", torch.float16),
                                    ("uniform_i16", "i16", torch.int16)):
            gen = torch.Generator(device="cuda").manual_seed(16)
            if dtype == torch.int16:
                src = torch.randint(-(1 << 15), 1 << 15, (n,), dtype=torch.int16, device="cuda", generator=gen)
            else:
                src = torch.randn(n, device="cuda", generator=gen).to(dtype)
            buf = torch.empty_like(src)

            def prep():
                buf.copy_(src)

            def keys16():
                return s.sort_keys16(buf, key_type)

            def keys_f32():
                f = src.float()
                s.sort_keys_typed(f, "f32")
                return f.to(dtype)

            def keys_torch():
                return torch.sort(src, stable=True)[0]

            def argsort16():
                return s.argsort16(src, key_type)

            def argsort_f32():
                k, i = s.argsort(src.float(), "f32")
                return k.to(dtype), i

            def argsort_torch():
                return torch.sort(src, stable=True)

            arms = {"keys16": (keys16, prep), "keys_f32": (keys_f32, None), "keys_torch": (keys_torch, None),
                    "argsort16": (argsort16, None), "argsort_f32": (argsort_f32, None), "argsort_torch": (argsort_torch, None)}
            prep()
            a, b = keys16(), keys_f32()
            torch.cuda.synchronize()
            keys_identical = bool(torch.equal(bits(a), bits(b)))
            del a, b
            (ka, ia), (kb, ib) = argsort16(), argsort_f32()
            torch.cuda.synchronize()
            argsort_identical = bool(torch.equal(bits(ka), bits(kb)) and torch.equal(ia, ib))
            del ka, ia, kb, ib
            torch.cuda.empty_cache()
            times = {a: [] for a in arms}
            for rep in range(args.warmup + args.runs):
                for a, (fn, p) in arms.items():
                    ms, r = timed(fn, p)
                    del r
                    if rep >= args.warmup:
                        times[a].append(ms)
            med = {a: statistics.median(t) for a, t in times.items()}
            # per-kernel times of one call each, profiled after the timed samples
            s.set_option("profile", 1)
            prof = {}
            prep()
            keys16()
            prof["keys16"] = [round(x, 3) for x in s.last_profile()]
            r = argsort16()
            prof["argsort16"] = [round(x, 3) for x in s.last_profile()]
            del r
            f = src.float()
            s.sort_keys_typed(f, "f32")
            prof["keys_f32_sort"] = [round(x, 3) for x in s.last_profile()]
            r = s.argsort(f, "f32")
            prof["argsort_f32_sort"] = [round(x, 3) for x in s.last_profile()]
            del r, f
            s.set_option("profile", 0)
            result["workloads"][wl] = {
                "outputs_identical": {"keys16_vs_f32": keys_identical, "argsort16_vs_f32": argsort_identical},
                "median_ms": {a: round(v, 3) for a, v in med.items()},
                "min_ms": {a: round(min(t), 3) for a, t in times.items()},
                "max_ms": {a: round(max(t), 3) for a, t in times.items()},
                "keys16_speedup_over_f32": round(med["keys_f32"] / med["keys16"], 3),
                "keys16_speedup_over_torch": round(med["keys_torch"] / med["keys16"], 3),
                "argsort16_speedup_over_f32": round(med["argsort_f32"] / med["argsort16"], 3),
                "argsort16_speedup_over_torch": round(med["argsort_torch"] / med["argsort16"], 3),
                "profile_ms": prof,
            }
            del src, buf
            torch.cuda.empty_cache()
    finally:
        s.close()
    result["sm_clock_at_end"] = card()["sm_clock_at_start"]
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
