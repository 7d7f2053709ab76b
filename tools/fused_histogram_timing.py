"""Fused against classic first pass (DESIGN §4.12), alternated in one process on the H100.

Inputs: 2^30 uniform uint32 keys (bench.py's workload), the entropy presets (AND of 2-6 random words), and a late-overflow
input (place-0 bin 7 gets c + 1 keys, all in the last tiles, so the fused pass aborts at its end and the fallback runs).
Each round sorts every input once with option fused_histogram 0 and once with 1, in alternating order; per input it prints
the mean sort time of each path, whether the fused result stood, and the per-entry profile of one extra sort
([histogram, scan, pass 0, pass 1, ...]; a fused sort reports its fused pass and the classic pass 0 in entry 2, and the
fallback's histogram in entry 0).  The card's name, power limit and SM clocks are printed with the results.

  python tools/fused_histogram_timing.py [--log2n 30] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timings stand without it
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import torch

    import gpusorting_b200 as g
    from tests.test_fused_layout_cpu import region_keys

    n = 1 << args.log2n
    c = region_keys(n)
    inputs = {}
    t = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(t, 0, 42)
    inputs["uniform"] = t
    for andc in (1, 2, 3, 4, 5):
        t = torch.empty(n, dtype=torch.int32, device="cuda")
        g.init_random(t, andc, 42)
        inputs[f"entropy_and{andc}"] = t
    late = inputs["uniform"].clone()
    low = late & 0xFF
    late = torch.where(low == 7, (late & ~0xFF) | ((late >> 8) & 0xFE), late)  # bin 7's keys to the even bins (+1/128 each)
    late[n - c - 1:] = (late[n - c - 1:] & ~0xFF) | 7  # c + 1 keys of bin 7, in the last tiles
    inputs["late_overflow"] = late

    s = g.OneSweepSorter(n, 4, 0)
    work = torch.empty(n, dtype=torch.int32, device="cuda")
    times = {name: {0: [], 1: []} for name in inputs}
    kept = {}
    print(json.dumps({"card_before": card()}), flush=True)
    for r in range(args.rounds + 1):  # round 0 warms up
        for name, src in inputs.items():
            for fused in ((0, 1) if r % 2 else (1, 0)):
                s.set_option("fused_histogram", fused)
                work.copy_(src)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                s.sort_keys(work)
                b.record()
                b.synchronize()
                if r:
                    times[name][fused].append(a.elapsed_time(b))
                if fused:
                    kept[name] = s.info("last_fused_kept")
    profiles = {}
    s.set_option("profile", 1)
    for name, src in inputs.items():
        for fused in (0, 1):
            s.set_option("fused_histogram", fused)
            work.copy_(src)
            s.sort_keys(work)
            profiles[f"{name}/{'fused' if fused else 'classic'}"] = [round(x, 4) for x in s.last_profile()]
    s.set_option("profile", 0)
    torch.cuda.synchronize()
    for name in inputs:
        m0 = sum(times[name][0]) / len(times[name][0])
        m1 = sum(times[name][1]) / len(times[name][1])
        print(json.dumps({"input": name, "n": n, "classic_ms": round(m0, 4), "fused_ms": round(m1, 4),
                          "gain_pct": round(100 * (m0 / m1 - 1), 2), "fused_kept": kept[name],
                          "classic_all": [round(x, 4) for x in times[name][0]], "fused_all": [round(x, 4) for x in times[name][1]],
                          "profile_classic": profiles[f"{name}/classic"], "profile_fused": profiles[f"{name}/fused"]}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)
    s.close()


if __name__ == "__main__":
    main()
