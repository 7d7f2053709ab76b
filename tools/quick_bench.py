"""Development timing script (not the contract bench): per-configuration sort time, per-kernel split and the
reference's CUDA OneSweep (oracle/_ref) on the same input.  Usage: python tools/quick_bench.py [log2n ...]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gpusorting_b200 as g  # noqa: E402
from tests import oraclelib  # noqa: E402

PEAK = 3350.0  # GB/s, H100 SXM data sheet (not a measured figure)
REPS = int(os.environ.get("OSB_REPS", "5"))


def time_ms(fn, reps=REPS, prep=None):
    best = []
    for _ in range(reps):
        if prep:
            prep()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best.append(a.elapsed_time(b))
    best.sort()
    return best[len(best) // 2], best[0]


def main():
    exps = [int(x) for x in sys.argv[1:]] or [28, 30]
    ref = oraclelib.load_ref()
    for e in exps:
        n = 1 << e
        src = torch.empty(n, dtype=torch.int32, device="cuda")
        g.init_random(src, 0, 10)
        work = torch.empty_like(src)
        s = g.OneSweepSorter(n, 4, 0)
        VARIANTS = [int(x) for x in os.environ.get("OSB_VARIANTS", "0,1,2").split(",")]
        MODES = [int(x) for x in os.environ.get("OSB_MODES", "0").split(",")]
        hist_ms, _ = time_ms(lambda: s.global_histogram(src))
        print(f"n=2^{e} global_histogram(+memset) {hist_ms:.3f} ms ({4*n/hist_ms/1e6:.0f} GB/s read)", flush=True)
        dst = torch.empty_like(src)
        for variant in VARIANTS:
            s.set_option("variant", variant)
            for mode in MODES:
                s.set_option("rank_mode", mode)
                med, best = time_ms(lambda: s.sort_keys(work), prep=lambda: work.copy_(src))
                print(f"n=2^{e} keys u32 variant={variant} rank_mode={mode}: median {med:.3f} ms best {best:.3f} ms -> {n/med/1e6:.1f} Gkeys/s, "
                      f"{32*n/med/1e6/PEAK*100:.1f}% of {PEAK} GB/s (32 B/key)", flush=True)
            s.set_option("rank_mode", 0)
            for shift in (0, 24):
                pass_ms, _ = time_ms(lambda: s.digit_binning_pass(src, dst, shift))
                print(f"   variant={variant} shift={shift}: hist+scan+one pass {pass_ms:.3f} ms => pass ~{pass_ms-hist_ms:.3f} ms "
                      f"({8*n/(pass_ms-hist_ms)/1e6:.0f} GB/s r+w)", flush=True)
        assert s.validate(work) == 0
        s.close()
        del dst
        if ref is not None and e <= 30:
            h = ref.lib.ref_create(n)
            alt = torch.empty_like(src)
            med, best = time_ms(lambda: ref.lib.ref_sort_keys(h, work.data_ptr(), alt.data_ptr(), n), prep=lambda: work.copy_(src))
            print(f"n=2^{e} REFERENCE CUDA OneSweep (sm_90a build): median {med:.3f} ms best {best:.3f} -> {n/med/1e6:.1f} Gkeys/s", flush=True)
            ref.lib.ref_destroy(h)
            del alt
        if os.environ.get("OSB_SKIP_PAIRS", "0") in ("", "0"):
            sp = g.OneSweepSorter(n, 4, 4)
            sp.set_option("profile", 1)
            v, vw = torch.arange(n, dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")
            med, best = time_ms(lambda: sp.sort_pairs(work, vw), prep=lambda: (work.copy_(src), vw.copy_(v)))
            pr = sp.last_profile()
            print(f"n=2^{e} pairs u32/u32: median {med:.3f} ms -> {n/med/1e6:.1f} Gpairs/s, {64*n/med/1e6/PEAK*100:.1f}% (64 B/pair); "
                  f"hist {pr[0]:.3f} ms, pass {sum(pr[2:])/len(pr[2:]):.3f} ms ({16*n/(sum(pr[2:])/len(pr[2:]))/1e6:.0f} GB/s)", flush=True)
            assert sp.validate(work) == 0
            sp.close()
            del v, vw
            torch.cuda.empty_cache()
            s8 = g.OneSweepSorter(n, 8, 0)
            s8.set_option("profile", 1)
            w8 = torch.empty(2 * n, dtype=torch.int32, device="cuda")
            g.init_random(w8, 0, 10)
            src8 = w8.view(torch.int64)
            work8 = torch.empty_like(src8)
            med, best = time_ms(lambda: s8.sort_keys(work8), prep=lambda: work8.copy_(src8))
            pr = s8.last_profile()
            print(f"n=2^{e} keys u64: median {med:.3f} ms -> {n/med/1e6:.1f} Gkeys/s, {128*n/med/1e6/PEAK*100:.1f}% (128 B/key); "
                  f"hist {pr[0]:.3f} ms, pass {sum(pr[2:])/len(pr[2:]):.3f} ms ({16*n/(sum(pr[2:])/len(pr[2:]))/1e6:.0f} GB/s)", flush=True)
            assert s8.validate(work8) == 0
            s8.close()
            del w8, src8, work8
        del src, work
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
