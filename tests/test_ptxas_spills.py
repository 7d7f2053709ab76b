"""CPU check of the compiled hot path: the DigitBinningPass in its default (atomic) rank mode and the GlobalHistogram must
not spill registers to local memory on sm_90a.

The Makefile keeps ptxas's `-v` report of osb_kernels.cu in gpusorting_b200/csrc/build/osb_kernels.ptxas.log.  A spill
there does not change any result, so no GPU test notices it, but on the H100 it puts local-memory round trips in front
of the pass's shared-memory atomics.  The test reads the report of the library as built; it skips when there is none."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gpusorting_b200", "csrc")
LOG = os.path.join(CSRC, "build", "osb_kernels.ptxas.log")
# what the Makefile rebuilds osb_kernels.o (and so the report) from
SOURCES = [os.path.join(CSRC, f) for f in ("osb_kernels.cu", "osb_common.cuh", "osb_kernels.cuh", "osb_internal.h")] + [
    os.path.join(ROOT, "include", "onesweep_b200.h")]

PROPS = re.compile(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
# digit_binning_wide_kernel<KeyT, PAIRS, K, WARPS, RANK_MODE, LOOK, MINB, HOT>
WIDE = re.compile(r"_ZN3osb25digit_binning_wide_kernelI([jm])Lb([01])ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])E")
HIST = re.compile(r"_ZN3osb23global_histogram_kernelI([jm])Lb([01])E")
RANK_ATOMIC = 0


def _report():
    if not os.path.exists(LOG):
        pytest.skip(f"{os.path.relpath(LOG, ROOT)} not found: build the library first (make -C gpusorting_b200/csrc)")
    newer = [os.path.relpath(f, ROOT) for f in SOURCES if os.path.getmtime(f) > os.path.getmtime(LOG)]
    if newer:
        pytest.skip(f"the ptxas report is older than {', '.join(newer)}: rebuild the library first")
    with open(LOG) as f:
        return parse_report(f.read())


def parse_report(text):
    """[(mangled name, spill store bytes, spill load bytes)] of every function ptxas reported."""
    return [(m.group(1), int(m.group(3)), int(m.group(4))) for m in PROPS.finditer(text)]


def test_parse_report_reads_ptxas_format():
    text = ("ptxas info    : Compiling entry function '_ZN3osb1kEv' for 'sm_90a'\n"
            "ptxas info    : Function properties for _ZN3osb1kEv\n"
            "    88 bytes stack frame, 88 bytes spill stores, 92 bytes spill loads\n"
            "ptxas info    : Used 64 registers, used 1 barriers, 88 bytes cumulative stack size\n")
    assert parse_report(text) == [("_ZN3osb1kEv", 88, 92)]


def test_hot_path_instantiations_do_not_spill():
    report = _report()
    guarded, seen = [], set()
    for name, st, ld in report:
        w = WIDE.match(name)
        if w and int(w.group(5)) == RANK_ATOMIC:
            key = ("u64" if w.group(1) == "m" else "u32") + ("/pairs" if w.group(2) == "1" else "/keys") + ("/hot" if w.group(8) == "1" else "")
            seen.add(key)
            guarded.append((f"digit_binning_wide_kernel {key}", st, ld))
        elif HIST.match(name):
            seen.add("global_histogram")
            guarded.append((f"global_histogram_kernel {name}", st, ld))
    want = {"u32/keys", "u32/keys/hot", "u32/pairs", "u32/pairs/hot", "u64/keys", "u64/keys/hot", "global_histogram"}
    assert want <= seen, f"instantiations missing from the ptxas report: {sorted(want - seen)}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, st, ld in guarded if st or ld]
    assert not spilling, "register spills on the hot path:\n" + "\n".join(spilling)
