"""CPU check of the fused first pass (DESIGN §4.12): its instantiation of digit_binning_wide_kernel in the default (atomic)
rank mode must not spill registers to local memory on sm_90a.  (The plain and HOT u32 keys passes, which read the gapped
source, are guarded by tests/test_ptxas_spills.py.)  Reads the ptxas report the Makefile keeps; skips when there is none."""
import re

from tests.test_ptxas_spills import _report

# digit_binning_wide_kernel<uint32_t, false, K, WARPS, RANK_MODE, LOOK, MINB, HOT = false, INDICES = false, FUSED = true>
FUSED = re.compile(r"_ZN3osb25digit_binning_wide_kernelIjLb0ELi\d+ELi\d+ELi(\d+)ELi\d+ELi\d+ELb0ELb0ELb1EE")


def test_fused_first_pass_does_not_spill():
    found = [(name, st, ld) for name, st, ld in _report() if (m := FUSED.match(name)) and m.group(1) == "0"]
    assert found, "the fused first pass (atomic rank mode) is missing from the ptxas report"
    spilling = [f"{name}: {st} B spill stores, {ld} B spill loads" for name, st, ld in found if st or ld]
    assert not spilling, "register spills in the fused first pass:\n" + "\n".join(spilling)
