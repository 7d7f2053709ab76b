"""CPU check of the 16-bit key sorts' compiled hot path: the DigitBinningPass instantiations for uint16_t keys (keys, pairs
and argsort, each plain and HOT) and their GlobalHistogram must appear in the ptxas report of osb_kernels.cu and must not
spill registers to local memory in the default (atomic) rank mode.  uint16_t mangles as `t` (uint32_t `j`, uint64_t `m`).
The test reads the report of the library as built; it skips when there is none or it is older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# digit_binning_wide_kernel<uint16_t, PAIRS, K, WARPS, RANK_MODE, LOOK, MINB, HOT, INDICES>
WIDE16 = re.compile(r"_ZN3osb25digit_binning_wide_kernelItLb([01])ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])E")
HIST16 = re.compile(r"_ZN3osb23global_histogram_kernelItLb0E")
RANK_ATOMIC = 0


def guarded16(report):
    """{what: (spill stores, spill loads)} of the atomic-mode 16-bit instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        w = WIDE16.match(name)
        if w and int(w.group(4)) == RANK_ATOMIC:
            kind = "argsort" if w.group(8) == "1" else ("pairs" if w.group(1) == "1" else "keys")
            out[f"u16/{kind}" + ("/hot" if w.group(7) == "1" else "")] = (st, ld)
        elif HIST16.match(name):
            out["u16/global_histogram"] = (st, ld)
    return out


def test_the_regex_reads_the_uint16_mangling():
    text = ("ptxas info    : Function properties for "
            "_ZN3osb25digit_binning_wide_kernelItLb1ELi16ELi16ELi0ELi8ELi2ELb1ELb1EEEvPT_S2_PjS3_mPKyPtPmS3_NS_10PassParamsENS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n")
    assert guarded16(parse_report(text)) == {"u16/argsort/hot": (4, 8)}


def test_keys16_instantiations_do_not_spill():
    got = guarded16(_report())
    want = {f"u16/{k}{h}" for k in ("keys", "pairs", "argsort") for h in ("", "/hot")} | {"u16/global_histogram"}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills on the 16-bit hot path:\n" + "\n".join(spilling)
