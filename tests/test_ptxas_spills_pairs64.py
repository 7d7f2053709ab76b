"""CPU check of the compiled hot path of 64-bit keys with uint32 payloads (osb200_create_pairs64): the DigitBinningPass
instantiations for uint64_t keys with payloads (pairs and argsort, each plain and HOT) and the single-block sort's uint64_t
pairs and indices instantiations (the small path, not the row sort) must appear in the ptxas report of osb_kernels.cu and
must not spill registers to local memory in the default (atomic) rank mode.  uint64_t mangles as `m`.
The test reads the report of the library as built; it skips when there is none or it is older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# digit_binning_wide_kernel<uint64_t, PAIRS = true, K, WARPS, RANK_MODE, LOOK, MINB, HOT, INDICES>
WIDE64 = re.compile(r"_ZN3osb25digit_binning_wide_kernelImLb1ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])E")
# segment_sort_kernel<uint64_t, PAIRS = true, K, WARPS, RANK_MODE, INDICES, ROWS = false>
SEG64 = re.compile(r"_ZN3osb19segment_sort_kernelImLb1ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb0EE")
RANK_ATOMIC = 0


def guarded64(report):
    """{what: (spill stores, spill loads)} of the atomic-mode 64-bit pairs instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        w = WIDE64.match(name)
        if w and int(w.group(3)) == RANK_ATOMIC:
            out["u64/" + ("argsort" if w.group(7) == "1" else "pairs") + ("/hot" if w.group(6) == "1" else "")] = (st, ld)
        s = SEG64.match(name)
        if s and int(s.group(3)) == RANK_ATOMIC:
            keys = int(s.group(1)) * int(s.group(2)) * 32
            out[f"small/u64/{keys}/" + ("indices" if s.group(4) == "1" else "pairs")] = (st, ld)
    return out


def test_the_regex_reads_the_uint64_pairs_mangling():
    text = ("ptxas info    : Function properties for "
            "_ZN3osb25digit_binning_wide_kernelImLb1ELi8ELi16ELi0ELi32ELi2ELb1ELb1EEEvPT_S2_PjS3_mPKyPtPmS3_NS_10PassParamsENS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for "
            "_ZN3osb25digit_binning_wide_kernelImLb0ELi16ELi16ELi0ELi32ELi2ELb0ELb0EEEvPT_S2_PjS3_mPKyPtPmS3_NS_10PassParamsENS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for "
            "_ZN3osb19segment_sort_kernelImLb1ELi16ELi16ELi0ELb0ELb0EEEvPT_PjPKymmjjjjNS_8KeyCodecEPKS1_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for "
            "_ZN3osb19segment_sort_kernelImLb1ELi16ELi16ELi0ELb1ELb1EEEvPT_PjPKymmjjjjNS_8KeyCodecEPKS1_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded64(parse_report(text)) == {"u64/argsort/hot": (4, 8), "small/u64/8192/pairs": (0, 0)}


def test_pairs64_instantiations_do_not_spill():
    got = guarded64(_report())
    want = {f"u64/{k}{h}" for k in ("pairs", "argsort") for h in ("", "/hot")}
    want |= {f"small/u64/8192/{m}" for m in ("pairs", "indices")}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills on the 64-bit pairs hot path:\n" + "\n".join(spilling)
