"""CPU check of the segment top-k's compiled kernels (osb200_topk_segments): the binning kernel, the warp class
(topk_segment_warp_kernel), the radix select in list mode (topk_segment_select_kernel) and the in-place sorts of the selected
rows (topk_segment_sort_warp_kernel, 1, 2, 4 and 8 keys per lane; topk_segment_sort_kernel, the 2,048-key geometry and the
16,384-key one, 8,192 for 64-bit keys), for 16-, 32- and 64-bit keys, must appear in the ptxas report of osb_kernels.cu and
must not spill registers to local memory in the default (atomic) rank mode.  uint16_t mangles as `t`, uint32_t as `j`,
uint64_t as `m`.  The test reads the report of the library as built; it skips when there is none or it is older than the
sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

BIN = re.compile(r"_ZN3osb23topk_segment_bin_kernelE")
# topk_segment_warp_kernel<KeyT, RANK_MODE>
WARP = re.compile(r"_ZN3osb24topk_segment_warp_kernelI([tjm])Li(\d+)EE")
# topk_segment_select_kernel<KeyT>
SELECT = re.compile(r"_ZN3osb26topk_segment_select_kernelI([tjm])EE")
# topk_segment_sort_warp_kernel<KeyT, K, RANK_MODE>
SORT_WARP = re.compile(r"_ZN3osb29topk_segment_sort_warp_kernelI([tjm])Li(\d+)ELi(\d+)EE")
# topk_segment_sort_kernel<KeyT, K, WARPS, RANK_MODE>
SORT = re.compile(r"_ZN3osb24topk_segment_sort_kernelI([tjm])Li(\d+)ELi(\d+)ELi(\d+)EE")
WIDTH = {"t": "u16", "j": "u32", "m": "u64"}
RANK_ATOMIC = 0


def guarded_topk_segments(report):
    """{what: (spill stores, spill loads)} of the atomic-mode segment top-k instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        if BIN.match(name):
            out["bin"] = (st, ld)
        w = WARP.match(name)
        if w and int(w.group(2)) == RANK_ATOMIC:
            out[f"warp/{WIDTH[w.group(1)]}"] = (st, ld)
        s = SELECT.match(name)
        if s:
            out[f"select/{WIDTH[s.group(1)]}"] = (st, ld)
        sw = SORT_WARP.match(name)
        if sw and int(sw.group(3)) == RANK_ATOMIC:
            out[f"sort_warp/{WIDTH[sw.group(1)]}/K{sw.group(2)}"] = (st, ld)
        b = SORT.match(name)
        if b and int(b.group(4)) == RANK_ATOMIC:
            out[f"sort/{WIDTH[b.group(1)]}/{int(b.group(2)) * int(b.group(3)) * 32}"] = (st, ld)
    return out


def test_the_regex_reads_the_topk_segments_kernels_mangling():
    text = ("ptxas info    : Function properties for _ZN3osb23topk_segment_bin_kernelEPKymmjPjPy\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb24topk_segment_warp_kernelImLi0EEEvPKT_PS1_PjmPKyPKjS7_jNS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb24topk_segment_warp_kernelImLi1EEEvPKT_PS1_PjmPKyPKjS7_jNS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb26topk_segment_select_kernelItEEvPKT_PS1_PjmjjNS_8KeyCodecEPKyPKjS8_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb29topk_segment_sort_warp_kernelIjLi4ELi0EEEvPT_PjmjPKjPKyNS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb24topk_segment_sort_kernelIjLi32ELi16ELi0EEEvPT_PjmjNS_8KeyCodecEPKymj\n"
            "    0 bytes stack frame, 12 bytes spill stores, 12 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb24topk_segment_sort_kernelIjLi8ELi8ELi1EEEvPT_PjmjNS_8KeyCodecEPKymj\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded_topk_segments(parse_report(text)) == {"bin": (0, 0), "warp/u64": (4, 8), "select/u16": (0, 0),
                                                         "sort_warp/u32/K4": (0, 0), "sort/u32/16384": (12, 12)}


def test_topk_segments_instantiations_do_not_spill():
    got = guarded_topk_segments(_report())
    want = {"bin"} | {f"warp/{w}" for w in WIDTH.values()} | {f"select/{w}" for w in WIDTH.values()}
    want |= {f"sort_warp/{w}/K{k}" for w in WIDTH.values() for k in (1, 2, 4, 8)}
    want |= {f"sort/{w}/{t}" for w in WIDTH.values() for t in (2048, 8192 if w == "u64" else 16384)}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills in the segment top-k:\n" + "\n".join(spilling)
