"""CPU check of the segment select's compiled kernels (osb200_select_segments): the binning kernels, the warp and block
classes (both rank modes, values only and with positions) and the split path's count, pick, equal-key count, scan, locate
and padding kernels, for 16-, 32- and 64-bit keys, must appear in the ptxas report of osb_kernels.cu, and none may spill
registers to local memory or use a stack frame.  uint16_t mangles as `t`, uint32_t as `j`, uint64_t as `m`.  The test reads
the report of the library as built; it skips when there is none or it is older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# select_segment_warp_kernel<KeyT, RANK_MODE, INDICES>, select_segment_block_kernel<KeyT, K, WARPS, RANK_MODE, INDICES>
WARP = re.compile(r"_ZN3osb\d+select_segment_warp_kernelI([tjm])Li(\d+)ELb([01])EE")
BLOCK = re.compile(r"_ZN3osb\d+select_segment_block_kernelI([tjm])Li(\d+)ELi(\d+)ELi(\d+)ELb([01])EE")
# select_{count,pick,eq_count,locate}_kernel<KeyT, LongSegGeo>, select_segment_unmapped_kernel<KeyT>
SPLIT = re.compile(r"_ZN3osb\d+select_(count|pick|eq_count|locate)_kernelI([tjm])NS_10LongSegGeoEEE")
UNMAPPED = re.compile(r"_ZN3osb\d+select_(segment_unmapped)_kernelI([tjm])EE")
PLAIN = re.compile(r"_ZN3osb\d+(select_segment_bin|select_long_segment_bin)_kernelE")
# long_{chunk_sum,chunk_scan,scan}_kernel<SelectSegScanGeo>: the scan of the equal-key counts
SCAN = re.compile(r"_ZN3osb\d+long_(chunk_sum|chunk_scan|scan)_kernelINS_16SelectSegScanGeoEEE")
WIDTH = {"t": "u16", "j": "u32", "m": "u64"}


def guarded_select_segments(report):
    """{what: (spill stores, spill loads)} of the segment select's instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        m = WARP.match(name)
        if m:
            out[f"warp/{WIDTH[m.group(1)]}/rank{m.group(2)}/idx{m.group(3)}"] = (st, ld)
        m = BLOCK.match(name)
        if m:
            out[f"block/{WIDTH[m.group(1)]}/K{m.group(2)}/rank{m.group(4)}/idx{m.group(5)}"] = (st, ld)
        m = SPLIT.match(name) or UNMAPPED.match(name)
        if m:
            out[f"{m.group(1)}/{WIDTH[m.group(2)]}"] = (st, ld)
        m = PLAIN.match(name)
        if m:
            out[m.group(1)] = (st, ld)
        m = SCAN.match(name)
        if m:
            out[f"scan/{m.group(1)}"] = (st, ld)
    return out


def test_the_regex_reads_the_select_segments_mangling():
    text = ("ptxas info    : Function properties for _ZN3osb27select_segment_block_kernelIjLi32ELi16ELi1ELb1EEEvPKT_PS1_PjPKymjNS_8KeyCodecEPKjS8_SB_j\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb26select_segment_warp_kernelItLi0ELb0EEEvPKT_PS1_PjmjPKyPKjS8_SA_jNS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb22select_eq_count_kernelImNS_10LongSegGeoEEEvPKT_T0_PKjjPKNS_11SelectStateEPjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb16long_scan_kernelINS_16SelectSegScanGeoEEEvPKNS_8SortPlanEjPjPKjT_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded_select_segments(parse_report(text)) == {"block/u32/K32/rank1/idx1": (4, 8), "warp/u16/rank0/idx0": (0, 0),
                                                           "eq_count/u64": (0, 0), "scan/scan": (0, 0)}


def test_select_segments_instantiations_do_not_spill():
    got = guarded_select_segments(_report())
    want = {f"warp/{w}/rank{r}/idx{i}" for w in WIDTH.values() for r in (0, 1) for i in (0, 1)}
    want |= {f"block/{w}/K{k}/rank{r}/idx{i}" for w, ks in (("u16", (8, 32)), ("u32", (8, 32)), ("u64", (8, 16)))
             for k in ks for r in (0, 1) for i in (0, 1)}
    want |= {f"{k}/{w}" for k in ("count", "pick", "eq_count", "locate", "segment_unmapped") for w in WIDTH.values()}
    want |= {"select_segment_bin", "select_long_segment_bin", "scan/chunk_sum", "scan/chunk_scan", "scan/scan"}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills in the segment select:\n" + "\n".join(spilling)


def test_select_segments_kernels_have_no_stack_frame():
    import os

    from tests.test_ptxas_spills import LOG

    text = open(LOG).read() if os.path.exists(LOG) else ""
    kernels = (r"select_(?:segment|segments|long_segment)\w*|select_\w+_kernelI[tjm]NS_10LongSegGeo\w*|"
               r"long_\w+_kernelINS_16SelectSegScanGeo\w*")
    frames = re.findall(rf"Function properties for (_ZN3osb\d+(?:{kernels}))\n\s+(\d+) bytes stack frame", text)
    assert all(int(f) == 0 for _, f in frames), [n for n, f in frames if int(f)]
