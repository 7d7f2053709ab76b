"""CPU check of the long-segment sort's compiled kernels (osb200_sort_long_segments): the long bin kernel, the tile map, the
count, the three scan kernels, the scatter (both rank modes, keys only and with indices) and the copy home, for 16-, 32- and
64-bit keys where the kernel is per key width, must appear in the ptxas report of osb_kernels.cu, and none may spill
registers to local memory in the default (atomic) rank mode.  uint16_t mangles as `t`, uint32_t as `j`, uint64_t as `m`.
The test reads the report of the library as built; it skips when there is none or it is older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# long_scatter_kernel<KeyT, RANK_MODE, INDICES, LongSegGeo, false>
SCATTER = re.compile(r"_ZN3osb19long_scatter_kernelI([tjm])Li(\d+)ELb([01])ENS_10LongSegGeoELb0EEE")
# long_count_kernel<KeyT, LongSegGeo>
COUNT = re.compile(r"_ZN3osb17long_count_kernelI([tjm])NS_10LongSegGeoEEE")
# long_segments_copy_home_kernel<KeyT>, long_segment_bin_kernel<KeyT>
PER_KEY = re.compile(r"_ZN3osb\d+long_(segments_copy_home|segment_bin)_kernelI([tjm])EE")
# long_{chunk_sum,chunk_scan,scan}_kernel<LongSegGeo>, long_segments_map_kernel
SCAN = re.compile(r"_ZN3osb\d+long_(chunk_sum|chunk_scan|scan)_kernelINS_10LongSegGeoEEE")
MAP = re.compile(r"_ZN3osb24long_segments_map_kernelE")
WIDTH = {"t": "u16", "j": "u32", "m": "u64"}
RANK_ATOMIC = 0


def guarded_long_segments(report):
    """{what: (spill stores, spill loads)} of the atomic-mode long-segment instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        m = SCATTER.match(name)
        if m and int(m.group(2)) == RANK_ATOMIC:
            out[f"scatter/{WIDTH[m.group(1)]}/" + ("indices" if m.group(3) == "1" else "keys")] = (st, ld)
        m = COUNT.match(name)
        if m:
            out[f"count/{WIDTH[m.group(1)]}"] = (st, ld)
        m = PER_KEY.match(name)
        if m:
            out[f"{m.group(1).replace('segments_', '')}/{WIDTH[m.group(2)]}"] = (st, ld)
        m = SCAN.match(name)
        if m:
            out[m.group(1)] = (st, ld)
        if MAP.match(name):
            out["map"] = (st, ld)
    return out


def test_the_regex_reads_the_long_segment_kernels_mangling():
    text = ("ptxas info    : Function properties for _ZN3osb19long_scatter_kernelImLi0ELb1ENS_10LongSegGeoELb0EEEvPKNS_8SortPlanEjPKT_PS5_S8_PjS9_T2_PKjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb19long_scatter_kernelImLi1ELb1ENS_10LongSegGeoELb0EEEvPKNS_8SortPlanEjPKT_PS5_S8_PjS9_T2_PKjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb17long_count_kernelItNS_10LongSegGeoEEEvPKNS_8SortPlanEjPKT_S7_S7_T0_PjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb23long_segment_bin_kernelIjEEvPKymmjPjPyPKT_PS5_S3_jS3_m\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb24long_segments_map_kernelEPKyPKjPjS4_Pymmm\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb26long_rows_copy_home_kernelIjEEvPKNS_8SortPlanEPKT_S6_PS4_PKjPjmj\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded_long_segments(parse_report(text)) == {"scatter/u64/indices": (4, 8), "count/u16": (0, 0), "segment_bin/u32": (0, 0),
                                                         "map": (0, 0)}


def test_long_segment_instantiations_do_not_spill():
    got = guarded_long_segments(_report())
    want = {f"scatter/{w}/{m}" for w in WIDTH.values() for m in ("keys", "indices")}
    want |= {f"{k}/{w}" for k in ("count", "copy_home", "segment_bin") for w in WIDTH.values()}
    want |= {"chunk_sum", "chunk_scan", "scan", "map"}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills in the long-segment sort:\n" + "\n".join(spilling)
