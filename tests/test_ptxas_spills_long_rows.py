"""CPU check of the long-row sort's compiled kernels (osb200_sort_long_rows): the count, the three scan kernels, the scatter
(both rank modes, keys only and with indices), the copy home and the head of the histogram, for 16-, 32- and 64-bit keys,
must appear in the ptxas report of osb_kernels.cu, and none may spill registers to local memory in the default (atomic)
rank mode.  uint16_t mangles as `t`, uint32_t as `j`, uint64_t as `m`.  The test reads the report of the library as
built; it skips when there is none or it is older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# long_scatter_kernel<KeyT, RANK_MODE, INDICES, LongRowGeo, false>
SCATTER = re.compile(r"_ZN3osb19long_scatter_kernelI([tjm])Li(\d+)ELb([01])ENS_10LongRowGeoELb0EEE")
# long_count_kernel<KeyT, LongRowGeo>
COUNT = re.compile(r"_ZN3osb17long_count_kernelI([tjm])NS_10LongRowGeoEEE")
# long_rows_copy_home_kernel<KeyT>, long_rows_head_hist_kernel<KeyT>
PER_KEY = re.compile(r"_ZN3osb\d+long_rows_(copy_home|head_hist)_kernelI([tjm])EE")
# long_{chunk_sum,chunk_scan,scan}_kernel<LongRowGeo>
SCAN = re.compile(r"_ZN3osb\d+long_(chunk_sum|chunk_scan|scan)_kernelINS_10LongRowGeoEEE")
WIDTH = {"t": "u16", "j": "u32", "m": "u64"}
RANK_ATOMIC = 0


def guarded_long_rows(report):
    """{what: (spill stores, spill loads)} of the atomic-mode long-row instantiations in a parsed report"""
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
            out[f"{m.group(1)}/{WIDTH[m.group(2)]}"] = (st, ld)
        m = SCAN.match(name)
        if m:
            out[m.group(1)] = (st, ld)
    return out


def test_the_regex_reads_the_long_row_kernels_mangling():
    text = ("ptxas info    : Function properties for _ZN3osb19long_scatter_kernelImLi0ELb1ENS_10LongRowGeoELb0EEEvPKNS_8SortPlanEjPKT_PS5_S8_PjS9_T2_PKjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb19long_scatter_kernelImLi1ELb1ENS_10LongRowGeoELb0EEEvPKNS_8SortPlanEjPKT_PS5_S8_PjS9_T2_PKjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb17long_count_kernelItNS_10LongRowGeoEEEvPKNS_8SortPlanEjPKT_S7_S7_T0_PjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb16long_scan_kernelINS_10LongRowGeoEEEvPKNS_8SortPlanEjPjPKjT_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded_long_rows(parse_report(text)) == {"scatter/u64/indices": (4, 8), "count/u16": (0, 0), "scan": (0, 0)}


def test_long_row_instantiations_do_not_spill():
    got = guarded_long_rows(_report())
    want = {f"scatter/{w}/{m}" for w in WIDTH.values() for m in ("keys", "indices")}
    want |= {f"{k}/{w}" for k in ("count", "copy_home", "head_hist") for w in WIDTH.values()}
    want |= {"chunk_sum", "chunk_scan", "scan"}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills in the long-row sort:\n" + "\n".join(spilling)
