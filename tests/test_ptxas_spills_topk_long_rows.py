"""CPU check of the split path of the row top-k's compiled kernels (osb200_topk_long_rows): the count, pick, tile fold,
compaction and finisher, and the in-place sort's scatter (both rank modes) and copy home, for 16-, 32- and 64-bit keys, must
appear in the ptxas report of osb_kernels.cu, and none may spill registers to local memory.  uint16_t mangles as `t`,
uint32_t as `j`, uint64_t as `m`.  The test reads the report of the library as built; it skips when there is none or it is
older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# topk_long_sort_scatter_kernel<KeyT, RANK_MODE>
SCATTER = re.compile(r"_ZN3osb\d+topk_long_sort_scatter_kernelI([tjm])Li(\d+)EE")
# topk_long_{count,pick,compact,finish,sort_copy_home}_kernel<KeyT>
PER_KEY = re.compile(r"_ZN3osb\d+topk_long_(count|pick|compact|finish|sort_copy_home)_kernelI([tjm])EE")
TILES = re.compile(r"_ZN3osb\d+topk_long_tiles_kernelE")
WIDTH = {"t": "u16", "j": "u32", "m": "u64"}


def guarded_topk_long_rows(report):
    """{what: (spill stores, spill loads)} of the split path's instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        m = SCATTER.match(name)
        if m:
            out[f"sort_scatter/{WIDTH[m.group(1)]}/rank{m.group(2)}"] = (st, ld)
        m = PER_KEY.match(name)
        if m:
            out[f"{m.group(1)}/{WIDTH[m.group(2)]}"] = (st, ld)
        if TILES.match(name):
            out["tiles"] = (st, ld)
    return out


def test_the_regex_reads_the_split_path_kernels_mangling():
    text = ("ptxas info    : Function properties for _ZN3osb29topk_long_sort_scatter_kernelImLi1EEEvPKNS_8SortPlanEjPKT_PS4_S7_PjS8_mjjPKjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb22topk_long_count_kernelItEEvPKT_mjjjjPKNS_11TopkLongRowEPjS7_S7_NS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb22topk_long_tiles_kernelEmjjjPKNS_11TopkLongRowEPKjPj\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded_topk_long_rows(parse_report(text)) == {"sort_scatter/u64/rank1": (4, 8), "count/u16": (0, 0), "tiles": (0, 0)}


def test_split_path_instantiations_do_not_spill():
    got = guarded_topk_long_rows(_report())
    want = {f"sort_scatter/{w}/rank{r}" for w in WIDTH.values() for r in (0, 1)}
    want |= {f"{k}/{w}" for k in ("count", "pick", "compact", "finish", "sort_copy_home") for w in WIDTH.values()}
    want |= {"tiles"}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills in the row top-k's split path:\n" + "\n".join(spilling)
