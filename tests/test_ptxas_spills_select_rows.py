"""CPU check of the row select's compiled kernels (osb200_select_rows): the short path's warp and block kernels (both rank
modes, values only and with positions) and the split path's count, pick, equal-key count and locate kernels, for 16-, 32-
and 64-bit keys, must appear in the ptxas report of osb_kernels.cu, and none may spill registers to local memory.  uint16_t
mangles as `t`, uint32_t as `j`, uint64_t as `m`.  The test reads the report of the library as built; it skips when there is
none or it is older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# select_rows_warp_kernel<KeyT, K, RANK_MODE, INDICES>, select_rows_block_kernel<KeyT, K, WARPS, RANK_MODE, INDICES>
WARP = re.compile(r"_ZN3osb\d+select_rows_warp_kernelI([tjm])Li(\d+)ELi(\d+)ELb([01])EE")
BLOCK = re.compile(r"_ZN3osb\d+select_rows_block_kernelI([tjm])Li(\d+)ELi(\d+)ELi(\d+)ELb([01])EE")
SPLIT = re.compile(r"_ZN3osb\d+select_(count|pick|eq_count|locate)_kernelI([tjm])EE")
WIDTH = {"t": "u16", "j": "u32", "m": "u64"}


def guarded_select_rows(report):
    """{what: (spill stores, spill loads)} of the row select's instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        m = WARP.match(name)
        if m:
            out[f"warp/{WIDTH[m.group(1)]}/K{m.group(2)}/rank{m.group(3)}/idx{m.group(4)}"] = (st, ld)
        m = BLOCK.match(name)
        if m:
            out[f"block/{WIDTH[m.group(1)]}/K{m.group(2)}/rank{m.group(4)}/idx{m.group(5)}"] = (st, ld)
        m = SPLIT.match(name)
        if m:
            out[f"{m.group(1)}/{WIDTH[m.group(2)]}"] = (st, ld)
    return out


def test_the_regex_reads_the_select_kernels_mangling():
    text = ("ptxas info    : Function properties for _ZN3osb24select_rows_block_kernelIjLi32ELi16ELi1ELb1EEEvPKT_PS1_PjmjNS_8KeyCodecENS_11SelectRanksE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb23select_rows_warp_kernelItLi8ELi0ELb0EEEvPKT_PS1_PjmjNS_8KeyCodecENS_11SelectRanksE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb22select_eq_count_kernelImEEvPKT_mjjjPKNS_11SelectStateEPjNS_8KeyCodecE\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded_select_rows(parse_report(text)) == {"block/u32/K32/rank1/idx1": (4, 8), "warp/u16/K8/rank0/idx0": (0, 0),
                                                       "eq_count/u64": (0, 0)}


def test_select_rows_instantiations_do_not_spill():
    got = guarded_select_rows(_report())
    want = {f"warp/{w}/K{k}/rank{r}/idx{i}" for w in WIDTH.values() for k in (1, 2, 4, 8) for r in (0, 1) for i in (0, 1)}
    want |= {f"block/{w}/K{k}/rank{r}/idx{i}" for w, ks in (("u16", (8, 32)), ("u32", (8, 32)), ("u64", (8, 16)))
             for k in ks for r in (0, 1) for i in (0, 1)}
    want |= {f"{k}/{w}" for k in ("count", "pick", "eq_count", "locate") for w in WIDTH.values()}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills in the row select:\n" + "\n".join(spilling)
