"""CPU check of the segment sort's compiled kernels (osb200_sort_segments): the binning kernel, the warp class
(segment_sort_warp_kernel) and the block classes (segment_list_sort_kernel, the 2,048- and 16,384-key geometries,
8,192 for 64-bit keys), for 16-, 32- and 64-bit keys, keys only and with indices, must appear in the ptxas report of
osb_kernels.cu and must not spill registers to local memory in the default (atomic) rank mode.  uint16_t mangles as `t`,
uint32_t as `j`, uint64_t as `m`.  The test reads the report of the library as built; it skips when there is none or it is
older than the sources."""
import re

from tests.test_ptxas_spills import _report, parse_report

# segment_bin_kernel<KeyT>
BIN = re.compile(r"_ZN3osb18segment_bin_kernelI([tjm])EE")
# segment_sort_warp_kernel<KeyT, RANK_MODE, INDICES>
WARP = re.compile(r"_ZN3osb24segment_sort_warp_kernelI([tjm])Li(\d+)ELb([01])EE")
# segment_list_sort_kernel<KeyT, PAIRS, K, WARPS, RANK_MODE, INDICES>
BLOCK = re.compile(r"_ZN3osb24segment_list_sort_kernelI([tjm])Lb([01])ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])EE")
WIDTH = {"t": "u16", "j": "u32", "m": "u64"}
RANK_ATOMIC = 0


def guarded_segments(report):
    """{what: (spill stores, spill loads)} of the atomic-mode segment sort instantiations in a parsed report"""
    out = {}
    for name, st, ld in report:
        m = BIN.match(name)
        if m:
            out[f"bin/{WIDTH[m.group(1)]}"] = (st, ld)
        w = WARP.match(name)
        if w and int(w.group(2)) == RANK_ATOMIC:
            out[f"warp/{WIDTH[w.group(1)]}/" + ("indices" if w.group(3) == "1" else "keys")] = (st, ld)
        b = BLOCK.match(name)
        if b and int(b.group(5)) == RANK_ATOMIC:
            keys = int(b.group(3)) * int(b.group(4)) * 32
            out[f"block/{WIDTH[b.group(1)]}/{keys}/" + ("indices" if b.group(6) == "1" else "keys")] = (st, ld)
    return out


def test_the_regex_reads_the_segment_kernels_mangling():
    text = ("ptxas info    : Function properties for _ZN3osb24segment_sort_warp_kernelImLi0ELb1EEEvPKT_PS1_PjPKyPKjS7_NS_8KeyCodecE\n"
            "    0 bytes stack frame, 4 bytes spill stores, 8 bytes spill loads\n"
            "ptxas info    : Function properties for "
            "_ZN3osb24segment_list_sort_kernelItLb0ELi8ELi8ELi0ELb0EEEvPT_PjPKymmjjNS_8KeyCodecEPKS1_PKjS5_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for "
            "_ZN3osb19segment_sort_kernelItLb0ELi8ELi8ELi0ELb0ELb1EEEvPT_PjPKymmjjjjNS_8KeyCodecEPKS1_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
            "ptxas info    : Function properties for _ZN3osb18segment_bin_kernelIjEEvPKymmjPjPyPKT_PS5_S3_\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert guarded_segments(parse_report(text)) == {"warp/u64/indices": (4, 8), "block/u16/2048/keys": (0, 0), "bin/u32": (0, 0)}


def test_segment_sort_instantiations_do_not_spill():
    got = guarded_segments(_report())
    want = {f"bin/{w}" for w in WIDTH.values()}
    want |= {f"warp/{w}/{m}" for w in WIDTH.values() for m in ("keys", "indices")}
    want |= {f"block/{w}/{t}/{m}" for w in WIDTH.values() for t in (2048, 8192 if w == "u64" else 16384)
             for m in ("keys", "indices")}
    assert want <= set(got), f"instantiations missing from the ptxas report: {sorted(want - set(got))}"
    spilling = [f"{what}: {st} B spill stores, {ld} B spill loads" for what, (st, ld) in sorted(got.items()) if st or ld]
    assert not spilling, "register spills in the segment sort:\n" + "\n".join(spilling)
