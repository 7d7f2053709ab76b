"""Every entry point on caller buffers that start at arbitrary offsets, as views such as v[1:] or x[a:a + n] do.

Each buffer is a view into a larger arena whose other bytes hold a sentinel pattern, placed at a chosen byte offset modulo
512 (computed from data_ptr(), so the caching allocator's own alignment plays no part).  Keys sit at 16-byte offsets, the
alignment the C-ABI asks of them; values sit at 4-byte offsets that are not multiples of 16, their natural alignment and
all the C-ABI asks of them.  Every output is compared element by element with numpy's stable argsort, and every arena byte
outside the buffers must come back bit-identical on both sides: a store before the first element (the few-bins scatter
places its runs from the destination's absolute address) is caught as well as one past the last.  The plan of every
multi-kernel sort is asserted (last_executed_passes), so the cases with an odd number of executed passes do reach the
copy-back, which moves 16-byte words only when both of its buffers are 16-byte aligned.  Keys at other offsets must be
rejected with OSB200_ERR_INVALID_ARG before anything is launched.  -m gpu"""
import numpy as np
import pytest
import torch

from tests.oraclelib import from_radix, to_radix
from tests.test_gpu_bounds import MASKS32, MASKS64, keys_for

pytestmark = pytest.mark.gpu

INVALID_ARG = -1
WINDOW = 512  # offsets are taken modulo this
GUARD = 1024  # sentinel bytes on each side of a buffer, besides those that place it at its offset
T32 = 16384  # 32-bit keys per tile of the keys pass; also the largest n of the single-block path
T8K = 8192  # pairs and 64-bit keys per tile (the single-block path of 64-bit keys ends here)
# the single-block path, one tile + 1, a ragged 3T + 17 (n % 4 == 1: a 4-byte tail in the vector copy-back) for 16,384-
# and 8,192-element tiles
SIZES = [1000, T32 + 1, 3 * T32 + 17, 3 * T8K + 17]
SIZES64 = [1000, T8K + 1, 3 * T8K + 17]
KEY_OFFSETS = [16, 48, 112, 144, 272, 496]
VALUE_OFFSETS = [4, 8, 12, 20, 124, 508]
TORCH = {np.dtype(np.uint32): torch.int32, np.dtype(np.uint64): torch.int64}


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


class Arena:
    """`a` on the device as the view `t`, which starts at byte offset `offset` modulo 512 inside a larger uint8 tensor
    filled with random sentinel bytes."""

    def __init__(self, a: np.ndarray, offset: int, salt: int):
        a = np.ascontiguousarray(a)
        self.dtype = a.dtype
        self.raw = torch.empty(GUARD + WINDOW + a.nbytes + GUARD, dtype=torch.uint8, device="cuda")
        self.lo = GUARD + (offset - (self.raw.data_ptr() + GUARD)) % WINDOW
        self.hi = self.lo + a.nbytes
        self.init = np.random.default_rng(salt).integers(0, 256, self.raw.numel(), dtype=np.uint8)
        self.init[self.lo:self.hi] = a.view(np.uint8)
        self.raw.copy_(torch.from_numpy(self.init))
        self.t = self.raw[self.lo:self.hi].view(TORCH[a.dtype])
        assert self.t.data_ptr() % WINDOW == offset and self.t.numel() == a.size

    def result(self, what: str) -> np.ndarray:
        """the view's contents, after asserting that no byte around it was written"""
        got = self.raw.cpu().numpy()
        assert np.array_equal(got[:self.lo], self.init[:self.lo]), f"{what}: bytes before the buffer were written"
        assert np.array_equal(got[self.hi:], self.init[self.hi:]), f"{what}: bytes past the buffer were written"
        return got[self.lo:self.hi].copy().view(self.dtype)

    def check(self, want: np.ndarray, what: str) -> None:
        got = self.result(what)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"{what}: {bad.size} of {want.size} elements differ, the first at {bad[0]}"

    def unchanged(self, what: str) -> None:
        self.check(self.init[self.lo:self.hi].view(self.dtype), what)


def executed_passes(radix: np.ndarray, begin: int = 0, end: int = None) -> int:
    """the digit places of [begin, end) in which the keys differ: the passes the device plan executes"""
    end = radix.dtype.itemsize * 8 if end is None else end
    count = 0
    for lo in range(begin, end, 8):
        d = (radix >> radix.dtype.type(lo)) & radix.dtype.type((1 << min(8, end - lo)) - 1)
        count += bool((d != d[0]).any())
    return count


def check_plan(s, n, executed, what, small=T32):
    """past the single-block path, the sort executed the passes its keys call for"""
    if n > small:
        assert s.info("last_executed_passes") == executed, f"{what}: executed passes"


def offset_pairs(rotate: int):
    """every key offset once, each with a value offset that changes with `rotate`"""
    r = rotate % len(VALUE_OFFSETS)
    return list(zip(KEY_OFFSETS, VALUE_OFFSETS[r:] + VALUE_OFFSETS[:r]))


def iota(n):
    return np.arange(n, dtype=np.uint32)


def rank_modes(s):
    return [0, 1] if s.info("atomic_order_ok") else [1]


# ---- 1. uint32 keys and pairs -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,andm,orm,executed", MASKS32)
def test_keys_and_pairs_u32(g, name, andm, orm, executed):
    """sort_keys, sort_pairs (payload = input position, so stability shows) and the module-level Sort"""
    rng = np.random.default_rng(100 + executed)
    with g.OneSweepSorter(max(SIZES), 4, 4) as s:
        for i, n in enumerate(SIZES):
            for ko, vo in offset_pairs(i):
                k = keys_for(rng, n, np.uint32, andm, orm)
                assert executed_passes(k) == executed
                order = np.argsort(k, kind="stable")
                what = f"{name} n={n} keys at +{ko} values at +{vo}"
                a = Arena(k, ko, 1)
                s.sort_keys(a.t)
                a.check(k[order], f"sort_keys {what}")
                check_plan(s, n, executed, f"sort_keys {what}")
                ak, av = Arena(k, ko, 2), Arena(iota(n), vo, 3)
                s.sort_pairs(ak.t, av.t)
                ak.check(k[order], f"sort_pairs keys {what}")
                av.check(order.astype(np.uint32), f"sort_pairs values {what}")
                check_plan(s, n, executed, f"sort_pairs {what}")
                ak, av = Arena(k, ko, 4), Arena(iota(n), vo, 5)
                g.Sort(ak.t, av.t)
                torch.cuda.synchronize()
                ak.check(k[order], f"Sort keys {what}")
                av.check(order.astype(np.uint32), f"Sort values {what}")


def test_every_16_byte_key_offset(g):
    """all 31 non-zero 16-byte key offsets of a 512-byte window, each with values at an offset of 4, 8 or 12 mod 16; three
    executed passes, so keys and values are both copied back"""
    n = T32 + 1
    rng = np.random.default_rng(110)
    with g.OneSweepSorter(n, 4, 4) as s:
        for j in range(1, WINDOW // 16):
            ko, vo = 16 * j, 16 * (7 * j % 32) + 4 * (1 + j % 3)
            k = keys_for(rng, n, np.uint32, 0x00FFFFFF, 0x7F000000)
            order = np.argsort(k, kind="stable")
            what = f"keys at +{ko} values at +{vo}"
            a = Arena(k, ko, 6)
            s.sort_keys(a.t)
            a.check(k[order], f"sort_keys {what}")
            check_plan(s, n, 3, f"sort_keys {what}")
            ak, av = Arena(k, ko, 7), Arena(iota(n), vo, 8)
            s.sort_pairs(ak.t, av.t)
            ak.check(k[order], f"sort_pairs keys {what}")
            av.check(order.astype(np.uint32), f"sort_pairs values {what}")
            check_plan(s, n, 3, f"sort_pairs {what}")


# ---- 2. typed keys ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,andm,orm,executed", MASKS32)
@pytest.mark.parametrize("key_type,descending", [("f32", True), ("i32", False)])
def test_typed_keys(g, key_type, descending, name, andm, orm, executed):
    """the last executed pass stores the keys decoded; with an odd pass count the decoded keys then go through the copy-back"""
    kind = key_type[0]
    rng = np.random.default_rng(200 + executed + 10 * descending)
    with g.OneSweepSorter(max(SIZES), 4, 4) as s:
        for i, n in enumerate(SIZES):
            for ko, vo in offset_pairs(i + 2):
                radix = keys_for(rng, n, np.uint32, andm, orm)
                bits = from_radix(radix, kind, descending)
                assert np.array_equal(to_radix(bits, kind, descending), radix)
                order = np.argsort(radix, kind="stable")
                what = f"{key_type} descending={descending} {name} n={n} keys at +{ko} values at +{vo}"
                a = Arena(bits, ko, 10)
                s.sort_keys_typed(a.t, key_type, descending)
                a.check(bits[order], f"sort_keys_typed {what}")
                check_plan(s, n, executed, f"sort_keys_typed {what}")
                ak, av = Arena(bits, ko, 11), Arena(iota(n), vo, 12)
                s.sort_pairs_typed(ak.t, av.t, key_type, descending)
                ak.check(bits[order], f"sort_pairs_typed keys {what}")
                av.check(order.astype(np.uint32), f"sort_pairs_typed values {what}")
                check_plan(s, n, executed, f"sort_pairs_typed {what}")


# ---- 3. bit ranges ------------------------------------------------------------------------------------------------------
# (begin, end, key mask, executed passes).  A last digit of <= 5 bits is scattered run by run in chunks aligned to the
# destination's 128-byte lines: (0, 12) and (5, 17) with two executed passes scatter it straight into the caller's buffers,
# (0, 12) with one executed pass into the alt buffers before the copy-back.
BIT_RANGES = [(0, 12, 0xFFFFFFFF, 2), (0, 12, 0x00000F00, 1), (0, 20, 0xFFFFFFFF, 3), (0, 20, 0x0000FF00, 1),
              (5, 17, 0xFFFFFFFF, 2)]


@pytest.mark.parametrize("begin,end,andm,executed", BIT_RANGES,
                         ids=[f"{b}_{e}_{x}_passes" for b, e, _, x in BIT_RANGES])
def test_sort_bits(g, begin, end, andm, executed):
    rng = np.random.default_rng(300 + begin + end + executed)
    mask = np.uint32(((1 << (end - begin)) - 1) << begin)
    with g.OneSweepSorter(max(SIZES), 4, 4) as s:
        for i, n in enumerate(SIZES):
            for ko, vo in offset_pairs(i + 4):
                k = keys_for(rng, n, np.uint32, andm, 0x5A5A5A5A & ~andm)
                assert executed_passes(k, begin, end) == executed
                order = np.argsort(k & mask, kind="stable")
                what = f"bits [{begin}, {end}) n={n} keys at +{ko} values at +{vo}"
                a = Arena(k, ko, 13)
                s.sort_bits(a.t, begin, end)
                a.check(k[order], f"sort_bits keys only {what}")
                check_plan(s, n, executed, f"sort_bits keys only {what}")
                ak, av = Arena(k, ko, 14), Arena(iota(n), vo, 15)
                s.sort_bits(ak.t, begin, end, av.t)
                ak.check(k[order], f"sort_bits keys {what}")
                av.check(order.astype(np.uint32), f"sort_bits values {what}")
                check_plan(s, n, executed, f"sort_bits pairs {what}")


# ---- 4. uint64 keys -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,andm,orm,executed", MASKS64)
def test_keys_u64(g, name, andm, orm, executed):
    rng = np.random.default_rng(400 + executed)
    with g.OneSweepSorter(max(SIZES64), 8, 0) as s:
        for n in SIZES64:
            for ko in KEY_OFFSETS:
                k = keys_for(rng, n, np.uint64, andm, orm)
                assert executed_passes(k) == executed
                what = f"u64 {name} n={n} keys at +{ko}"
                a = Arena(k, ko, 16)
                s.sort_keys(a.t)
                a.check(np.sort(k), f"sort_keys {what}")
                check_plan(s, n, executed, what, small=T8K)


# ---- 5. argsort through the C-ABI ---------------------------------------------------------------------------------------
def constant_places_input(rng, n, varying):
    """32-bit radix keys in which only the byte places in `varying` differ between keys"""
    r = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    mask = np.uint32(sum(0xFF << (8 * p) for p in varying))
    return (r & mask) | (np.uint32(0x5AA53CC3) & ~mask)


ARGSORT_PLACES = [((), 0), ((3,), 1), ((0, 1, 3), 3), ((0, 1, 2, 3), 4)]


@pytest.mark.parametrize("key_type,descending", [("u32", False), ("f32", True)])
def test_argsort_at_offsets(g, key_type, descending):
    """input, output keys and indices at three independent 16-byte offsets; the input must come back as it was"""
    kind = key_type[0]
    rng = np.random.default_rng(500 + descending)
    j = 0
    with g.OneSweepSorter(3 * T8K + 17, 4, 4) as s:
        for n in (1000, 3 * T8K + 17):
            for varying, executed in ARGSORT_PLACES:
                oi, oo, ox = KEY_OFFSETS[j % 6], KEY_OFFSETS[(j + 2) % 6], KEY_OFFSETS[(j + 3) % 6]
                j += 1
                radix = constant_places_input(rng, n, varying)
                assert executed_passes(radix) == executed
                bits = from_radix(radix, kind, descending)
                order = np.argsort(radix, kind="stable")
                what = f"argsort {key_type} n={n} {executed} passes, in/out/indices at +{oi}/+{oo}/+{ox}"
                ai = Arena(bits, oi, 17)
                ao = Arena(rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32), oo, 18)
                ax = Arena(rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32), ox, 19)
                st = g.lib.osb200_argsort(s._h, ai.t.data_ptr(), ao.t.data_ptr(), ax.t.data_ptr(), n,
                                          g.onesweep.KEY_TYPES[key_type], int(descending), None)
                assert st == 0, what
                torch.cuda.synchronize()
                ai.unchanged(f"{what}: the input")
                ao.check(bits[order], f"{what}: keys")
                ax.check(order.astype(np.uint32), f"{what}: indices")
                check_plan(s, n, executed, what)


# ---- 6. segmented sort --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pairs", [False, True])
def test_segmented_sort_at_offsets(g, pairs):
    """keys at +48 B, values at +20 B; elements before the first offset and after the last belong to no segment"""
    rng = np.random.default_rng(600)
    lens = np.array([3, 0, 2048, 2049, 1, 16384, 777, 5, 0, 16383])
    head, tail = 1001, 999
    offs = np.concatenate([[head], head + np.cumsum(lens)]).astype(np.int64)
    total = int(offs[-1]) + tail
    keys = rng.integers(0, 1 << 32, total, dtype=np.uint64).astype(np.uint32) & np.uint32(0xFFF0F)
    want_k, want_v = keys.copy(), iota(total)
    for a, b in zip(offs[:-1], offs[1:]):
        o = np.argsort(keys[a:b], kind="stable")
        want_k[a:b], want_v[a:b] = keys[a:b][o], (a + o).astype(np.uint32)
    with g.OneSweepSorter(total, 4, 4 if pairs else 0) as s:
        ak = Arena(keys, 48, 20)
        av = Arena(iota(total), 20, 21) if pairs else None
        s.segmented_sort(ak.t, torch.from_numpy(offs).cuda(), av.t if pairs else None)
        ak.check(want_k, "segmented_sort keys")
        if pairs:
            av.check(want_v, "segmented_sort values")


# ---- 7. kernel-level entry points ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("shift", [8, 29])
def test_digit_binning_pass_at_offsets(g, shift):
    """src and dst at 16-byte offsets, their values at 4-byte offsets; shift 29 leaves a 3-bit digit (the few-bins
    scatter); the source must come back as it was"""
    rng = np.random.default_rng(700 + shift)
    dmask = np.uint32((1 << min(8, 32 - shift)) - 1)
    with g.OneSweepSorter(3 * T32 + 17, 4, 4) as s:
        for i, n in enumerate([1000, 3 * T8K + 17, 3 * T32 + 17]):
            for pairs in (False, True):
                ks, kd = KEY_OFFSETS[i], KEY_OFFSETS[i + 3]
                vs, vd = VALUE_OFFSETS[i], VALUE_OFFSETS[i + 3]
                k = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
                order = np.argsort((k >> np.uint32(shift)) & dmask, kind="stable")
                what = f"digit_binning_pass shift={shift} n={n} pairs={pairs}"
                src = Arena(k, ks, 22)
                dst = Arena(rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32), kd, 23)
                sv = Arena(iota(n), vs, 24) if pairs else None
                dv = Arena(rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32), vd, 25) if pairs else None
                s.digit_binning_pass(src.t, dst.t, shift, sv.t if pairs else None, dv.t if pairs else None)
                dst.check(k[order], f"{what}: keys")
                src.unchanged(f"{what}: the source keys")
                if pairs:
                    dv.check(order.astype(np.uint32), f"{what}: values")
                    sv.unchanged(f"{what}: the source values")


@pytest.mark.parametrize("key_bytes", [4, 8])
def test_global_histogram_and_validate_at_offsets(g, key_bytes):
    dtype = np.uint32 if key_bytes == 4 else np.uint64
    rng = np.random.default_rng(800 + key_bytes)
    with g.OneSweepSorter(3 * T32 + 17, key_bytes, 0) as s:
        for i, n in enumerate([5, 1000, 3 * T8K + 17, 3 * T32 + 17]):
            ko = KEY_OFFSETS[(i + 1) % 6]
            k = keys_for(rng, n, dtype, np.iinfo(dtype).max, 0)
            what = f"{8 * key_bytes}-bit keys n={n} at +{ko}"
            a = Arena(k, ko, 26)
            hist = s.global_histogram(a.t).cpu().numpy()
            want = np.stack([np.bincount(((k >> dtype(8 * p)) & dtype(255)).astype(np.int64), minlength=256)
                             for p in range(key_bytes)])
            assert np.array_equal(hist, want), f"global_histogram {what}"
            a.unchanged(f"global_histogram {what}")
            # the first and the last key out of order, and random keys
            srt = np.sort(k)
            ends = srt.copy()
            ends[0], ends[-1] = np.iinfo(dtype).max, 0
            for name, x in (("sorted", srt), ("ends out of order", ends), ("random", k)):
                b = Arena(x, ko, 27)
                assert s.validate(b.t) == int(np.count_nonzero(x[:-1] > x[1:])), f"validate {name} {what}"
                b.unchanged(f"validate {name} {what}")


# ---- 8. HOT passes ------------------------------------------------------------------------------------------------------
def test_hot_passes_at_offsets(g):
    """low-entropy keys (AND of three random words: digit 0 holds about a third of every place) with a constant top byte:
    three executed passes, all HOT, and the copy-back; keys at +48 B, values at +4 B"""
    n = (1 << 22) + 4099
    rng = np.random.default_rng(900)
    r = rng.integers(0, 1 << 32, (3, n), dtype=np.uint64).astype(np.uint32)
    k = (r[0] & r[1] & r[2] & np.uint32(0x00FFFFFF)) | np.uint32(0x5A000000)
    del r
    assert executed_passes(k) == 3
    order = np.argsort(k, kind="stable")
    with g.OneSweepSorter(n, 4, 4) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            what = f"rank_mode={mode}"
            a = Arena(k, 48, 30)
            s.sort_keys(a.t)
            a.check(k[order], f"sort_keys {what}")
            check_plan(s, n, 3, f"sort_keys {what}")
            assert s.info("last_hot_mask") != 0, f"sort_keys {what}: no HOT pass"
            ak, av = Arena(k, 48, 31), Arena(iota(n), 4, 32)
            s.sort_pairs(ak.t, av.t)
            ak.check(k[order], f"sort_pairs keys {what}")
            av.check(order.astype(np.uint32), f"sort_pairs values {what}")
            check_plan(s, n, 3, f"sort_pairs {what}")
            assert s.info("last_hot_mask") != 0, f"sort_pairs {what}: no HOT pass"


# ---- 9. graph capture ---------------------------------------------------------------------------------------------------
def test_graph_replays_with_offset_values(g):
    """a captured sort_pairs with values at +4 B replayed on new inputs written into the same views; every input executes
    an odd number of passes, so each replay copies the values back"""
    n = 3 * T8K + 17
    rng = np.random.default_rng(1000)
    odd = [(andm, orm, executed) for _, andm, orm, executed in MASKS32 if executed % 2]
    inputs = [(keys_for(rng, n, np.uint32, andm, orm), executed) for andm, orm, executed in odd + odd]
    with g.OneSweepSorter(n, 4, 4) as s:
        k0 = inputs[0][0]
        order = np.argsort(k0, kind="stable")
        ak, av = Arena(k0, 144, 40), Arena(iota(n), 4, 41)
        s.sort_pairs(ak.t, av.t)  # eager, before the capture
        ak.check(k0[order], "eager keys")
        av.check(order.astype(np.uint32), "eager values")
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            s.sort_pairs(ak.t, av.t)
        for i, (k, executed) in enumerate(inputs[1:]):
            ak.t.copy_(torch.from_numpy(k.view(np.int32)))
            av.t.copy_(torch.from_numpy(iota(n).view(np.int32)))
            graph.replay()
            torch.cuda.synchronize()
            order = np.argsort(k, kind="stable")
            ak.check(k[order], f"replay {i} keys")
            av.check(order.astype(np.uint32), f"replay {i} values")
            assert s.info("last_executed_passes") == executed, f"replay {i}"
        del graph


# ---- 10. misaligned keys ------------------------------------------------------------------------------------------------
def rejected(g, call, what):
    with pytest.raises(g.OneSweepError) as e:
        call()
    assert e.value.status == INVALID_ARG, what


def test_misaligned_keys_are_rejected_without_a_launch(g):
    """keys at +4, +8 and +12 B (64-bit keys at +8 B) on every entry point that checks key alignment, and each of the
    argsort's three pointers: OSB200_ERR_INVALID_ARG, no byte of any arena written, and the handle still sorts.  The sizes
    are small enough that none of these calls would issue a 16-byte access even if its check were missing."""
    n = 3
    rng = np.random.default_rng(1100)
    k = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    with g.OneSweepSorter(3 * T8K + 17, 4, 4) as s:
        for off in (4, 8, 12):
            a, v, ok = Arena(k, off, 50), Arena(iota(n), 4, 51), Arena(k, 16, 52)
            calls = {
                "sort_keys": lambda: s.sort_keys(a.t),
                "sort_pairs": lambda: s.sort_pairs(a.t, v.t),
                "sort_keys_typed": lambda: s.sort_keys_typed(a.t, "f32", True),
                "sort_pairs_typed": lambda: s.sort_pairs_typed(a.t, v.t, "i32"),
                "sort_bits keys only": lambda: s.sort_bits(a.t, 0, 20),
                "sort_bits pairs": lambda: s.sort_bits(a.t, 0, 20, v.t),
                "global_histogram": lambda: s.global_histogram(a.t),
                "digit_binning_pass src": lambda: s.digit_binning_pass(a.t, ok.t, 8),
                "digit_binning_pass dst": lambda: s.digit_binning_pass(ok.t, a.t, 8),
            }
            for name, call in calls.items():
                rejected(g, call, f"{name}: keys at +{off}")
            ins = [Arena(k, 16, 53), Arena(k, 32, 54), Arena(k, 48, 55)]
            for p in range(3):
                ptrs = [x.t.data_ptr() for x in ins]
                ptrs[p] += off
                st = g.lib.osb200_argsort(s._h, ptrs[0], ptrs[1], ptrs[2], n, 0, 0, None)
                assert st == INVALID_ARG, f"argsort pointer {p} at +{off}"
            torch.cuda.synchronize()
            for x in (a, v, ok, *ins):
                x.unchanged(f"keys at +{off}: a rejected call wrote")
        # the handle still sorts: a multi-kernel pairs sort with an odd number of passes and values at +4 B
        n = 3 * T8K + 17
        k = keys_for(rng, n, np.uint32, 0x00FFFFFF, 0)
        order = np.argsort(k, kind="stable")
        ak, av = Arena(k, 16, 56), Arena(iota(n), 4, 57)
        s.sort_pairs(ak.t, av.t)
        ak.check(k[order], "aligned sort after the rejections: keys")
        av.check(order.astype(np.uint32), "aligned sort after the rejections: values")
        check_plan(s, n, 3, "aligned sort after the rejections")
    n = 3
    k = keys_for(rng, n, np.uint64, (1 << 64) - 1, 0)
    with g.OneSweepSorter(3 * T8K + 17, 8, 0) as s:
        a, ok = Arena(k, 8, 60), Arena(k, 16, 61)
        one = Arena(k[:1], 8, 62)  # (one 64-bit key: no 16-byte vector even without the check)
        calls = {
            "sort_keys": lambda: s.sort_keys(a.t),
            "sort_keys_typed": lambda: s.sort_keys_typed(a.t, "i64"),
            "sort_bits": lambda: s.sort_bits(a.t, 0, 40),
            "global_histogram": lambda: s.global_histogram(one.t),
            "digit_binning_pass src": lambda: s.digit_binning_pass(a.t, ok.t, 8),
            "digit_binning_pass dst": lambda: s.digit_binning_pass(ok.t, a.t, 8),
        }
        for name, call in calls.items():
            rejected(g, call, f"u64 {name}: keys at +8")
        torch.cuda.synchronize()
        for x in (a, ok, one):
            x.unchanged("u64 keys at +8: a rejected call wrote")
        n = 3 * T8K + 17
        k = keys_for(rng, n, np.uint64, 0xFFFFFF, 0x7766554433000000)
        b = Arena(k, 16, 63)
        s.sort_keys(b.t)
        b.check(np.sort(k), "u64 aligned sort after the rejections")
        check_plan(s, n, 3, "u64 aligned sort after the rejections", small=T8K)
