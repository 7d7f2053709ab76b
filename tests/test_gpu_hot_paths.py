"""Every feature of the DigitBinningPass through its HOT instantiation: typed keys in both directions, typed pairs, bit ranges
(whose narrow last digit always makes the pass hot and takes the few-bins scatter), both ranking modes, and the
forward-progress fallback (stalled tiles re-reduced inside the striding kernel, on encoded keys too).

The scan kernel calls a digit place hot when n >= 2^22 and one bin holds at least n/8 keys; smaller inputs never reach the
HOT kernel.  Every case asserts the plan's hot (and skip) mask, so a test cannot pass on the plain kernel by accident, and
is repeated with hot_passes = 0 against the same numpy reference (stable argsort of the radix key or of the masked bit
range).  -m gpu"""
import numpy as np
import pytest
import torch

from tests.oraclelib import from_radix, to_radix

pytestmark = pytest.mark.gpu

N32 = (1 << 22) + 4099           # 32-bit keys: 256 full 16,384-key tiles and a ragged one (pairs: 8,192-pair tiles)
N64 = (1 << 22) + 8192 * 3 + 1   # 64-bit keys: 8,192-key tiles, the last one holds a single key

TYPES = [("u32", np.uint32, "u"), ("i32", np.uint32, "i"), ("f32", np.uint32, "f"),
         ("u64", np.uint64, "u"), ("i64", np.uint64, "i"), ("f64", np.uint64, "f")]


def dev(a):
    return torch.from_numpy(a.view(np.int32 if a.dtype.itemsize == 4 else np.int64).copy()).cuda()


def host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def rank_modes(s):
    """1 = ballot ranking (the HOT kernel then ranks the hot digit like any other); 0 = atomic ranking with the ballot for
    the tile's hot digit, where the device supports it"""
    return [0, 1] if s.info("atomic_order_ok") else [1]


def float_specials(utype):
    """+-0, smallest and largest subnormals, +-max, +-inf and NaNs of both signs with several payloads (bit patterns)"""
    fi = np.finfo(np.float32 if utype == np.uint32 else np.float64)
    nb = np.dtype(utype).itemsize * 8
    exp_all = ((1 << (nb - 1 - fi.nmant)) - 1) << fi.nmant
    top = (1 << fi.nmant) - 1
    pos = [0, 1, top, fi.max.view(utype).item(), exp_all, exp_all | 1, exp_all | (1 << (fi.nmant - 1)), exp_all | top,
           exp_all | 0x5A5]
    return np.array(pos + [(1 << (nb - 1)) | p for p in pos], dtype=utype)


def hot_input(rng, n, utype, kind, descending, low_byte=None):
    """Typed bits of n keys: about 80 % share one value, the rest are spread over the whole key space.  Built as radix keys:
    the common one is 0x7F..FF, so in every place but the top one its digit is the digit of the all-ones padding of the
    ragged last tile.  low_byte: every radix key gets this low byte, so pass 0 is skipped and the first executed pass (the
    one that encodes) is pass 1.  Floats also get every special value, 64 times each."""
    hi = np.iinfo(utype).max
    enc = rng.integers(0, hi, n, dtype=utype, endpoint=True)
    enc[rng.random(n) < 0.8] = hi >> 1
    if low_byte is not None:
        enc = (enc & ~utype(0xFF)) | utype(low_byte)
    bits = from_radix(enc, kind, descending)
    if kind == "f" and low_byte is None:
        sp = float_specials(utype)
        bits[rng.choice(n, 64 * sp.size, replace=False)] = np.repeat(sp, 64)
    return bits


def check_plan(s, hot, skip, hot_mask):
    assert s.info("last_skip_mask") == skip
    assert s.info("last_hot_mask") == (hot_mask if hot else 0)


@pytest.mark.parametrize("low_byte", [None, 0x5A], ids=["all_places", "pass0_skipped"])
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("name,utype,kind", TYPES)
def test_typed_keys_hot(g, name, utype, kind, descending, low_byte):
    """The first executed pass encodes and the last one decodes, both in the HOT kernel; pass 1 encodes when pass 0 is
    skipped."""
    kb = np.dtype(utype).itemsize
    n = N32 if kb == 4 else N64
    rng = np.random.default_rng(kb * 100 + "uif".index(kind) * 10 + descending * 2 + (low_byte is not None))
    bits = hot_input(rng, n, utype, kind, descending, low_byte)
    want = bits[np.argsort(to_radix(bits, kind, descending), kind="stable")]
    skip = 0 if low_byte is None else 1
    with g.OneSweepSorter(n, kb, 0) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for hot in (1, 0):
                s.set_option("hot_passes", hot)
                t = dev(bits)
                s.sort_keys_typed(t, name, descending)
                assert np.array_equal(host(t, utype), want), f"rank_mode={mode} hot_passes={hot}"
                check_plan(s, hot, skip, ((1 << kb) - 1) & ~skip)


@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("name,kind", [("f32", "f"), ("i32", "i")])
def test_typed_pairs_hot(g, name, kind, descending):
    """payload = input index: ~80 % of the keys are equal, so any instability shows in the payloads"""
    n = N32
    bits = hot_input(np.random.default_rng(7 + descending), n, np.uint32, kind, descending)
    order = np.argsort(to_radix(bits, kind, descending), kind="stable")
    with g.OneSweepSorter(n, 4, 4) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for hot in (1, 0):
                s.set_option("hot_passes", hot)
                tk, tv = dev(bits), dev(np.arange(n, dtype=np.uint32))
                s.sort_pairs_typed(tk, tv, name, descending)
                assert np.array_equal(host(tk), bits[order]), f"keys rank_mode={mode} hot_passes={hot}"
                assert np.array_equal(host(tv), order.astype(np.uint32)), f"payloads rank_mode={mode} hot_passes={hot}"
                check_plan(s, hot, 0, 0xF)


def expected_hot_bits(begin, end, and_count):
    """the narrow last digit (<= 8 bins for the ranges here) always has a bin with >= n/8 keys; with AND-of-4 keys (each bit
    set with probability 1/16) every place is dominated by its zero digit"""
    places = (end - begin + 7) // 8
    return (1 << places) - 1 if and_count else 1 << (places - 1)


@pytest.mark.parametrize("and_count", [0, 3], ids=["uniform", "low_entropy"])
@pytest.mark.parametrize("begin,end", [(0, 3), (31, 32), (5, 8), (9, 12), (0, 11)])
def test_sort_bits_u32_hot(g, oracle, begin, end, and_count):
    n = N32
    k = oracle.init_random_u32(n, and_count, 1000 + begin * 37 + end)
    v = np.arange(n, dtype=np.uint32)
    order = np.argsort((k >> np.uint32(begin)) & np.uint32((1 << (end - begin)) - 1), kind="stable")
    with g.OneSweepSorter(n, 4, 4) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for hot in (1, 0):
                s.set_option("hot_passes", hot)
                tk = dev(k)
                s.sort_bits(tk, begin, end)
                assert np.array_equal(host(tk), k[order]), f"keys rank_mode={mode} hot_passes={hot}"
                check_plan(s, hot, 0, expected_hot_bits(begin, end, and_count))
                tk, tv = dev(k), dev(v)
                s.sort_bits(tk, begin, end, tv)
                assert np.array_equal(host(tk), k[order]) and np.array_equal(host(tv), v[order]), \
                    f"pairs rank_mode={mode} hot_passes={hot}"
                check_plan(s, hot, 0, expected_hot_bits(begin, end, and_count))


@pytest.mark.parametrize("and_count", [0, 3], ids=["uniform", "low_entropy"])
@pytest.mark.parametrize("begin,end", [(60, 63), (0, 3)])
def test_sort_bits_u64_hot(g, oracle, begin, end, and_count):
    n = N64
    k = oracle.init_random_u64(n, and_count, 2000 + begin * 37 + end)
    order = np.argsort((k >> np.uint64(begin)) & np.uint64((1 << (end - begin)) - 1), kind="stable")
    with g.OneSweepSorter(n, 8, 0) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for hot in (1, 0):
                s.set_option("hot_passes", hot)
                t = dev(k)
                s.sort_bits(t, begin, end)
                assert np.array_equal(host(t, np.uint64), k[order]), f"rank_mode={mode} hot_passes={hot}"
                check_plan(s, hot, 0, 1)


@pytest.mark.parametrize("stall_every", [1, 3])
def test_stalled_tiles_in_the_hot_kernel(g, oracle, stall_every):
    """Tiles with tile % N == N-1 withhold their reduction; their successors hit the spin cap and re-reduce them, here while
    the resident CTAs of the HOT kernel stride over the tiles.  In the first pass of a typed sort the re-reduction must count
    the digits of the ENCODED keys."""
    n = N32
    rng = np.random.default_rng(stall_every)
    k = hot_input(rng, n, np.uint32, "u", False)
    f = hot_input(rng, n, np.uint32, "f", False)
    want_f = f[np.argsort(to_radix(f, "f"), kind="stable")]
    u = oracle.init_random_u32(n, 0, 40 + stall_every)
    order_k = np.argsort(k, kind="stable")
    order_u = np.argsort(u & np.uint32(7), kind="stable")
    v = np.arange(n, dtype=np.uint32)
    with g.OneSweepSorter(n, 4, 4) as s:
        s.set_option("spin_cap", 16)
        s.set_option("debug_stall_every", stall_every)
        for hot in (1, 0):
            s.set_option("hot_passes", hot)
            t = dev(k)
            s.sort_keys(t)
            assert np.array_equal(host(t), k[order_k]), f"keys hot_passes={hot}"
            check_plan(s, hot, 0, 0xF)
            tk, tv = dev(k), dev(v)
            s.sort_pairs(tk, tv)
            assert np.array_equal(host(tk), k[order_k]) and np.array_equal(host(tv), v[order_k]), f"pairs hot_passes={hot}"
            check_plan(s, hot, 0, 0xF)
            t = dev(f)
            s.sort_keys_typed(t, "f32")
            assert np.array_equal(host(t), want_f), f"typed f32 hot_passes={hot}"
            check_plan(s, hot, 0, 0xF)
            t = dev(u)
            s.sort_bits(t, 0, 3)
            assert np.array_equal(host(t), u[order_u]), f"bits (0, 3) hot_passes={hot}"
            check_plan(s, hot, 0, 1)
            tk, tv = dev(u), dev(v)
            s.sort_bits(tk, 0, 3, tv)
            assert np.array_equal(host(tk), u[order_u]) and np.array_equal(host(tv), v[order_u]), \
                f"bits (0, 3) pairs hot_passes={hot}"
