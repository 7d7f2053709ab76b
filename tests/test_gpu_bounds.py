"""Nothing is written past n: every entry point sorts the first n elements of a longer buffer, whose remaining elements
hold a sentinel pattern and must come back bit-identical -- keys and values, on the one-launch small-n path, across the
ragged last tile's scatter, the typed decode-on-store and the copy-back that follows an odd number of executed passes
(including its sub-16-byte tail).  The sorted prefix is checked against numpy at the same time.  The segmented sort must
likewise leave the elements outside every segment alone.  -m gpu"""
import numpy as np
import pytest
import torch

from tests.oraclelib import from_radix, to_radix

pytestmark = pytest.mark.gpu

PAD = 4099  # sentinel elements after the n sorted ones; the sorters are created for n + PAD elements (>= n + 16 bytes)


def dev(a):
    return torch.from_numpy(a.view(np.int32 if a.dtype.itemsize == 4 else np.int64).copy()).cuda()


def host(t, dtype):
    return t.cpu().numpy().view(dtype)


def sentinel(dtype, count, salt):
    i = np.arange(count, dtype=np.uint64)
    s = (np.uint64(0xA5A5A5A5C3C3C3C3) ^ (i * np.uint64(0x9E3779B97F4A7C15)) ^ np.uint64(salt)).astype(np.uint64)
    return s.astype(dtype)


def padded(a, salt):
    """device buffer of a.size + PAD elements: a, then the sentinel"""
    return dev(np.concatenate([a, sentinel(a.dtype, PAD, salt)]))


def check(t, n, want, salt, what):
    got = host(t, want.dtype)
    assert np.array_equal(got[:n], want), f"{what}: sorted prefix"
    assert np.array_equal(got[n:], sentinel(want.dtype, PAD, salt)), f"{what}: elements past n were written"


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


# radix-key masks (and, or) of 32-bit keys and the passes their plan executes: 4 (even: no copy-back), 1 and 3 (the result
# is in the alt buffers and is copied back)
MASKS32 = [("all_bytes_vary", 0xFFFFFFFF, 0, 4), ("only_byte_1_varies", 0x0000FF00, 0x12340056, 1),
           ("bytes_0_1_2_vary", 0x00FFFFFF, 0x7F000000, 3)]
MASKS64 = [("all_bytes_vary", (1 << 64) - 1, 0, 8), ("only_byte_1_varies", 0xFF00, 0x0123456789AB0056, 1),
           ("bytes_0_1_2_vary", 0xFFFFFF, 0x7766554433000000, 3)]


def sizes(tile):
    """small path (<= 16,384 32-bit or 8,192 64-bit keys: one launch), one tile + 1, a ragged 3T + 17 (n % 4 == 1: a 4-byte
    copy-back tail for 32-bit keys), 4T + 2 (n % 4 == 2)"""
    return sorted({1000, 8192, 16384, tile + 1, 3 * tile + 17, 4 * tile + 2})


def keys_for(rng, n, dtype, andm, orm):
    hi = np.iinfo(dtype).max
    return (rng.integers(0, hi, n, dtype=dtype, endpoint=True) & dtype(andm)) | dtype(orm)


@pytest.mark.parametrize("name,andm,orm,executed", MASKS32)
def test_keys_and_pairs_u32_stay_in_bounds(g, name, andm, orm, executed):
    rng = np.random.default_rng(executed)
    with g.OneSweepSorter(4 * 16384 + 2 + PAD, 4, 4) as s:
        for n in sizes(16384) + [3 * 8192 + 17]:  # (the last one: ragged 8,192-pair tiles)
            k = keys_for(rng, n, np.uint32, andm, orm)
            order = np.argsort(k, kind="stable")
            t = padded(k, 1)
            s.sort_keys(t, n)
            check(t, n, k[order], 1, f"sort_keys {name} n={n}")
            if n > 16384:
                assert s.info("last_executed_passes") == executed
            tk, tv = padded(k, 2), padded(np.arange(n, dtype=np.uint32), 3)
            s.sort_pairs(tk, tv, n)
            check(tk, n, k[order], 2, f"sort_pairs keys {name} n={n}")
            check(tv, n, order.astype(np.uint32), 3, f"sort_pairs values {name} n={n}")


@pytest.mark.parametrize("name,andm,orm,executed", MASKS32)
def test_typed_f32_descending_stays_in_bounds(g, name, andm, orm, executed):
    """the last executed pass stores decoded keys (the ragged-tile / typed scatter); radix keys with constant bytes give an
    odd number of passes, so the decoded keys also go through the copy-back"""
    rng = np.random.default_rng(10 + executed)
    with g.OneSweepSorter(4 * 16384 + 2 + PAD, 4, 4) as s:
        for n in sizes(16384) + [3 * 8192 + 17]:
            bits = from_radix(keys_for(rng, n, np.uint32, andm, orm), "f", True)
            order = np.argsort(to_radix(bits, "f", True), kind="stable")
            t = padded(bits, 4)
            s.sort_keys_typed(t, "f32", descending=True, n=n)
            check(t, n, bits[order], 4, f"sort_keys_typed {name} n={n}")
            if n > 16384:
                assert s.info("last_executed_passes") == executed
            tk, tv = padded(bits, 5), padded(np.arange(n, dtype=np.uint32), 6)
            s.sort_pairs_typed(tk, tv, "f32", descending=True, n=n)
            check(tk, n, bits[order], 5, f"sort_pairs_typed keys {name} n={n}")
            check(tv, n, order.astype(np.uint32), 6, f"sort_pairs_typed values {name} n={n}")


@pytest.mark.parametrize("andm", [0xFFFFFFFF, 0x0000FF00], ids=["three_passes", "one_pass"])
def test_sort_bits_odd_pass_count_stays_in_bounds(g, andm):
    """bits [0, 20): three places, an odd count, so the result is always copied back"""
    rng = np.random.default_rng(20)
    with g.OneSweepSorter(4 * 16384 + 2 + PAD, 4, 4) as s:
        for n in sizes(16384) + [3 * 8192 + 17]:
            k = keys_for(rng, n, np.uint32, andm, 0)
            order = np.argsort(k & np.uint32(0xFFFFF), kind="stable")
            t = padded(k, 7)
            s.sort_bits(t, 0, 20, n=n)
            check(t, n, k[order], 7, f"sort_bits keys n={n}")
            if n > 16384:
                assert s.info("last_executed_passes") == (3 if andm == 0xFFFFFFFF else 1)
            tk, tv = padded(k, 8), padded(np.arange(n, dtype=np.uint32), 9)
            s.sort_bits(tk, 0, 20, tv, n=n)
            check(tk, n, k[order], 8, f"sort_bits pairs keys n={n}")
            check(tv, n, order.astype(np.uint32), 9, f"sort_bits pairs values n={n}")


@pytest.mark.parametrize("name,andm,orm,executed", MASKS64)
def test_keys_u64_stay_in_bounds(g, name, andm, orm, executed):
    rng = np.random.default_rng(30 + executed)
    with g.OneSweepSorter(4 * 8192 + 2 + PAD, 8, 0) as s:
        for n in sizes(8192):
            k = keys_for(rng, n, np.uint64, andm, orm)
            t = padded(k, 10)
            s.sort_keys(t, n)
            check(t, n, np.sort(k), 10, f"sort_keys u64 {name} n={n}")
            if n > 8192:
                assert s.info("last_executed_passes") == executed


@pytest.mark.parametrize("pairs", [False, True])
def test_segmented_sort_leaves_the_outside_alone(g, pairs):
    """elements before the first offset and after the last one belong to no segment; segments of odd lengths, empty ones and
    one of a full tile sit in between"""
    rng = np.random.default_rng(40)
    lens = np.array([3, 0, 2048, 2049, 1, 16384, 777, 5, 0, 16383])
    head = 1001
    offs = np.concatenate([[head], head + np.cumsum(lens)]).astype(np.int64)
    total = int(offs[-1]) + PAD
    keys = rng.integers(0, 1 << 32, total, dtype=np.uint64).astype(np.uint32) & np.uint32(0xFFF0F)
    want_k, want_v = keys.copy(), np.arange(total, dtype=np.uint32)
    for a, b in zip(offs[:-1], offs[1:]):
        o = np.argsort(keys[a:b], kind="stable")
        want_k[a:b], want_v[a:b] = keys[a:b][o], (a + o).astype(np.uint32)
    with g.OneSweepSorter(total, 4, 4 if pairs else 0) as s:
        tk = dev(keys)
        tv = torch.arange(total, dtype=torch.int32, device="cuda") if pairs else None
        s.segmented_sort(tk, torch.from_numpy(offs).cuda(), tv)
        assert np.array_equal(host(tk, np.uint32), want_k)
        if pairs:
            assert np.array_equal(host(tv, np.uint32), want_v)
