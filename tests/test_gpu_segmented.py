"""Small-n path and segmented sort (SURVEY 8f rank 4; reference: SplitSort, GPUSortingCUDA/SegSort/SplitSort/SplitSort.cuh:702-938,
whose test -- SplitSortDispatcher -- checks every segment for sortedness; here every segment is compared bit-exactly with
a stable numpy sort, payload = input index so stability is observable).  One thread block sorts one segment in shared
memory; the same kernel serves every osb200_sort_* call with n <= one tile.  -m gpu"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def seg_oracle(keys: np.ndarray, offs: np.ndarray):
    """per-segment stable ascending sort of unsigned keys; returns (keys, permutation of input indices)"""
    out_k = keys.copy()
    out_v = np.arange(keys.size, dtype=np.uint32)
    for a, b in zip(offs[:-1], offs[1:]):
        o = np.argsort(keys[a:b], kind="stable")
        out_k[a:b] = keys[a:b][o]
        out_v[a:b] = (a + o).astype(np.uint32)
    return out_k, out_v


def run_segmented(g, lens, mask, pairs, seed, max_len=None, mode=None):
    rng = np.random.default_rng(seed)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = int(offs[-1])
    keys = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32) & np.uint32(mask)
    wk, wv = seg_oracle(keys, offs)
    with g.OneSweepSorter(max(n, 16), 4, 4 if pairs else 0) as s:
        if mode is not None:
            s.set_option("rank_mode", mode)
        tk = torch.from_numpy(keys.view(np.int32).copy()).cuda()
        tv = torch.arange(n, dtype=torch.int32, device="cuda") if pairs else None
        to = torch.from_numpy(offs).cuda()
        s.segmented_sort(tk, to, tv, max_segment_len=max_len)
        assert np.array_equal(tk.cpu().numpy().view(np.uint32), wk)
        if pairs:
            assert np.array_equal(tv.cpu().numpy().view(np.uint32), wv)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("pairs", [False, True])
def test_segmented_random_lengths(pairs, mode):
    import gpusorting_b200 as g

    with g.OneSweepSorter(16, 4, 0) as s:
        if mode not in ([0, 1] if s.info("atomic_order_ok") else [1]):
            pytest.skip("the atomic rank mode does not keep lane order on this device")
    rng = np.random.default_rng(3)
    # short segments (the 2,048-key geometry), empty ones and single keys included
    lens = rng.integers(0, 2049, 700)
    lens[:6] = [0, 1, 2, 2048, 2047, 0]
    run_segmented(g, lens, 0xFFFFFFFF, pairs, 11, mode=mode)
    run_segmented(g, lens, 0xFF, pairs, 12, mode=mode)  # many ties: stability
    # up to a full tile (the 16,384-key geometry)
    lens = rng.integers(0, 16385, 60)
    lens[:5] = [16384, 16383, 2049, 0, 1]
    run_segmented(g, lens, 0xFFFFFFFF, pairs, 13, mode=mode)
    run_segmented(g, lens, 0xF0F, pairs, 14, mode=mode)


def test_segmented_many_tiny_segments_and_bounds():
    import gpusorting_b200 as g

    run_segmented(g, np.full(50000, 7), 0xFFFFFFFF, True, 21)
    run_segmented(g, np.random.default_rng(5).integers(0, 40, 100000), 0xFFFF, True, 22)
    # a segment longer than the stated bound is left untouched; longer than a tile is refused
    lens = np.array([100, 5000, 100])
    rng = np.random.default_rng(1)
    keys = rng.integers(0, 1 << 32, int(lens.sum()), dtype=np.uint64).astype(np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    with g.OneSweepSorter(1 << 16, 4, 0) as s:
        tk = torch.from_numpy(keys.view(np.int32).copy()).cuda()
        s.segmented_sort(tk, torch.from_numpy(offs).cuda(), max_segment_len=2048)
        got = tk.cpu().numpy().view(np.uint32)
        assert np.array_equal(got[:100], np.sort(keys[:100])) and np.array_equal(got[5100:], np.sort(keys[5100:]))
        assert np.array_equal(got[100:5100], keys[100:5100])
        with pytest.raises(g.OneSweepError):
            s.segmented_sort(tk, torch.from_numpy(offs).cuda(), max_segment_len=16385)


@pytest.mark.parametrize("mode", [0, 1])
def test_small_n_path_equals_the_ordinary_path(oracle, mode):
    """every n up to one tile: one launch of the segment kernel (small_path = 1) against the ordinary multi-kernel path
    (small_path = 0) and the oracle -- keys, pairs, bit ranges, typed descending, u64"""
    import gpusorting_b200 as g

    with g.OneSweepSorter(1 << 15, 4, 4) as s, g.OneSweepSorter(1 << 14, 8, 0) as s8:
        s.set_option("rank_mode", mode)
        s8.set_option("rank_mode", mode)
        cap = s.info("small_path_max_n")
        assert cap == 16384 and s8.info("small_path_max_n") == 8192
        for n in [2, 3, 33, 1000, 2048, 2049, 7680, cap - 1, cap]:
            k = oracle.init_random_u32(n, 0, 500 + n)
            v = np.arange(n, dtype=np.uint32)
            km = k & np.uint32(0x3FF)
            for small in (1, 0):
                s.set_option("small_path", small)
                t = torch.from_numpy(k.view(np.int32).copy()).cuda()
                s.sort_keys(t)
                assert np.array_equal(t.cpu().numpy().view(np.uint32), oracle.sort_keys(k)), (n, small)
                tk, tv = torch.from_numpy(km.view(np.int32).copy()).cuda(), torch.from_numpy(v.view(np.int32).copy()).cuda()
                s.sort_pairs(tk, tv)
                wk, wv = oracle.sort_pairs(km, v)
                assert np.array_equal(tk.cpu().numpy().view(np.uint32), wk) and np.array_equal(tv.cpu().numpy().view(np.uint32), wv), (n, small)
                # bits [5, 17): stable on the other bits
                tk, tv = torch.from_numpy(k.view(np.int32).copy()).cuda(), torch.from_numpy(v.view(np.int32).copy()).cuda()
                s.sort_bits(tk, 5, 17, tv)
                o = np.argsort((k >> np.uint32(5)) & np.uint32(0xFFF), kind="stable")
                assert np.array_equal(tk.cpu().numpy().view(np.uint32), k[o]) and np.array_equal(tv.cpu().numpy().view(np.uint32), v[o]), (n, small)
                # typed: float32 descending
                f = (k.astype(np.int64) - (1 << 31)).astype(np.float32)
                t = torch.from_numpy(f.copy()).cuda()
                s.sort_keys_typed(t, "f32", descending=True)
                assert np.array_equal(t.cpu().numpy(), np.sort(f)[::-1]), (n, small)
            s.set_option("small_path", 1)
            if n <= 8192:
                k8 = oracle.init_random_u64(n, 0, 900 + n)  # random in both words: every one of the 8 digit passes moves keys
                for small in (1, 0):
                    s8.set_option("small_path", small)
                    t = torch.from_numpy(k8.view(np.int64).copy()).cuda()
                    s8.sort_keys(t)
                    assert np.array_equal(t.cpu().numpy().view(np.uint64), np.sort(k8)), (n, small)


@pytest.mark.parametrize("pairs", [False, True])
def test_repeated_exact_sorts_2pow28(pairs):
    """Guards the ranking's order assumptions at a size where tiles outnumber the resident CTAs many times over: a
    development build of the pairs kernel whose lookback ran ahead of the rank phase produced rare order violations that
    only showed at n >= 2^28 and only in some runs.  Several full-size sorts, compared element by
    element with torch's stable sort."""
    import gpusorting_b200 as g

    n = 1 << 28
    sign = -(1 << 31)
    with g.OneSweepSorter(n, 4, 4 if pairs else 0) as s:
        for rep in range(4):
            k = torch.empty(n, dtype=torch.int32, device="cuda")
            v = torch.empty(n, dtype=torch.int32, device="cuda") if pairs else None
            g.init_random(k, 0, 31 + rep, payload=v, payload_is_index=pairs)
            if rep & 1:
                k &= 0xFFFFF  # duplicate-rich: instability shows in the payloads
            want, order = torch.sort(k ^ sign, stable=True)
            want ^= sign
            if pairs:
                s.sort_pairs(k, v)
                assert torch.equal(v.to(torch.int64) & 0xFFFFFFFF, order), f"payload order, rep {rep}"
            else:
                s.sort_keys(k)
            assert torch.equal(k, want), f"keys, rep {rep}"
            del k, v, want, order
            torch.cuda.empty_cache()
