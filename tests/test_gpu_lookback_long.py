"""The lookback of the u32 keys DigitBinningPass (lookback_wide: a window of 16 predecessor tiles per round trip) on sorts
long enough to fill that window many times over: 129 tiles of 16,384 keys, the last one ragged.  Stalled tiles
(debug_stall_every, spin_cap 16) withhold their reductions at periods shorter and longer than the window and than one
block of 8 tiles, so the walk stops, re-reduces and publishes on the owner's behalf at every position of a window; the grid
cap (debug_max_ctas) runs the tiles from one CTA, a few, or a full grid.  Both rank modes, typed descending keys and a bit
range.  Every output is compared element by element with the oracle.  -m gpu"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N = (1 << 21) + 12345  # 129 tiles
STALLS = [2, 3, 9, 17, 31, 33]
CAPS = [1, 3, 0]  # 0: as many CTAs as can be resident


def dev(a):
    return torch.from_numpy(a.view(np.int32).copy()).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32)


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


@pytest.fixture(scope="module")
def sorter(g):
    with g.OneSweepSorter(N, 4, 0) as s:
        assert s.info("tile_keys") == 16384
        yield s


def rank_modes(s):
    return [0, 1] if s.info("atomic_order_ok") else [1]


def configure(s, cap, stall, mode):
    s.set_option("rank_mode", mode)
    s.set_option("debug_max_ctas", cap)
    s.set_option("spin_cap", 16)
    s.set_option("debug_stall_every", stall)


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("stall", STALLS)
def test_keys_with_stalled_tiles(sorter, oracle, stall, cap):
    k = oracle.init_random_u32(N, 0, 100 + stall)
    want = oracle.sort_keys(k)
    for mode in rank_modes(sorter):
        configure(sorter, cap, stall, mode)
        t = dev(k)
        sorter.sort_keys(t)
        assert np.array_equal(host(t), want), f"stall_every={stall} max_ctas={cap} rank_mode={mode}"


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("stall", [3, 17])
def test_typed_descending_keys_with_stalled_tiles(sorter, stall, cap):
    """The first pass re-reduces stalled tiles over the ENCODED keys; the last one decodes in the scatter."""
    f = (np.random.default_rng(stall).standard_normal(N) * 100).astype(np.float32)
    want = np.sort(f)[::-1]
    for mode in rank_modes(sorter):
        configure(sorter, cap, stall, mode)
        t = dev(f.view(np.uint32).copy())
        sorter.sort_keys_typed(t, "f32", descending=True)
        assert np.array_equal(host(t).view(np.float32), want), f"stall_every={stall} max_ctas={cap} rank_mode={mode}"


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("stall", [9, 31])
def test_bit_range_with_stalled_tiles(sorter, oracle, stall, cap):
    """A sort on bits [5, 27): three digit passes, the last one narrower than 8 bits."""
    begin, end = 5, 27
    k = oracle.init_random_u32(N, 0, 200 + stall)
    want = k[np.argsort((k >> np.uint32(begin)) & np.uint32((1 << (end - begin)) - 1), kind="stable")]
    for mode in rank_modes(sorter):
        configure(sorter, cap, stall, mode)
        t = dev(k)
        sorter.sort_bits(t, begin, end)
        assert np.array_equal(host(t), want), f"stall_every={stall} max_ctas={cap} rank_mode={mode}"


@pytest.mark.parametrize("cap", CAPS)
def test_keys_without_stalls(sorter, oracle, cap):
    k = oracle.init_random_u32(N, 0, 7)
    want = oracle.sort_keys(k)
    for mode in rank_modes(sorter):
        configure(sorter, cap, 0, mode)
        t = dev(k)
        sorter.sort_keys(t)
        assert np.array_equal(host(t), want), f"max_ctas={cap} rank_mode={mode}"
