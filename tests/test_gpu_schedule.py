"""The persistent DigitBinningPass's tile schedule.  A CTA's first tile is its block index; every later tile comes from the
pass's ticket, and its keys are loaded while the CTA still works on the tile before.  The option "debug_max_ctas" caps
the grid, so that few CTAs run many tiles each: one CTA must sort everything through tickets alone.  The sizes leave a
ragged last tile, so the prefetch also reads near n.  Every output is compared element by element with the oracle, with
and without stalled tiles (the lookback's fallback re-reduction).  The plain pairs and u64 passes run one CTA per tile and
ignore the cap; their cases check that they still sort right with the option set (their HOT passes are capped).  -m gpu"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CAPS = [1, 3, 0]  # 0: as many CTAs as can be resident
STALLS = [0, 2]


def dev(a):
    return torch.from_numpy(a.view(np.int32 if a.dtype.itemsize == 4 else np.int64).copy()).cuda()


def host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def configure(s, cap, stall):
    s.set_option("debug_max_ctas", cap)
    if stall:
        s.set_option("spin_cap", 16)
        s.set_option("debug_stall_every", stall)


@pytest.mark.parametrize("stall", STALLS)
@pytest.mark.parametrize("cap", CAPS)
def test_keys_with_a_capped_grid(g, oracle, cap, stall):
    n = 7 * 16384 + 1234  # 16,384-key tiles
    k = oracle.init_random_u32(n, 0, 11 + cap)
    with g.OneSweepSorter(n, 4, 0) as s:
        assert s.info("tile_keys") == 16384
        configure(s, cap, stall)
        t = dev(k)
        s.sort_keys(t)
        assert np.array_equal(host(t), oracle.sort_keys(k)), f"keys cap={cap} stall={stall}"


@pytest.mark.parametrize("stall", STALLS)
@pytest.mark.parametrize("cap", CAPS)
def test_pairs_with_a_capped_grid(g, oracle, cap, stall):
    n = 9 * 8192 + 777  # 8,192-pair tiles
    k = oracle.init_random_u32(n, 0, 21 + cap)
    v = np.arange(n, dtype=np.uint32)
    with g.OneSweepSorter(n, 4, 4) as s:
        configure(s, cap, stall)
        tk, tv = dev(k), dev(v)
        s.sort_pairs(tk, tv)
        wk, wv = oracle.sort_pairs(k, v)
        assert np.array_equal(host(tk), wk) and np.array_equal(host(tv), wv), f"pairs cap={cap} stall={stall}"


@pytest.mark.parametrize("stall", STALLS)
@pytest.mark.parametrize("cap", CAPS)
def test_u64_with_a_capped_grid(g, oracle, cap, stall):
    n = 5 * 8192 + 4321  # 8,192-key tiles
    k = oracle.init_random_u64(n, 0, 31 + cap)
    with g.OneSweepSorter(n, 8, 0) as s:
        assert s.info("tile_keys") == 8192
        configure(s, cap, stall)
        t = dev(k)
        s.sort_keys(t)
        assert np.array_equal(host(t, np.uint64), np.sort(k)), f"u64 cap={cap} stall={stall}"


@pytest.mark.parametrize("cap", [1, 3])
def test_typed_keys_with_a_capped_grid(g, cap):
    """The first pass encodes each tile's keys after its prefetch, the last one decodes them in the scatter."""
    n = 16384 * 4 + 99
    f = (np.random.default_rng(cap).standard_normal(n) * 100).astype(np.float32)
    with g.OneSweepSorter(n, 4, 0) as s:
        configure(s, cap, 0)
        t = dev(f.view(np.uint32).copy())
        s.sort_keys_typed(t, "f32", descending=True)
        assert np.array_equal(host(t).view(np.float32), np.sort(f)[::-1])


@pytest.mark.parametrize("cap", [1, 3])
def test_hot_passes_with_a_capped_grid(g, oracle, cap):
    """Low-entropy keys run in the HOT instantiation, which draws its tiles from the same ticket."""
    n = (1 << 22) + 4099
    k = oracle.init_random_u32(n, 4, 5)
    v = np.arange(n, dtype=np.uint32)
    wk, wv = oracle.sort_pairs(k, v)
    with g.OneSweepSorter(n, 4, 4) as s:
        configure(s, cap, 0)
        t = dev(k)
        s.sort_keys(t)
        assert s.info("last_hot_mask") != 0
        assert np.array_equal(host(t), wk)
        tk, tv = dev(k), dev(v)
        s.sort_pairs(tk, tv)
        assert np.array_equal(host(tk), wk) and np.array_equal(host(tv), wv)


def test_debug_max_ctas_rejects_negative_values(g):
    with g.OneSweepSorter(1024, 4, 0) as s:
        with pytest.raises(g.OneSweepError):
            s.set_option("debug_max_ctas", -1)
