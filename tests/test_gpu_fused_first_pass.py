"""The fused first pass of whole-key u32 keys-only sorts (DESIGN §4.12): the first digit pass counts the global histogram
and scatters digit d into the fixed region [d c, (d + 1) c) of the alt buffer; the next executed pass reads that gapped
layout; a place-0 bin of more than c keys falls back to the classic GlobalHistogram, Scan and first pass.

Every case is sorted with the fused path on and off and compared element by element with numpy; the plan (skipped, hot
and executed passes) must be the classic plan, and last_fused_kept must say which of the two results stood.  -m gpu"""
import numpy as np
import pytest
import torch

from tests.test_fused_layout_cpu import TILE, fused_eligible, region_keys

pytestmark = pytest.mark.gpu

N = 1 << 21  # 128 tiles


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32).copy()).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32)


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


@pytest.fixture()
def sorter(g):
    s = g.OneSweepSorter((1 << 22) + (1 << 16), 4, 0)
    yield s
    s.close()


def plan_of(s):
    return s.info("last_skip_mask"), s.info("last_hot_mask"), s.info("last_executed_passes")


def sort_both(s, keys, sort=lambda s, t: s.sort_keys(t)):
    """(output, kept, plan) with the fused path on, then off"""
    out = []
    for fused in (1, 0):
        s.set_option("fused_histogram", fused)
        t = dev(keys)
        sort(s, t)
        out.append((host(t), s.info("last_fused_kept"), plan_of(s)))
    s.set_option("fused_histogram", 1)
    return out


def check(s, keys, kept, want=None, sort=lambda s, t: s.sort_keys(t)):
    (on, k_on, plan_on), (off, k_off, plan_off) = sort_both(s, keys, sort)
    want = np.sort(keys, kind="stable") if want is None else want
    assert np.array_equal(on, want) and np.array_equal(off, want)
    assert k_on == kept and k_off == 0
    assert plan_on == plan_off


WINDOW = 16 * TILE  # a bin's keys spread over 16 tiles: ~600 per tile at n = 2^21, below the T/16 of a low-entropy tile


def with_place0_bin(n, count, start, seed, b=7):
    """random keys whose place-0 bin b holds `count` keys, at random positions of [start, start + WINDOW)"""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    low = rng.integers(0, 255, size=n).astype(np.uint32)
    low += low >= b  # uniform over the other 255 bins
    k = (k & np.uint32(0xFFFFFF00)) | low
    pos = start + rng.choice(WINDOW, count, replace=False)
    k[pos] = (k[pos] & np.uint32(0xFFFFFF00)) | np.uint32(b)
    return k


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("extra", [0, 1])
def test_region_of_exactly_c_keys_and_one_more(sorter, where, extra):
    """the overflow (extra = 1) shows in the first tiles, in the middle ones or in the last ones"""
    count = region_keys(N) + extra
    start = {"first": 0, "middle": N // 2 - WINDOW // 2, "last": N - WINDOW}[where]
    k = with_place0_bin(N, count, start, 11)
    check(sorter, k, kept=1 - extra)


@pytest.mark.parametrize("tile", [0, 77, 127])
def test_a_low_entropy_tile_stops_the_fused_pass(sorter, tile):
    """a tile whose place-0 digit holds more than a sixteenth of its keys stops the fused pass, although no region overflows"""
    rng = np.random.default_rng(tile)
    k = rng.integers(0, 1 << 32, size=N, dtype=np.uint64).astype(np.uint32)
    k = (k & np.uint32(0xFFFFFF00)) | rng.integers(1, 256, size=N).astype(np.uint32)  # digit 0 nowhere ...
    lo = tile * TILE
    k[lo:lo + TILE // 16 + 1] &= np.uint32(0xFFFFFF00)  # ... but in T/16 + 1 keys of one tile
    check(sorter, k, kept=0)
    k[lo + TILE // 16] |= np.uint32(1)  # exactly a sixteenth
    check(sorter, k, kept=1)


def test_region_boundaries_inside_tiles_and_warps_and_empty_regions(sorter):
    """place-0 bins of irregular sizes: regions that end inside a tile and inside a warp's 32 keys, empty regions and
    one-key regions, so that the gapped pass looks regions up key by key"""
    rng = np.random.default_rng(5)
    c = region_keys(N)
    counts = np.zeros(256, dtype=np.int64)
    empty = rng.choice(256, 16, replace=False)
    rest = rng.permutation(np.setdiff1d(np.arange(256), empty))
    single, full = rest[:8], rest[8:]
    counts[single] = 1
    r = N - 8
    counts[full] = r // len(full)
    counts[full[: r % len(full)]] += 1
    wiggle = rng.integers(0, 300, size=len(full) // 2)
    counts[full[0::2][: len(wiggle)]] += wiggle
    counts[full[1::2][: len(wiggle)]] -= wiggle
    assert counts.sum() == N and counts.max() <= c and (counts % 32 != 0).any()
    low = rng.permutation(np.repeat(np.arange(256, dtype=np.uint32), counts))
    k = (rng.integers(0, 1 << 24, size=N, dtype=np.uint32) << np.uint32(8)) | low
    check(sorter, k, kept=1)


@pytest.mark.parametrize("case", ["place1_hot", "place1_skipped", "places123_skipped"])
def test_gapped_source_read_by_a_later_place(sorter, case):
    n = (1 << 22) + 4099  # hot passes need n >= 2^22
    rng = np.random.default_rng(3)
    k = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    if case == "place1_hot":
        k[rng.random(n) < 0.3] &= np.uint32(0xFFFF00FF)
    elif case == "place1_skipped":
        k = (k & np.uint32(0xFFFF00FF)) | np.uint32(0x5A00)
    else:  # only place 0 executes: the fused result cannot stand (it would leave the keys gapped)
        k = (k & np.uint32(0xFF)) | np.uint32(0x12345600)
    check(sorter, k, kept=0 if case == "places123_skipped" else 1)
    if case == "place1_hot":
        assert sorter.info("last_hot_mask") & 2
    elif case == "place1_skipped":
        assert sorter.info("last_skip_mask") == 2


def test_typed_keys(sorter):
    rng = np.random.default_rng(8)
    x = rng.integers(-(1 << 31), 1 << 31, size=N + 333, dtype=np.int64).astype(np.int32)
    check(sorter, x.view(np.uint32), kept=1, want=np.sort(x)[::-1].view(np.uint32),
          sort=lambda s, t: s.sort_keys_typed(t, "i32", descending=True))
    f = rng.standard_normal(N + 17).astype(np.float32)
    check(sorter, f.view(np.uint32), kept=1, want=np.sort(f).view(np.uint32),
          sort=lambda s, t: s.sort_keys_typed(t, "f32"))


@pytest.mark.parametrize("option,value", [("debug_stall_every", 7), ("debug_max_ctas", 1), ("debug_max_ctas", 3),
                                          ("rank_mode", 1), ("short_circuit", 0)])
@pytest.mark.parametrize("overflow", [False, True])
def test_options(sorter, option, value, overflow):
    if option == "debug_stall_every":
        sorter.set_option("spin_cap", 64)
    sorter.set_option(option, value)
    c = region_keys(N)
    k = with_place0_bin(N, c + 1 if overflow else 1000, N // 3, 21)
    k[: N // 2] &= np.uint32(0xFFFF00FF)  # place 1 hot-ish in the first half: more work for the gapped pass's ranking
    check(sorter, k, kept=0 if overflow else 1)


@pytest.mark.parametrize("n", [63 * TILE, 63 * TILE + 1, 64 * TILE + 1, 200 * TILE - 5])
def test_sizes_around_the_threshold(sorter, n):
    k = np.random.default_rng(n).integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    check(sorter, k, kept=1 if fused_eligible(n) else 0)


def test_graph_replays_alternating_kept_and_fallback(g, sorter):
    n = N
    uniform = np.random.default_rng(1).integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    overflow = with_place0_bin(n, region_keys(n) + 1, n - WINDOW, 2)
    work = dev(uniform)
    sorter.sort_keys(work)  # kernels configured and loaded before the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sorter.sort_keys(work)
    for i in range(4):
        src = uniform if i % 2 == 0 else overflow
        work.copy_(dev(src))
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(host(work), np.sort(src)), i
        assert sorter.info("last_fused_kept") == (1 if i % 2 == 0 else 0), i


def test_past_2_31_keys(g):
    n = (1 << 31) + 12345
    free, _ = torch.cuda.mem_get_info()
    if free < 26 * (1 << 30):
        pytest.skip("needs ~26 GiB of free device memory")
    s = g.OneSweepSorter(n, 4, 0)
    try:
        t = torch.empty(n, dtype=torch.int32, device="cuda")
        g.init_random(t, 0, 77)

        def summary(t):  # the key sum and the histogram of the low 16 bits, in chunks (no n-sized temporaries)
            total, hist = 0, torch.zeros(1 << 16, dtype=torch.int64, device="cuda")
            for c in torch.split(t, 1 << 27):
                total += int(c.to(torch.int64).sum())
                hist += torch.bincount((c & 0xFFFF).to(torch.int64), minlength=1 << 16)
            return total, hist

        before = summary(t)
        s.sort_keys(t)
        assert s.info("last_fused_kept") == 1
        assert s.validate(t) == 0
        after = summary(t)
        assert after[0] == before[0] and torch.equal(after[1], before[1])
        del t
    finally:
        s.close()
        torch.cuda.empty_cache()
