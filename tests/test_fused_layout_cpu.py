"""The layout of a fused sort (DESIGN §4.12), restated in numpy: the region capacity c(n), which sorts are fused, where the
fused first pass puts each key, how the next pass finds it again, and when the fused result stands.  Checked against the
library's workspace size, which holds the 256 regions; tests/test_gpu_fused_first_pass.py checks the rest on the device."""
import numpy as np
import pytest

TILE = 16384          # keys per tile of the u32 keys pass
MIN_TILES = 64        # smaller sorts keep the classic launch plan
RADIX = 256


def region_keys(n):
    """c(n): n/256 plus 1/32 of it plus 1,024 keys, rounded up to whole 128-byte lines"""
    q = (n + 255) // 256
    return (q + q // 32 + 1024 + 31) // 32 * 32


def fused_eligible(n):
    return n < (1 << 32) and (n + TILE - 1) // TILE >= MIN_TILES


def fused_scatter(keys):
    """(alt buffer with -1 in the gaps, kept): what the fused first pass leaves; not kept where a bin overflows its region
    or a tile's place-0 digit holds more than a sixteenth of the tile"""
    n = len(keys)
    c = region_keys(n)
    d = keys & 0xFF
    counts = np.bincount(d, minlength=RADIX)
    pad = (-n) % TILE
    per_tile = np.stack([np.bincount(t, minlength=RADIX) for t in np.split(np.concatenate((d, np.full(pad, -1) % RADIX)), (n + pad) // TILE)])
    per_tile[-1, RADIX - 1] -= pad  # the ragged last tile's padding is not counted
    if counts.max() > c or per_tile.max() > TILE // 16:
        return None, False
    alt = np.full(RADIX * c, -1, dtype=np.int64)
    order = np.argsort(d, kind="stable")
    dense_base = np.concatenate(([0], np.cumsum(counts)[:-1]))
    rank = np.arange(n) - dense_base[d[order]]
    alt[d[order] * c + rank] = keys[order]
    return alt, True


def gapped_read(alt, counts, c):
    """the keys the next pass reads at logical positions 0..n-1: position p of region r (dense range [B0[r], B0[r+1])) is
    at p + r c - B0[r]"""
    n = int(counts.sum())
    dense_base = np.concatenate(([0], np.cumsum(counts)[:-1]))
    p = np.arange(n)
    r = np.searchsorted(dense_base, p, side="right") - 1  # the largest r with B0[r] <= p: never an empty region
    return alt[p + r * c - dense_base[r]]


def test_region_capacity():
    assert region_keys(1 << 30) == 4_326_400
    for n in (1 << 20, 63 * TILE + 1, (1 << 30) + 7, (1 << 32) - 1):
        c = region_keys(n)
        assert c % 32 == 0 and c >= n / 256
        assert RADIX * c * 4 % 128 == 0


def test_threshold():
    assert not fused_eligible(63 * TILE) and fused_eligible(63 * TILE + 1)
    assert fused_eligible((1 << 32) - 1) and not fused_eligible(1 << 32)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gapped_layout_round_trips(seed):
    rng = np.random.default_rng(seed)
    n = 70_001
    counts = rng.integers(0, 2 * n // RADIX, size=RADIX)
    counts[rng.choice(RADIX, 20, replace=False)] = 0
    counts[rng.choice(RADIX, 5, replace=False)] = 1
    d = rng.permutation(np.repeat(np.arange(RADIX), counts))
    keys = (rng.integers(0, 1 << 24, size=len(d)) << 8) | d
    alt, kept = fused_scatter(keys)
    assert kept
    got = gapped_read(alt, np.bincount(d, minlength=RADIX), region_keys(len(d)))
    assert np.array_equal(got, keys[np.argsort(d, kind="stable")])


def test_a_bin_over_capacity_or_a_low_entropy_tile_falls_back():
    n = 1 << 21
    c = region_keys(n)
    keys = np.arange(n, dtype=np.int64) % 255 + 1
    keys[: 16 * c : 16] = 0  # c keys of digit 0, a sixteenth of each of the first tiles
    assert fused_scatter(keys)[1]
    keys[16 * c] = 0
    assert not fused_scatter(keys)[1]
    keys = np.arange(n, dtype=np.int64) % 255 + 1
    keys[TILE : TILE + TILE // 16] = 0
    assert fused_scatter(keys)[1]
    keys[TILE + TILE // 16] = 0
    assert not fused_scatter(keys)[1]


def test_workspace_holds_the_regions():
    import gpusorting_b200 as g

    smallest_tile = 8192  # the handle's descriptors and reductions are sized for the smallest u32 tile of any variant
    control = 2 * 8 * RADIX * 8 + 64 + 64 + 64
    for n in (63 * TILE, 63 * TILE + 1, 1 << 20, (1 << 30) + 5):
        alt = max(n, RADIX * region_keys(n)) if fused_eligible(n) else n
        tiles = (n + smallest_tile - 1) // smallest_tile
        rest = tiles * RADIX * 8 + (tiles + 8) * RADIX * 2 * 4 + control
        assert g.lib.osb200_workspace_bytes(n, 4, 0) == 4 * alt + rest, n
        assert g.lib.osb200_workspace_bytes(n, 4, 4) == 4 * alt + 4 * n + rest, n


WINDOW_N = (1 << 32) - (1 << 20) - 3  # the fused sort of tests/test_gpu_large_n_new_paths.py


def test_regions_reach_past_element_2pow32():
    """the largest fused sorts put their last regions beyond element 2^32 of the alt buffer: at WINDOW_N keys element 2^32
    falls inside region 248, and regions 249-255 start past it"""
    n = WINDOW_N
    c = region_keys(n)
    assert fused_eligible(n) and (n + TILE - 1) // TILE == 262_080 and c == 17_298_304
    assert RADIX * c > 1 << 32 and (1 << 32) // c == 248
    assert 248 * c < (1 << 32) < 249 * c
    # the smallest n whose regions pass element 2^32
    assert RADIX * region_keys(4_164_562_689) > 1 << 32 >= RADIX * region_keys(4_164_562_688)


def test_workspace_holds_the_regions_past_2pow32():
    import gpusorting_b200 as g

    n = WINDOW_N
    alt = RADIX * region_keys(n)
    assert alt > n  # the alt buffer is sized for the regions, not for the n keys
    tiles = (n + 8191) // 8192  # as in test_workspace_holds_the_regions
    rest = tiles * RADIX * 8 + (tiles + 8) * RADIX * 2 * 4 + 2 * 8 * RADIX * 8 + 64 + 64 + 64
    assert g.lib.osb200_workspace_bytes(n, 4, 0) == 4 * alt + rest
