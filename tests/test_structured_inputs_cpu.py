"""The structured inputs of tests/test_gpu_structured_inputs.py have the properties they claim, and expected_plan restates
the scan kernel's rule at both sides of each of its edges.

Each generator is run at the sizes and tile sizes the GPU tests use (16,384 keys: u32 keys; 12,288: 16-bit keys; 8,192: u32
pairs and argsort, u64 keys, 16-bit pairs, 64-bit pairs) and checked here, on the CPU: per-tile digit counts (exactly T,
exactly k, no digit of T/8 keys, a tie), where the outlier is, how long the runs are, the global counts at the hot rule's
boundary, and that the plan it promises is expected_plan of its image.  Without these checks a GPU case could pass
without ever reaching the state it is meant to test."""
import numpy as np
import pytest
import torch

from tests import bigcheck, oraclelib
from tests import structured as st

TILES = [16384, 12288, 8192]
LAY = {16: st.layout(16), 32: st.layout(32), 64: st.layout(64)}
WIDTH = {16384: 32, 12288: 16, 8192: 64}  # a key width that tile size serves (8,192 serves every width)


def plan_of(image, lay):
    return st.expected_plan(image, lay.places)


def others_constant(image, lay, p):
    for q, place in enumerate(lay.places):
        if q != p:
            d = st.digit(image, place)
            assert bool((d == d[0]).all()), f"place {q} is not constant"


def check_single(image, plan, lay, p):
    """structure in place p only: the other places are constant, and the promise is the scan kernel's plan"""
    others_constant(image, lay, p)
    assert plan == plan_of(image, lay)
    every = (1 << len(lay.places)) - 1
    assert plan.skip == every & ~(1 << p) and plan.executed == 1


# ---- runs ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", TILES)
def test_runs(T):
    lay = LAY[WIDTH[T]]
    p = len(lay.places) - 1
    lengths = st.run_lengths(T)
    assert {1, 31, 32, 33, 32 * st.KEYS_PER_THREAD[T], T // 8, T - 1, T, T + 1, 3 * T // 2} == set(lengths)
    # the GPU cases: past 2^22 one order per run length, in turn; at 3T + 5 every order
    for n, R, order in ([(st.hot_n(T), R, st.RUN_ORDERS[j % 3]) for j, R in enumerate(lengths)] +
                        [(3 * T + 5, R, order) for R in lengths for order in st.RUN_ORDERS]):
        i = torch.arange(n)
        img, plan = st.runs(n, T, lay, p, R, R, order)
        check_single(img, plan, lay, p)
        assert plan.hot == 0
        d = st.digit(img, lay.places[p])
        # every run is R keys long (the last one may be shorter) and borders sit at multiples of R
        assert bool((d == d[(i // R) * R]).all()), f"R={R} {order}: a run changes its digit"
        if order == "asc":
            assert torch.equal(d, (i // R) % 256)
        elif order == "desc":
            assert torch.equal(d, 255 - (i // R) % 256)


@pytest.mark.parametrize("bits", [1, 3, 5])
def test_runs_and_tile_blocks_in_a_narrow_digit(bits):
    """the few-bins scatter (digits of <= 5 bits): at most 8 bins always make the pass hot, 32 bins do not"""
    T = 8192
    n = st.hot_n(T)
    lay = st.layout(32, 2, 10 + bits)
    assert lay.places[-1] == (10, bits)
    p = len(lay.places) - 1
    for img, plan in (st.runs(n, T, lay, p, 1, T + 1, "random"), st.runs(n, T, lay, p, 2, 33, "asc"),
                      st.tile_blocks(n, T, lay, p, 3)):
        check_single(img, plan, lay, p)
        assert plan.hot == ((1 << p) if bits <= 3 else 0)
        assert int(st.digit(img, lay.places[p]).max()) < 1 << bits
    # bits outside the range are random: they show the order of equal keys
    assert bool(((img >> 10 + bits) != (img[0] >> 10 + bits)).any())


# ---- single-digit tiles --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", TILES)
def test_tile_blocks(T):
    n = st.hot_n(T)
    lay = LAY[WIDTH[T]]
    img, plan = st.tile_blocks(n, T, lay, 0, 5)
    check_single(img, plan, lay, 0)
    assert plan.hot == 0
    c = st.tile_counts(st.digit(img, lay.places[0]), T, 256)
    live = torch.full((c.shape[0],), T)
    live[-1] = n - (c.shape[0] - 1) * T
    assert torch.equal(c.max(1).values, live), "a tile holds more than one digit"
    top = c.argmax(1)
    assert bool((top[1:] == top[:-1]).any()) and bool((top[1:] != top[:-1]).any()), "neighbours always / never share"


# ---- whole keys ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", st.WHOLE_SHAPES)
@pytest.mark.parametrize("width", [16, 32, 64])
def test_whole_keys(width, shape):
    n = st.hot_n(8192)
    lay = LAY[width]
    img, plan = st.whole_keys(n, 8192, lay, 7, shape)
    assert plan == plan_of(img, lay) == st.Plan(0, 0, len(lay.places))
    o = st.ordered(img, width)
    up = o[1:] >= o[:-1]
    down = o[1:] <= o[:-1]
    if shape == "sorted":
        assert bool(up.all())
    elif shape == "reversed":
        assert bool(down.all())
    elif shape == "nearly":
        moved = int((o != torch.sort(o).values).sum())
        assert 0 < moved <= 2 * (n // 100), moved
        assert int((~up).sum()) <= 4 * (n // 100)
    elif shape == "runs8":
        for k in range(8):
            a, b = k * n // 8, (k + 1) * n // 8
            assert bool(up[a:b - 1].all())
        assert 1 <= int((~up).sum()) <= 7
    else:
        h = n // 2
        assert bool(up[: h - 1].all()) and bool(down[h:].all())


# ---- one outlier ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("above", [False, True])
@pytest.mark.parametrize("T", TILES)
def test_outlier(T, above):
    lay = LAY[WIDTH[T]]
    for n in (st.hot_n(T), 3 * T + 5, 777):
        for pos in sorted({x for x in (0, T - 1, T, n - 1) if x < n}):
            img, plan = st.outlier(n, T, lay, 1, 11, pos, above)
            check_single(img, plan, lay, 1)
            d = st.digit(img, lay.places[1])
            odd = torch.nonzero(d != d[(pos + 1) % n]).reshape(-1)
            assert odd.tolist() == [pos]
            assert (int(d[pos]) > int(d[(pos + 1) % n])) == above
            # the scan kernel's skip rule at c = n - 1: executed; hot once n >= 2^22
            assert plan.hot == ((1 << 1) if n >= st.HOT_MIN_N else 0)
        assert n % T, "n - 1 is in a ragged last tile"


# ---- hot digits, global and per tile -------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", TILES)
def test_hot_block(T):
    n = st.hot_n(T)
    lay = LAY[WIDTH[T]]
    extra = T // 3 + 7
    img, plan = st.hot_block(n, T, lay, 0, 13, extra)
    check_single(img, plan, lay, 0)
    assert plan.hot == 1
    d = st.digit(img, lay.places[0])
    m = -(-n // 8) + extra
    assert bool((d[:m] == d[0]).all())
    c = st.tile_counts(d, T, 256)
    after = c[-(-m // T):-1]  # full tiles behind the block
    assert bool((after.max(1).values < T // 8).all()), "a tile behind the block has a hot digit"
    assert after.shape[0] >= 0.8 * c.shape[0], "most tiles have no hot digit"


@pytest.mark.parametrize("T", TILES)
def test_tile_local_hot(T):
    n = st.hot_n(T)
    lay = LAY[WIDTH[T]]
    img, plan = st.tile_local_hot(n, T, lay, 0, 17)
    check_single(img, plan, lay, 0)
    assert plan.hot == 1
    d = st.digit(img, lay.places[0])
    h = int(d[0])
    lead = st._ceil(st._ceil(n, 8), T)
    c = st.tile_counts(d, T, 256)
    assert bool((c[:lead, h] == T).all()) and int(c[:, h].sum()) * 8 >= n
    full = c[lead:-1]
    top2 = full.topk(2, dim=1)
    m = top2.indices[:, 0]
    assert bool((m != h).all()), "a tile's own hot digit is the global one"
    assert bool((top2.values[:, 0] >= T // 8).all()) and bool((top2.values[:, 1] < T // 8).all())
    assert set(top2.values[:, 0].tolist()) == set(st.local_hot_counts(T))


@pytest.mark.parametrize("lead", [False, True])
@pytest.mark.parametrize("below", [False, True])
@pytest.mark.parametrize("T", TILES)
def test_tile_threshold(T, below, lead):
    n = st.whole_tiles_n(T)
    assert n >= st.HOT_MIN_N and n % (8 * T) == 0
    lay = LAY[WIDTH[T]]
    k = T // 8 - below
    img, plan = st.tile_threshold(n, T, lay, 0, 19, k, lead)
    check_single(img, plan, lay, 0)
    assert plan.hot == (1 if lead or not below else 0)
    d = st.digit(img, lay.places[0])
    c = st.tile_counts(d, T, 256)
    body = c[n // 8 // T:] if lead else c
    top2 = body.topk(2, dim=1)
    assert bool((top2.values[:, 0] == k).all()), "a tile does not hold exactly k keys of its digit"
    assert bool((top2.indices[:, 0] == top2.indices[0, 0]).all())
    assert bool((top2.values[:, 1] < k).all())
    m = int(top2.indices[0, 0])
    if lead:
        h = int(d[0])
        assert h != m and bool((c[: n // 8 // T, h] == T).all()) and int((d == h).sum()) == n // 8
    else:  # the global bin of m at the hot rule's edge: 8c == n, or below it
        assert 8 * int((d == m).sum()) == (n if not below else n - 8 * (n // T))


@pytest.mark.parametrize("T", TILES)
def test_tile_tie(T):
    n = st.whole_tiles_n(T)
    lay = LAY[WIDTH[T]]
    img, plan = st.tile_tie(n, T, lay, 0, 23)
    check_single(img, plan, lay, 0)
    assert plan.hot == 1
    c = st.tile_counts(st.digit(img, lay.places[0]), T, 256)
    top3 = c.topk(3, dim=1)
    assert bool((top3.values[:, 0] == top3.values[:, 1]).all()) and bool((top3.values[:, 0] >= T // 8).all())
    assert bool((top3.values[:, 2] < T // 8).all())
    assert set(top3.values[:, 0].tolist()) == set(st.tie_counts(T))
    pair = top3.indices[:, :2].sort(1).values
    assert bool((pair == pair[0]).all())


@pytest.mark.parametrize("n,c,hot", [(1 << 22, 1 << 19, True), (1 << 22, (1 << 19) - 1, False),
                                     ((1 << 22) - 1, 1 << 19, False)])
def test_global_boundary(n, c, hot):
    lay = LAY[32]
    img, plan = st.global_boundary(n, 16384, lay, 2, 29, c)
    check_single(img, plan, lay, 2)
    assert plan.hot == (4 if hot else 0)
    counts = torch.bincount(st.digit(img, lay.places[2]), minlength=256)
    assert int(counts.max()) == c and int((counts == c).sum()) == 1


# ---- expected_plan at its edges ------------------------------------------------------------------------------------------
def test_expected_plan_edges():
    lay = st.layout(32, 0, 11)  # places (0, 8) and (8, 3): the narrow last digit counts as a place
    assert lay.places == ((0, 8), (8, 3))
    # skip rule: c == n against c == n - 1
    n = 1000
    img = torch.full((n,), 0x5A5, dtype=torch.int64)
    assert st.expected_plan(img, lay.places) == st.Plan(3, 0, 0)
    img[n - 1] = 0x3A5  # the narrow digit differs in one key
    assert st.expected_plan(img, lay.places) == st.Plan(1, 0, 1)
    img[0] = 0x3A4  # and the low digit in one key
    assert st.expected_plan(img, lay.places) == st.Plan(0, 0, 2)
    # hot rule: 8c == n against 8c == n - 1 (n >= 2^22), and n = 2^22 - 1 against 2^22
    for n, c, hot in ((st.HOT_MIN_N + 8, (st.HOT_MIN_N + 8) // 8, True), (st.HOT_MIN_N + 9, (st.HOT_MIN_N + 8) // 8, False),
                      (st.HOT_MIN_N, st.HOT_MIN_N // 2, True), (st.HOT_MIN_N - 1, st.HOT_MIN_N // 2, False)):
        d = torch.arange(n, dtype=torch.int64) % 255 + 1  # no other bin comes near n/8
        d[:c] = 0
        img = d | (d % 8) << 8  # the 3-bit place has 8 bins: one holds n/8 keys, hot from 2^22
        want_hot = (1 if hot else 0) | (2 if n >= st.HOT_MIN_N else 0)
        assert st.expected_plan(img, lay.places) == st.Plan(0, want_hot, 2), (n, c)
    # a place of one bin and n keys is skipped, not hot
    img = torch.full((st.HOT_MIN_N,), 7, dtype=torch.int64)
    assert st.expected_plan(img, lay.places) == st.Plan(3, 0, 0)
    # and a place where one key differs is hot
    img[5] = 8
    assert st.expected_plan(img, lay.places) == st.Plan(2, 1, 1)


# ---- the typed bits ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("kind", ["u", "i", "f"])
def test_to_bits_inverts_to_radix(kind, descending):
    """to_bits agrees with oraclelib.from_radix, and the image is the radix image of the bits it makes"""
    rng = np.random.default_rng(31)
    for width, utype in ((32, np.uint32), (64, np.uint64)):
        u = rng.integers(0, np.iinfo(utype).max, 4099, dtype=utype, endpoint=True)
        u[:4] = [0, 1, np.iinfo(utype).max, np.iinfo(utype).max >> 1]
        img = torch.from_numpy(u.view(np.int64 if width == 64 else np.uint32).astype(np.int64))
        bits = st.to_bits(img, width, kind, descending).numpy().view(utype)
        assert np.array_equal(bits, oraclelib.from_radix(u, kind, descending))
        assert np.array_equal(oraclelib.to_radix(bits, kind, descending), u)
    img = torch.arange(1 << 16, dtype=torch.int64)
    bits = st.to_bits(img, 16, kind, descending)
    assert torch.equal(bigcheck.radix16(bits, kind + "16", descending), img.to(torch.int32))
