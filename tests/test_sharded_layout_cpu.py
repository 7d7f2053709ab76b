"""The sharded sort's host-side exchange layout (osb200_sharded_exchange_layout) against a plain restatement of both plans,
for world sizes 1 to 64, over random and adversarial histograms.  CPU only: the layout is a pure function of the
all-gathered histograms, and osb200_sharded_sort_keys_u32 runs exactly this function on every rank."""
import ctypes

import numpy as np
import pytest

ADDR0 = 0x7F3A_0000_0000  # receive buffers at plausible device addresses, 4-byte aligned but not line aligned


def capacity(max_n_local, slack_percent):
    return max_n_local + max_n_local // 100 * slack_percent + 4096


def ref_fine_dest(hist):
    """Greedy contiguous split: bucket d goes to the rank whose ideal share contains the bucket's midpoint, in exact
    rational arithmetic (the library's long double computes the same floor for these magnitudes)."""
    world = hist.shape[0]
    bucket = [int(x) for x in hist.sum(axis=0, dtype=np.uint64)]
    total = sum(bucket)
    dest, before, prev = [], 0, 0
    for d in range(256):
        q = prev
        if total:
            q = max(prev, min(world - 1, (2 * before + bucket[d]) * world // (2 * total)))
        dest.append(q)
        prev = q
        before += bucket[d]
    return np.array(dest, np.int64)


def ref_layout(hist, capacity_, force_fine, recv_addrs):
    """Every rank's layout as int64 arrays [world, ...], or None where the library must return OSB200_ERR_SIZE."""
    world = hist.shape[0]
    h = hist.astype(np.int64)  # the cases stay below 2^52 keys in all
    k = max(world - 1, 0).bit_length()
    coarse = world > 1 and (1 << k) == world and not force_fine
    if coarse:
        per = 256 >> k
        bin_hist = np.zeros((world, 256), np.int64)
        bin_hist[:, :world] = h.reshape(world, world, per).sum(axis=2)  # [source, coarse bin]
        coarse = bool((bin_hist.sum(axis=0) <= capacity_).all())
    if coarse:
        xshift, bins = 32 - k, world
        dest = np.minimum(np.arange(256), world - 1)
        bin_of = np.arange(256) // per  # fine bucket -> coarse bin
    else:
        xshift, bins = 24, 256
        bin_hist = h
        dest = ref_fine_dest(hist)
        bin_of = np.arange(256)
    onehot = (dest[:, None] == np.arange(world)[None, :]).astype(np.int64)  # [bin, destination]
    col = bin_hist.sum(axis=0)
    recv_count = col @ onehot
    if (recv_count > capacity_).any():
        return None
    # bucket-major, source-minor: a bin's keys follow the earlier bins of its destination, and within the bin the sources
    # come in rank order
    excl = np.cumsum(col) - col
    first_bin = np.array([np.flatnonzero(dest == q)[0] if (dest == q).any() else 0 for q in range(world)])
    prior = excl - excl[first_bin[dest]]
    recv_off = prior[None, :] + np.cumsum(bin_hist, axis=0) - bin_hist
    if coarse:
        recv_off[:, world:] = 0
    send_cnt = bin_hist @ onehot  # [source, destination]
    recv_from = h @ onehot[bin_of]  # [source, destination] counted from the fine histograms
    zero = np.zeros((world, 1), np.int64)
    addrs = np.asarray(recv_addrs, np.int64)
    return {"xshift": xshift, "bins": bins, "dest": dest, "recv_count": recv_count, "recv_off": recv_off,
            "pass_hist": bin_hist, "out_base": addrs[dest][None, :] // 4 + recv_off,
            "send_off": np.hstack([zero, np.cumsum(send_cnt, axis=1)]),
            "recv_from_off": np.hstack([zero, np.cumsum(recv_from.T, axis=1)])}


def layout_all(hist, capacity_, force_fine, recv_addrs=None):
    """The library's layout for every rank: a list of dicts, or of the status each rank returned."""
    from gpusorting_b200 import OneSweepError, sharded

    res = []
    for r in range(hist.shape[0]):
        try:
            res.append(sharded.exchange_layout(hist, r, capacity_, force_fine, recv_addrs))
        except OneSweepError as e:
            res.append(e.status)
    return res


def check_case(hist, capacity_, force_fine):
    world = hist.shape[0]
    addrs = np.array([ADDR0 + q * (1 << 33) + 4 * (2 * q + 1) for q in range(world)], np.uint64)
    got = layout_all(hist, capacity_, force_fine, addrs)
    want = ref_layout(hist, capacity_, force_fine, addrs)
    if want is None:
        assert got == [-2] * world, "every rank returns OSB200_ERR_SIZE together"
        return "size"
    assert all(isinstance(g, dict) for g in got), got
    for r, g in enumerate(got):
        assert (g["xshift"], g["bins"]) == (want["xshift"], want["bins"])
        for key in ("dest", "recv_count"):
            assert np.array_equal(g[key].astype(np.int64), want[key]), (r, key)
        for key in ("recv_off", "pass_hist", "out_base", "send_off", "recv_from_off"):
            assert np.array_equal(g[key].astype(np.int64), want[key][r]), (r, key)

    # properties, independently of the restatement
    k = max(world - 1, 0).bit_length()
    per = 256 >> k
    coarse_fits = world > 1 and (1 << k) == world and bool(
        (hist.reshape(world, world, per).sum(axis=(0, 2), dtype=np.uint64) <= capacity_).all())
    g0 = got[0]
    bins, dest = g0["bins"], g0["dest"].astype(np.int64)
    # coarse exactly when the world is a power of two > 1, force_fine is off and every coarse bin fits; else fine
    assert (bins, g0["xshift"]) == ((world, 32 - k) if coarse_fits and not force_fine else (256, 24))
    for g in got[1:]:  # every rank derives the same destinations and counts
        assert np.array_equal(g["dest"], g0["dest"]) and np.array_equal(g["recv_count"], g0["recv_count"])
        assert (g["bins"], g["xshift"]) == (bins, g0["xshift"])
    assert (np.diff(dest) >= 0).all() and dest.min() >= 0 and dest.max() < world
    assert int(g0["recv_count"].sum()) == int(hist.sum(dtype=np.uint64))
    assert (g0["recv_count"] <= capacity_).all()
    for r, g in enumerate(got):  # pass_hist is the rank's count of the pass's digit
        if bins == 256:
            assert np.array_equal(g["pass_hist"], hist[r])
        else:
            assert np.array_equal(g["pass_hist"][:world], hist[r].reshape(world, per).sum(axis=1))
            assert not g["pass_hist"][world:].any()
    # the (bin, source) slots tile every destination exactly, without overlap, and the bases encode them
    starts = np.stack([g["recv_off"] for g in got]).astype(np.int64)
    lens = np.stack([g["pass_hist"] for g in got]).astype(np.int64)
    for q in range(world):
        sel = (dest[None, :] == q) & (lens > 0)
        s, n = starts[sel], lens[sel]
        o = np.argsort(s, kind="stable")
        s, n = s[o], n[o]
        assert s.size == 0 or s[0] == 0
        assert np.array_equal(s[1:], (s + n)[:-1]), f"slots at destination {q} overlap or leave a gap"
        assert int(n.sum()) == int(g0["recv_count"][q])
    for g in got:
        assert np.array_equal(g["out_base"], addrs[dest] // np.uint64(4) + g["recv_off"])
    # staged: what r sends to q is what q expects from r; the send ranges tile r's bin-major pass output
    sent = np.stack([np.diff(g["send_off"].astype(np.int64)) for g in got])  # [source, destination]
    expected = np.stack([np.diff(g["recv_from_off"].astype(np.int64)) for g in got])  # [destination, source]
    assert (sent >= 0).all() and np.array_equal(sent, expected.T)
    assert np.array_equal(sent.sum(axis=1), hist.sum(axis=1, dtype=np.uint64).astype(np.int64))
    assert np.array_equal(expected.sum(axis=1), g0["recv_count"].astype(np.int64))
    return "coarse" if bins != 256 else "fine"


def histograms(world, rng):
    """(name, hist[world, 256]) cases: random and adversarial."""
    cases = []
    h = rng.integers(0, 1000, size=(world, 256)).astype(np.uint64)
    h[:, 40:50] = 0
    cases.append(("uniform", h))
    cases.append(("empty", np.zeros((world, 256), np.uint64)))
    h = np.zeros((world, 256), np.uint64)
    h[:, 0] = rng.integers(0, 50, size=world)
    cases.append(("one_bucket_low", h))
    h = np.zeros((world, 256), np.uint64)
    h[:, 255] = 7
    cases.append(("one_bucket_high", h))
    h = np.zeros((world, 256), np.uint64)
    h[:, 0x42] = 100_000  # one top byte: fits one rank's buffer only for two ranks and 100 % slack, else SIZE
    cases.append(("one_bucket_full", h))
    h = rng.integers(0, 1000, size=(world, 256)).astype(np.uint64)
    h[0, 64:] = 0  # rank 0 holds only small keys
    cases.append(("skewed_rank0", h))
    h = np.zeros((world, 256), np.uint64)
    h[:, :64] = rng.integers(100, 200, size=(world, 64))  # all keys below 2^30, spread over that quarter's 64 top bytes
    cases.append(("one_quarter", h))
    h = rng.integers(0, 3, size=(world, 256)).astype(np.uint64) * (rng.random((world, 256)) < 0.05)
    cases.append(("sparse", h.astype(np.uint64)))
    h = rng.integers(1 << 36, 1 << 37, size=(world, 256)).astype(np.uint64)  # bases and offsets far beyond 2^32
    cases.append(("huge", h))
    return cases


@pytest.mark.parametrize("world", list(range(1, 65)))
def test_layout_matches_restatement(world):
    rng = np.random.default_rng(1000 + world)
    for name, hist in histograms(world, rng):
        n_local = hist.sum(axis=1, dtype=np.uint64)
        max_n = max(int(n_local.max()), 1)
        for slack in (0, 12, 50, 100):
            for force_fine in (False, True):
                check_case(hist, capacity(max_n, slack), force_fine)
        # the capacity at the edge of the coarse split: exactly enough, then one key short (falls back to fine or SIZE)
        k = max(world - 1, 0).bit_length()
        if world > 1 and (1 << k) == world:
            need = int(hist.reshape(world, world, -1).sum(axis=(0, 2)).max())
            assert check_case(hist, need, False) == "coarse"
            if need > 0:
                assert check_case(hist, need - 1, False) in ("fine", "size")


def test_outcomes_named_in_the_sort():
    """The cases the sharded sort documents: coarse when it fits, fine when one coarse bin overflows, SIZE for all."""
    from gpusorting_b200 import OneSweepError, sharded

    n = 1 << 20
    world = 4
    uniform = np.full((world, 256), n // 256, np.uint64)
    lay = sharded.exchange_layout(uniform, 1, capacity(n, 12))
    assert (lay["bins"], lay["xshift"]) == (4, 30)
    # every key below 2^30: the coarse split sends everything to rank 0, 4 n > 1.5 n; the 64 top bytes spread over 4 ranks
    quarter = np.zeros((world, 256), np.uint64)
    quarter[:, :64] = n // 64
    lay = sharded.exchange_layout(quarter, 2, capacity(n, 50))
    assert (lay["bins"], lay["xshift"]) == (256, 24)
    assert lay["recv_count"].max() <= capacity(n, 50)
    # one top byte: no split fits
    one = np.zeros((world, 256), np.uint64)
    one[:, 0x42] = n
    for r in range(world):
        with pytest.raises(OneSweepError) as e:
            sharded.exchange_layout(one, r, capacity(n, 50))
        assert e.value.status == -2
    # every key equal, two ranks, 100 % slack: everything goes to one rank and still fits
    eq = np.zeros((2, 256), np.uint64)
    eq[:, 0x7F] = n
    lay = sharded.exchange_layout(eq, 1, capacity(n, 100))
    assert lay["bins"] == 2 and list(lay["recv_count"]) == [2 * n, 0]
    assert lay["recv_off"][0] == n  # rank 1's keys follow rank 0's


def test_fine_layout_is_the_plan():
    from gpusorting_b200 import sharded

    rng = np.random.default_rng(5)
    for world in (1, 3, 8, 64):
        hist = rng.integers(0, 5000, size=(world, 256)).astype(np.uint64)
        for r in range(world):
            dest, recv_count, recv_off = sharded.plan(hist, r)
            lay = sharded.exchange_layout(hist, r, 1 << 40, force_fine=True)
            assert np.array_equal(lay["dest"], dest) and np.array_equal(lay["recv_count"], recv_count)
            assert np.array_equal(lay["recv_off"], recv_off)


def test_capacity_formula_and_bad_arguments():
    import gpusorting_b200 as g
    from gpusorting_b200 import sharded

    for n, slack in ((1, 0), (99, 50), (1 << 30, 12), (12345, 400)):
        assert sharded.capacity(n, slack) == capacity(n, slack)
    assert g.lib.osb200_sharded_capacity(100, -1) == 0 and g.lib.osb200_sharded_capacity(100, 401) == 0
    hist = np.ones((4, 256), np.uint64)
    with pytest.raises(g.OneSweepError) as e:
        sharded.exchange_layout(hist, 4, 1 << 20)  # rank out of range
    assert e.value.status == -1
    with pytest.raises(g.OneSweepError) as e:
        sharded.exchange_layout(hist, 0, 1 << 20, recv_addrs=[ADDR0, ADDR0 + 2, ADDR0, ADDR0])  # not 4-byte aligned
    assert e.value.status == -1
    with pytest.raises(g.OneSweepError) as e:
        sharded.exchange_layout(np.ones((65, 256), np.uint64), 0, 1 << 20)
    assert e.value.status == -1
    # out_base without receive addresses (and the reverse) is refused
    buf = (ctypes.c_uint64 * 1024)()
    p = ctypes.addressof(buf)
    args = [p, 4, 0, 1 << 20, 0]
    outs = [p + 8 * 300, p + 8 * 301, p + 8 * 302, p + 8 * 560, p + 8 * 570, p + 8 * 830]  # xshift .. pass_hist
    assert g.lib.osb200_sharded_exchange_layout(*args, None, *outs, p + 8 * 10, p + 8 * 20, p + 8 * 30) == -1
    assert g.lib.osb200_sharded_exchange_layout(*args, p, *outs, None, p + 8 * 20, p + 8 * 30) == -1
