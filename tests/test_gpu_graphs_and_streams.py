"""Sorts captured in CUDA graphs, sorts running concurrently, and the descriptor epochs both depend on.  -m gpu

The chained scan's inclusive descriptors are not cleared between eager sorts: every word carries the epoch of the pass
that wrote it, and the host hands each pass a new epoch.  A graph replays the epochs of its capture, so a captured sort
clears its descriptors before its first pass and after its last.  Every pass overwrites the descriptors of all its tiles,
so a replay meets words of its own epoch where the previous replay's last executed pass is the same digit place as its
own first executed one.  The input sequences below are ordered to produce that: keys whose top byte alone varies (only
the last pass runs) follow uniform keys, uniform keys follow keys whose low byte alone varies (only the first pass runs).
Between them come inputs that change the device plan in other ways: entropy preset 4 (AND of 4 words) runs the HOT
passes, a constant top byte skips one pass (an odd number of executed passes: the copy-back runs), all-equal keys skip
every pass.  Each graph case captures one call and replays it at least four times, with different contents copied into
the static tensors before every replay, and checks the plan each replay ran.  The epoch cases move the handle's epoch
counter (option "debug_epoch") across the wrap-around and back onto the epochs of a captured sort.  The concurrent cases
enqueue everything first and check every result at the end.

Every output is compared element by element with an independent answer (numpy's stable argsort, or torch.sort with
stable=True on sign-flipped keys); pairs carry payload = input index, so stability shows."""
import numpy as np
import pytest
import torch

from tests.oraclelib import from_radix, to_radix

pytestmark = pytest.mark.gpu

N32 = (1 << 22) + 4099          # reaches the HOT passes; 16,384-key (8,192-pair) tiles, the last one ragged
N64 = (1 << 20) + 77
EPOCH_MAX = (1 << 24) - 1
SIGN32 = -(1 << 31)
SIGN64 = -(1 << 63)


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


def load(t, a):
    """copies the numpy array `a` into the static tensor `t` (same width), on the current stream"""
    t.copy_(torch.from_numpy(a.view(np.int32 if a.dtype.itemsize == 4 else np.int64)))


def static(n, dtype=torch.int32):
    return torch.zeros(n, dtype=dtype, device="cuda")


def capture(fn):
    """one graph holding what fn() enqueues"""
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def radix_inputs(rng, n, utype, hot_keys=None):
    """(name, radix keys, skip mask, hot) in replay order; hot: whether the plan must run HOT passes (None: not asserted).
    hot_keys: the low-entropy input (default: 80 % of the keys share one value, which makes every place hot)"""
    nb = np.dtype(utype).itemsize * 8
    places = nb // 8
    every = (1 << places) - 1
    top, low = utype(0xFF << (nb - 8)), utype(0xFF)
    c = utype(0x5A5A5A5A5A5A5A5A if nb == 64 else 0x5A5A5A5A)

    def u():
        return rng.integers(0, np.iinfo(utype).max, n, dtype=utype, endpoint=True)

    if hot_keys is None:
        hot_keys = u()
        hot_keys[rng.random(n) < 0.8] = c
    return [
        ("uniform_a", u(), 0, False),
        ("top_byte_only", (u() & top) | (c & ~top), every & ~(1 << (places - 1)), None),
        ("hot", hot_keys, 0, n >= 1 << 22),
        ("low_byte_only", (u() & low) | (c & ~low), every & ~1, None),
        ("uniform_b", u(), 0, False),
        ("const_top_byte", (u() & ~top) | (c & top), 1 << (places - 1), None),
        ("all_equal", np.full(n, c, utype), every, None),
    ]


def u32_inputs(oracle, n, seed):
    rng = np.random.default_rng(seed)
    return radix_inputs(rng, n, np.uint32, hot_keys=oracle.init_random_u32(n, 3, seed))  # entropy preset 4


def check_plan(s, name, skip, hot):
    assert s.info("last_skip_mask") == skip, f"{name}: skip mask"
    if hot is not None:
        assert (s.info("last_hot_mask") != 0) == hot, f"{name}: hot mask"


def f32_specials():
    """+-0, +-inf, NaNs of both signs with several payloads, the smallest subnormals, +-max"""
    return np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFBFFFFF,
                     0x00000001, 0x80000001, 0x7F7FFFFF, 0xFF7FFFFF], dtype=np.uint32)


def with_specials_and_ties(rng, bits):
    """every special value 64 times, and 10 % of the keys drawn from 40 values (ties)"""
    b = bits.copy()
    sp = f32_specials()
    b[rng.choice(b.size, 64 * sp.size, replace=False)] = np.repeat(sp, 64)
    tie = rng.random(b.size) < 0.1
    b[tie] = rng.choice(b[:40], int(tie.sum()))
    return b


# ---- graph capture and replay, one entry point at a time ---------------------------------------------------------------

@pytest.mark.parametrize("pairs", [False, True], ids=["keys", "pairs"])
def test_graph_replays_u32(g, oracle, pairs):
    n = N32
    idx = np.arange(n, dtype=np.uint32)
    with g.OneSweepSorter(n, 4, 4 if pairs else 0) as s:
        tk = static(n)
        tv = static(n) if pairs else None

        def run():
            s.sort_pairs(tk, tv) if pairs else s.sort_keys(tk)

        def fill(k):
            load(tk, k)
            if pairs:
                load(tv, idx)

        def check(name, k):
            order = np.argsort(k, kind="stable")
            assert np.array_equal(host(tk), k[order]), name
            if pairs:
                assert np.array_equal(host(tv), order.astype(np.uint32)), f"{name}: payloads"

        warm = oracle.init_random_u32(n, 0, 99)
        fill(warm)
        run()  # eager, before the capture
        check("eager", warm)
        graph = capture(run)
        for name, k, skip, hot in u32_inputs(oracle, n, 1):
            fill(k)
            graph.replay()
            check(name, k)
            check_plan(s, name, skip, hot)


def test_graph_replays_u64(g):
    n = N64
    rng = np.random.default_rng(2)
    with g.OneSweepSorter(n, 8, 0) as s:
        t = static(n, torch.int64)
        warm = rng.integers(0, 1 << 63, n, dtype=np.uint64)
        load(t, warm)
        s.sort_keys(t)
        assert np.array_equal(host(t, np.uint64), np.sort(warm))
        graph = capture(lambda: s.sort_keys(t))
        for name, k, skip, hot in radix_inputs(rng, n, np.uint64):
            load(t, k)
            graph.replay()
            assert np.array_equal(host(t, np.uint64), np.sort(k)), name
            check_plan(s, name, skip, hot)


def test_graph_replays_f32_descending(g):
    """float keys in descending order: NaNs of both signs, +-0.0, infinities, subnormals and ties"""
    n = N32
    rng = np.random.default_rng(3)
    with g.OneSweepSorter(n, 4, 0) as s:
        t = static(n)
        run = lambda: s.sort_keys_typed(t, "f32", descending=True)  # noqa: E731
        warm = (rng.standard_normal(n) * 100).astype(np.float32).view(np.uint32)
        load(t, warm)
        run()
        assert np.array_equal(host(t), warm[np.argsort(to_radix(warm, "f", True), kind="stable")])
        graph = capture(run)
        for name, enc, skip, hot in radix_inputs(rng, n, np.uint32):
            bits = from_radix(enc, "f", descending=True)
            if name.startswith("uniform"):
                bits = with_specials_and_ties(rng, bits)
            load(t, bits)
            graph.replay()
            want = bits[np.argsort(to_radix(bits, "f", descending=True), kind="stable")]
            assert np.array_equal(host(t), want), name
            check_plan(s, name, skip, hot)


def test_graph_replays_i32_pairs(g):
    n = (1 << 21) + 555
    rng = np.random.default_rng(4)
    idx = np.arange(n, dtype=np.uint32)
    with g.OneSweepSorter(n, 4, 4) as s:
        tk, tv = static(n), static(n)
        run = lambda: s.sort_pairs_typed(tk, tv, "i32")  # noqa: E731
        warm = rng.integers(-300, 300, n).astype(np.int32).view(np.uint32)
        load(tk, warm)
        load(tv, idx)
        run()
        assert np.array_equal(host(tv), np.argsort(warm.view(np.int32), kind="stable").astype(np.uint32))
        graph = capture(run)
        for name, enc, skip, hot in radix_inputs(rng, n, np.uint32):
            bits = from_radix(enc, "i")
            load(tk, bits)
            load(tv, idx)
            graph.replay()
            order = np.argsort(to_radix(bits, "i"), kind="stable")
            assert np.array_equal(host(tk), bits[order]), name
            assert np.array_equal(host(tv), order.astype(np.uint32)), f"{name}: payloads"
            check_plan(s, name, skip, hot)


def test_graph_replays_sort_bits_with_values(g, oracle):
    """bits [3, 22): three places (bits 3-10, 11-18, 19-21), so the copy-back runs whenever no place is skipped"""
    n = (1 << 20) + 123
    rng = np.random.default_rng(5)
    idx = np.arange(n, dtype=np.uint32)

    def u():
        return rng.integers(0, 1 << 32, n, dtype=np.uint32)

    def only(lo, hi):  # bits [lo, hi) of [3, 22) vary, the rest of the range is constant
        m = np.uint32(((1 << hi) - 1) ^ ((1 << lo) - 1))
        rest = np.uint32(((1 << 22) - 1) ^ ((1 << 3) - 1)) & ~m
        return (u() & ~rest) | (np.uint32(0x2AAAA8) & rest)

    inputs = [
        ("uniform_a", u(), 0),
        ("place2_only", only(19, 22), 0b011),  # its one executed pass is uniform_a's last
        ("preset4", oracle.init_random_u32(n, 3, 5), 0),
        ("place0_only", only(3, 11), 0b110),
        ("uniform_b", u(), 0),  # its first executed pass is place0_only's only one
        ("all_equal", np.full(n, 0xDEADBEEF, np.uint32), 0b111),
    ]
    with g.OneSweepSorter(n, 4, 4) as s:
        tk, tv = static(n), static(n)
        run = lambda: s.sort_bits(tk, 3, 22, values=tv)  # noqa: E731
        load(tk, oracle.init_random_u32(n, 0, 55))
        load(tv, idx)
        run()
        graph = capture(run)
        for name, k, skip in inputs:
            load(tk, k)
            load(tv, idx)
            graph.replay()
            order = np.argsort((k >> np.uint32(3)) & np.uint32((1 << 19) - 1), kind="stable")
            assert np.array_equal(host(tk), k[order]), name
            assert np.array_equal(host(tv), order.astype(np.uint32)), f"{name}: payloads"
            assert s.info("last_skip_mask") == skip, name


def test_graph_replays_small_path(g, oracle):
    n = 10_000
    with g.OneSweepSorter(n, 4, 0) as s:
        assert n <= s.info("small_path_max_n")
        t = static(n)
        warm = oracle.init_random_u32(n, 0, 66)
        load(t, warm)
        s.sort_keys(t)
        assert np.array_equal(host(t), np.sort(warm))
        graph = capture(lambda: s.sort_keys(t))
        for name, k, _, _ in u32_inputs(oracle, n, 6):
            load(t, k)
            graph.replay()
            assert np.array_equal(host(t), np.sort(k)), name


def test_graph_replays_segmented_sort(g):
    """The offsets change between replays too (their count stays): empty segments, one of 16,384 keys, and keys past the
    last offset, which must stay where they are."""
    n, segs = 600_000, 64
    rng = np.random.default_rng(7)
    idx = np.arange(n, dtype=np.uint32)

    def offsets(longest):
        lengths = rng.integers(0, 9000, segs)
        lengths[rng.choice(segs, 5, replace=False)] = 0
        if longest:
            lengths[rng.integers(segs)] = 16384
        return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)

    inputs = [(rng.integers(0, 1 << 32, n, dtype=np.uint32), offsets(i % 2 == 0)) for i in range(5)]
    inputs.append((rng.integers(0, 4, n, dtype=np.uint32), offsets(True)))  # ties: stability shows in the payloads
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        tk, tv, to = static(n), static(n), torch.zeros(segs + 1, dtype=torch.int64, device="cuda")
        run = lambda: s.segmented_sort(tk, to, values=tv, max_segment_len=16384)  # noqa: E731
        for i, (k, off) in enumerate(inputs):
            load(tk, k)
            load(tv, idx)
            to.copy_(torch.from_numpy(off))
            if i == 0:
                run()  # eager, before the capture
                graph = capture(run)
            else:
                graph.replay()
            end = int(off[-1])
            seg = np.repeat(np.arange(segs), np.diff(off))
            order = np.concatenate([np.lexsort((k[:end], seg)), np.arange(end, n)])
            assert np.array_equal(host(tk), k[order]), f"input {i}"
            assert np.array_equal(host(tv), order.astype(np.uint32)), f"input {i}: payloads"


@pytest.mark.parametrize("pairs", [False, True], ids=["keys", "pairs"])
def test_graph_replays_digit_binning_pass(g, oracle, pairs):
    """one pass, one captured epoch: every replay meets the previous replay's descriptors under it"""
    n, shift = N32, 8
    idx = np.arange(n, dtype=np.uint32)
    with g.OneSweepSorter(n, 4, 4 if pairs else 0) as s:
        src, dst = static(n), static(n)
        sv, dv = (static(n), static(n)) if pairs else (None, None)
        run = lambda: s.digit_binning_pass(src, dst, shift, src_values=sv, dst_values=dv)  # noqa: E731
        load(src, oracle.init_random_u32(n, 0, 88))
        if pairs:
            load(sv, idx)
        run()
        graph = capture(run)
        for name, k, _, _ in u32_inputs(oracle, n, 8):
            load(src, k)
            if pairs:
                load(sv, idx)
            graph.replay()
            order = np.argsort((k >> np.uint32(shift)) & np.uint32(0xFF), kind="stable")
            assert np.array_equal(host(dst), k[order]), name
            if pairs:
                assert np.array_equal(host(dv), order.astype(np.uint32)), f"{name}: payloads"


# ---- graphs and eager sorts on one handle --------------------------------------------------------------------------------

def test_one_graph_two_sorts_on_one_handle(g, oracle):
    """A pairs sort and a keys sort of another size (other tiles) in one graph, on one pairs-capable handle"""
    n1, n2 = N32, (1 << 20) + 4321
    idx = np.arange(n1, dtype=np.uint32)
    with g.OneSweepSorter(n1, 4, 4) as s:
        k1, v1, k2 = static(n1), static(n1), static(n2)

        def run():
            s.sort_pairs(k1, v1)
            s.sort_keys(k2)

        load(k1, oracle.init_random_u32(n1, 0, 90))
        load(v1, idx)
        load(k2, oracle.init_random_u32(n2, 0, 91))
        run()
        graph = capture(run)
        a, b = u32_inputs(oracle, n1, 9), u32_inputs(oracle, n2, 10)
        for i in range(len(a)):
            (na, ka, _, _), (nb, kb, _, _) = a[i], b[(i + 3) % len(b)]
            load(k1, ka)
            load(v1, idx)
            load(k2, kb)
            graph.replay()
            order = np.argsort(ka, kind="stable")
            assert np.array_equal(host(k1), ka[order]), f"pairs {na}"
            assert np.array_equal(host(v1), order.astype(np.uint32)), f"pairs {na}: payloads"
            assert np.array_equal(host(k2), np.sort(kb)), f"keys {nb}"


def test_two_graphs_on_one_handle_replayed_alternately(g, oracle):
    na, nb = N32, (1 << 20) + 5
    with g.OneSweepSorter(na, 4, 0) as s:
        ta, tb = static(na), static(nb)
        load(ta, oracle.init_random_u32(na, 0, 92))
        s.sort_keys(ta)
        ga = capture(lambda: s.sort_keys(ta))
        gb = capture(lambda: s.sort_keys(tb))
        ins_a, ins_b = u32_inputs(oracle, na, 11), u32_inputs(oracle, nb, 12)
        for i in range(len(ins_a)):
            for graph, t, (name, k, _, _) in ((ga, ta, ins_a[i]), (gb, tb, ins_b[(i + 2) % len(ins_b)])):
                load(t, k)
                graph.replay()
                assert np.array_equal(host(t), np.sort(k)), f"round {i}, n = {t.numel()}: {name}"


def test_eager_sorts_between_replays(g, oracle):
    """The eager sorts are smaller: the graph's tiles past them keep what the previous replay wrote"""
    n, ne = N32, N32 // 4
    with g.OneSweepSorter(n, 4, 0) as s:
        t, e = static(n), static(ne)
        load(t, oracle.init_random_u32(n, 0, 93))
        s.sort_keys(t)
        graph = capture(lambda: s.sort_keys(t))
        ins, eag = u32_inputs(oracle, n, 13), u32_inputs(oracle, ne, 14)
        for i, (name, k, _, _) in enumerate(ins):
            load(t, k)
            graph.replay()
            assert np.array_equal(host(t), np.sort(k)), f"replay {name}"
            ename, ek, _, _ = eag[(i + 2) % len(eag)]
            load(e, ek)
            s.sort_keys(e)
            assert np.array_equal(host(e), np.sort(ek)), f"eager {ename} after replay {name}"


def test_module_sort_inside_a_capture(g, oracle):
    """Sort() keeps one cached handle per stream: a warm-up call on the capture stream creates it outside the capture"""
    n = N32
    cs = torch.cuda.Stream()
    t = static(n)
    warm = oracle.init_random_u32(n, 0, 94)
    load(t, warm)
    torch.cuda.synchronize()
    with torch.cuda.stream(cs):
        g.Sort(t)
    cs.synchronize()
    assert np.array_equal(host(t), np.sort(warm))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=cs):
        g.Sort(t)
    for name, k, _, _ in u32_inputs(oracle, n, 15):
        load(t, k)
        graph.replay()
        assert np.array_equal(host(t), np.sort(k)), name


# ---- epochs ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["u32", "pairs", "u64"])
def test_epoch_wrap_around(g, kind):
    """A one-pass sort at epoch 1 leaves its words in every tile.  The sort that crosses the wrap-around skips its first
    two places (constant low 16 bits), so its third place runs at epoch 1 on those words: only the clear at the
    wrap-around hides them.  Then a sort of uniform keys crosses the wrap-around with every pass executed."""
    kb, n, places = (8, N64, 8) if kind == "u64" else (4, N32, 4)
    utype = np.uint64 if kb == 8 else np.uint32
    pairs = kind == "pairs"
    rng = np.random.default_rng(16)
    idx = np.arange(n, dtype=np.uint32)
    with g.OneSweepSorter(n, kb, 4 if pairs else 0) as s:
        tk = static(n, torch.int64 if kb == 8 else torch.int32)
        tv = static(n) if pairs else None

        def sort_and_check(what, k, end_bit=None):
            load(tk, k)
            if pairs:
                load(tv, idx)
            if end_bit is not None:
                s.sort_bits(tk, 0, end_bit, values=tv)
                order = np.argsort(k & utype((1 << end_bit) - 1), kind="stable")
            else:
                s.sort_pairs(tk, tv) if pairs else s.sort_keys(tk)
                order = np.argsort(k, kind="stable")
            assert np.array_equal(host(tk, utype), k[order]), what
            if pairs:
                assert np.array_equal(host(tv), order.astype(np.uint32)), f"{what}: payloads"

        def u():
            return rng.integers(0, np.iinfo(utype).max, n, dtype=utype, endpoint=True)

        sort_and_check("one place at epoch 1", u(), end_bit=8)
        assert s.info("epoch") == 1
        s.set_option("debug_epoch", EPOCH_MAX - 2)
        assert s.info("epoch") == EPOCH_MAX - 2
        sort_and_check("low 16 bits constant, across the wrap-around", (u() & ~utype(0xFFFF)) | utype(0x1234))
        assert s.info("last_skip_mask") == 0b11
        assert s.info("epoch") == places - 2  # passes at 2^24 - 2, 2^24 - 1, then 1, 2, ...
        s.set_option("debug_epoch", EPOCH_MAX - 2)
        sort_and_check("uniform, across the wrap-around", u())
        assert s.info("epoch") == places - 2
        sort_and_check("uniform, after the wrap-around", u())


@pytest.mark.parametrize("pairs", [False, True], ids=["keys", "pairs"])
def test_captured_epochs_reused_by_an_eager_sort(g, oracle, pairs):
    """An eager sort on the epochs of a captured one, between two replays.  The replay before it runs only its first pass,
    the eager sort starts with that pass: the capture's clear after its passes hides the replay's words.  The eager sort
    ends with its last pass, the replay after it runs only that one: the capture's clear before its passes hides the
    eager sort's words."""
    n = N32
    rng = np.random.default_rng(17)
    idx = np.arange(n, dtype=np.uint32)
    with g.OneSweepSorter(n, 4, 4 if pairs else 0) as s:
        tk, ek = static(n), static(n)
        tv, ev = (static(n), static(n)) if pairs else (None, None)

        def sort(k, v):
            s.sort_pairs(k, v) if pairs else s.sort_keys(k)

        def fill_and_check(what, k, v, keys, run, skip):
            load(k, keys)
            if pairs:
                load(v, idx)
            run()
            order = np.argsort(keys, kind="stable")
            assert np.array_equal(host(k), keys[order]), what
            if pairs:
                assert np.array_equal(host(v), order.astype(np.uint32)), f"{what}: payloads"
            assert s.info("last_skip_mask") == skip, what

        def u():
            return rng.integers(0, 1 << 32, n, dtype=np.uint32)

        fill_and_check("eager, before the capture", tk, tv, oracle.init_random_u32(n, 0, 95), lambda: sort(tk, tv), 0)
        e0 = s.info("epoch")
        graph = capture(lambda: sort(tk, tv))
        assert s.info("epoch") == e0 + 4
        fill_and_check("replay, low byte only", tk, tv, (u() & np.uint32(0xFF)) | np.uint32(0x5A5A5A00), graph.replay,
                       0b1110)
        s.set_option("debug_epoch", e0)  # the eager sort runs its passes at the captured epochs
        fill_and_check("eager, captured epochs", ek, ev, u(), lambda: sort(ek, ev), 0)
        assert s.info("epoch") == e0 + 4
        fill_and_check("replay, top byte only", tk, tv, (u() & np.uint32(0xFF000000)) | np.uint32(0x5A5A5A), graph.replay,
                       0b0111)
        fill_and_check("replay, uniform", tk, tv, u(), graph.replay, 0)


def test_debug_epoch_range(g):
    with g.OneSweepSorter(1 << 16, 4, 0) as s:
        s.set_option("debug_epoch", 0)
        s.set_option("debug_epoch", EPOCH_MAX)
        assert s.info("epoch") == EPOCH_MAX
        for bad in (-1, EPOCH_MAX + 1):
            with pytest.raises(g.OneSweepError):
                s.set_option("debug_epoch", bad)


# ---- concurrency -----------------------------------------------------------------------------------------------------

def device_case(g, kind, n, seed):
    """(keys, payloads or None, expected keys, expected payloads or None) on the device; keys are ordered as unsigned"""
    if kind == "u64":
        gen = torch.Generator(device="cuda").manual_seed(seed)
        k = torch.randint(-(1 << 63), (1 << 63) - 1, (n,), dtype=torch.int64, device="cuda", generator=gen)
        want, _ = torch.sort(k ^ SIGN64, stable=True)
        return k, None, want ^ SIGN64, None
    k = torch.empty(n, dtype=torch.int32, device="cuda")
    v = torch.empty(n, dtype=torch.int32, device="cuda") if kind == "pairs" else None
    g.init_random(k, 3 if kind == "u32_preset4" else 0, seed, payload=v, payload_is_index=v is not None)
    want, order = torch.sort(k ^ SIGN32, stable=True)
    return k, v, want ^ SIGN32, (order.to(torch.int32) if v is not None else None)


def concurrent_rounds(g, kinds, n, rounds, seed, before=None):
    """One handle and one stream per kind, `rounds` sorts on each, all enqueued before any is checked"""
    sorters = [g.OneSweepSorter(n, 8 if kind == "u64" else 4, 4 if kind == "pairs" else 0) for kind in kinds]
    streams = [torch.cuda.Stream() for _ in kinds]
    cases = [[device_case(g, kind, n, seed + 10 * r + i) for i, kind in enumerate(kinds)] for r in range(rounds)]
    torch.cuda.synchronize()
    if before is not None:
        before()
    for r in range(rounds):
        for s, st, (k, v, _, _) in zip(sorters, streams, cases[r]):
            s.sort_keys(k, stream=st) if v is None else s.sort_pairs(k, v, stream=st)
    torch.cuda.synchronize()
    try:
        for r in range(rounds):
            for kind, (k, v, want, order) in zip(kinds, cases[r]):
                assert torch.equal(k, want), f"{kind}, round {r}"
                if v is not None:
                    assert torch.equal(v, order), f"{kind}, round {r}: payloads"
    finally:
        for s in sorters:
            s.close()


def test_four_handles_on_four_streams(g):
    """Concurrent passes cannot all be resident (a plain u32 pass wants 264 CTAs, a HOT pass 132), so a tile can wait on a
    predecessor whose CTA has not started yet, until the spin cap's fallback re-reduces that tile"""
    concurrent_rounds(g, ["u32", "u32_preset4", "pairs", "u64"], 1 << 24, 3, 100)


def test_sorts_beside_matmuls_on_another_stream(g):
    """The u32 sorts while a bounded loop of bf16 matmuls holds SMs from another stream, as other work on a shared GPU"""
    a = torch.randn(4096, 4096, dtype=torch.bfloat16, device="cuda")
    b = torch.randn(4096, 4096, dtype=torch.bfloat16, device="cuda")
    ms = torch.cuda.Stream()

    def matmuls():
        with torch.cuda.stream(ms):
            for _ in range(100):
                torch.mm(a, b)

    concurrent_rounds(g, ["u32", "u32_preset4"], 1 << 24, 3, 200, before=matmuls)


def test_back_to_back_sorts_on_one_stream(g, oracle):
    n = N32
    st = torch.cuda.Stream()
    ins = u32_inputs(oracle, n, 30)[:6] + [("uniform_c", oracle.init_random_u32(n, 0, 31), 0, False),
                                           ("preset3", oracle.init_random_u32(n, 2, 32), 0, None)]
    tensors = [torch.from_numpy(k.view(np.int32)).cuda() for _, k, _, _ in ins]
    torch.cuda.synchronize()
    with g.OneSweepSorter(n, 4, 0) as s:
        for t in tensors:
            s.sort_keys(t, stream=st)
        st.synchronize()
    for (name, k, _, _), t in zip(ins, tensors):
        assert np.array_equal(host(t), np.sort(k)), name


def test_keys_written_on_a_side_stream_then_sorted_there(g, oracle):
    """torch ops on a side stream produce the keys and the sort follows on that stream with no synchronisation; the sleep
    keeps the producer busy long after the sort has been enqueued"""
    n = N32
    k = oracle.init_random_u32(n, 0, 40)
    mask = np.uint32(0x9E3779B9)
    src = torch.from_numpy(k.view(np.int32)).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with g.OneSweepSorter(n, 4, 0) as s:
        with torch.cuda.stream(side):
            t = src.clone()
            torch.cuda._sleep(20_000_000)
            t ^= int(mask.view(np.int32))
            s.sort_keys(t)
        torch.cuda.synchronize()
    assert np.array_equal(host(t), np.sort(k ^ mask))


def test_module_sort_from_two_streams(g, oracle):
    from gpusorting_b200 import onesweep

    n = N32
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    assert s1.cuda_stream != s2.cuda_stream
    k1, k2 = oracle.init_random_u32(n, 0, 50), oracle.init_random_u32(n, 3, 51)
    t1, t2 = (torch.from_numpy(k.view(np.int32)).cuda() for k in (k1, k2))
    torch.cuda.synchronize()
    g.Sort(t1, stream=s1)
    g.Sort(t2, stream=s2)
    d = t1.device.index
    h1, h2 = onesweep._CACHE[(d, 4, 0, s1.cuda_stream)], onesweep._CACHE[(d, 4, 0, s2.cuda_stream)]
    assert h1 is not h2 and h1._h.value != h2._h.value
    torch.cuda.synchronize()
    assert np.array_equal(host(t1), np.sort(k1))
    assert np.array_equal(host(t2), np.sort(k2))
