"""osb200_topk_long_rows, OneSweepSorter.topk_long_rows and gpusorting_b200.topk_long_rows: the row top-k for any k up to the
row length, with long rows split across thread blocks.

The oracle is test_gpu_topk's: numpy's stable argsort of each row's radix image, cut to k.  sorted=True must equal it bit for
bit, keys and indices, and equal topk_rows wherever that call takes the arguments; sorted=False must hold the same (key,
position) pairs.  The split path is reached by few long rows, by k above topk_rows' capacity C (16,384 keys, 8,192 for 64-bit
keys) and by the "debug_long_rows" hook, which sends every row of 2 or more keys to it (most tests set it, so that rows of
any length and k <= C take the split path); "debug_topk_capacity" moves the
candidate count at which a row stops and is finished in shared memory.
The test whose name contains "past_2pow" needs about 30 GB: -k "not past_2pow" leaves it out of a quick run.  -m gpu"""
import numpy as np
import pytest
import torch

from tests.test_gpu_topk import TYPES, dev, host, order_of, same, width

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
SM_COUNT = None


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    global SM_COUNT
    SM_COUNT = torch.cuda.get_device_properties(0).multi_processor_count
    return g


def cap(t):
    return 8192 if width(t) == 64 else 16384


def random_bits(rng, n, t):
    c = TYPES[t][1]
    return rng.integers(0, np.iinfo(c).max, n, dtype=c, endpoint=True)


def sorter(g, n, t):
    return g.OneSweepSorter(max(n, 1), 8 if width(t) == 64 else 4, 4)


def check(s, x, bits2d, t, largest, k, what, against_rows=True):
    """topk_long_rows sorted and unsorted against the stable-sort oracle, and against topk_rows where it takes the call"""
    order = order_of(bits2d, t, largest)
    want_i = order[:, :k]
    want_k = np.take_along_axis(bits2d, want_i, axis=-1)
    vals, idx = s.topk_long_rows(x, k, t, largest, True)
    assert vals.shape == idx.shape == (bits2d.shape[0], k) and vals.dtype == x.dtype and idx.dtype == torch.int32
    gk, gi = host(vals, t), idx.cpu().numpy().view(np.uint32).astype(np.int64)
    same(gk, want_k, f"{what}, k={k}: keys")
    same(gi, want_i, f"{what}, k={k}: indices")
    if against_rows and k <= cap(t):
        rk, ri = s.topk_rows(x, k, t, largest, True)
        same(gk, host(rk, t), f"{what}, k={k}: keys against topk_rows")
        same(gi, ri.cpu().numpy().view(np.uint32), f"{what}, k={k}: indices against topk_rows")
    uk, ui = s.topk_long_rows(x, k, t, largest, False)
    uk, ui = host(uk, t), ui.cpu().numpy().view(np.uint32).astype(np.int64)
    o = np.argsort(ui, axis=-1, kind="stable")
    same(np.take_along_axis(ui, o, axis=-1), np.sort(want_i, axis=-1), f"{what}, k={k}, unsorted: positions")
    same(np.take_along_axis(uk, o, axis=-1), np.take_along_axis(bits2d, np.sort(want_i, axis=-1), axis=-1),
         f"{what}, k={k}, unsorted: keys with their positions")


# ---- 1. every dtype, both orders, the k of the issue ------------------------------------------------------------------------
@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("largest", [False, True])
def test_dtypes_and_k(g, t, largest):
    rng = np.random.default_rng(11 + width(t))
    rows, row_len = 3, 40_000
    bits = random_bits(rng, rows * row_len, t).reshape(rows, row_len)
    if TYPES[t][3] != "u":  # some ties
        bits[:, ::7] = bits[0, 5]
    x = dev(bits.reshape(-1), t).reshape(rows, row_len)
    c = cap(t)
    ks = {1, 50, 16_384, 16_385, row_len - 1, row_len} | ({8192, 8193} if width(t) == 64 else set())
    with sorter(g, rows * row_len, t) as s:
        s.set_option("debug_long_rows", 1)  # k <= C too on the split path
        for k in sorted(ks):
            check(s, x, bits, t, largest, k, f"{t} largest={largest}", against_rows=k <= c)


# ---- 2. row lengths and batches ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hook", [0, 1])
@pytest.mark.parametrize("rows", [1, 8, 64])
def test_lengths_and_batches(g, rows, hook):
    """hook = 1 (debug_long_rows) sends the rows of at most 65,536 keys to the split path too"""
    rng = np.random.default_rng(rows)
    with sorter(g, rows * 151_936, "f32") as s:
        s.set_option("debug_long_rows", hook)
        for row_len in (8193, 2 * 8192 - 1, 2 * 8192 + 1, 3 * 8192 - 1, 3 * 8192 + 1, 32_000, 128_256, 151_936):
            vals = (rng.standard_normal(rows * row_len) * 3).astype(np.float32)
            bits = vals.view(np.uint32).reshape(rows, row_len)
            x = dev(bits.reshape(-1), "f32").reshape(rows, row_len)
            for k in (50, 1024):
                check(s, x, bits, "f32", True, k, f"[{rows}, {row_len}] f32")
            bf = torch.from_numpy(vals).cuda().to(torch.bfloat16).reshape(rows, row_len)
            want = torch.sort(bf.float(), dim=-1, descending=True, stable=True)
            got_v, got_i = s.topk_long_rows(bf, 50, "bf16", True, True)
            assert torch.equal(got_v.float(), want.values[:, :50]) and torch.equal(got_i.long(), want.indices[:, :50])


def test_one_row_of_2pow26_keys_k_2pow20(g):
    n, k = 1 << 26, 1 << 20
    torch.manual_seed(5)
    x = torch.randn(1, n, device="cuda")
    with sorter(g, n, "f32") as s:
        for largest in (True, False):
            want = torch.sort(x, dim=-1, descending=largest, stable=True)
            v, i = s.topk_long_rows(x, k, "f32", largest, True)
            assert torch.equal(v, want.values[:, :k]) and torch.equal(i.long(), want.indices[:, :k])
            v, i = s.topk_long_rows(x, k, "f32", largest, False)
            i, o = torch.sort(i.long(), dim=-1)
            assert torch.equal(i, torch.sort(want.indices[:, :k], dim=-1).values)
            assert torch.equal(torch.gather(v, 1, o), torch.gather(x, 1, i))


# ---- 3. the test hooks ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", ["u16", "f32", "i64"])
def test_debug_long_rows_down_to_two_keys(g, t):
    rng = np.random.default_rng(23)
    with sorter(g, 1 << 24, t) as s:
        s.set_option("debug_long_rows", 1)
        try:
            for rows, row_len in ((40, 2), (33, 3), (20, 31), (9, 300), (5, 5000), (3, 8192), (2, 8193), (2, 20_000)):
                bits = random_bits(rng, rows * row_len, t).reshape(rows, row_len)
                bits[:, 1::3] = bits[:, :1]  # ties
                x = dev(bits.reshape(-1), t).reshape(rows, row_len)
                for k in sorted({1, 2, row_len // 2 or 1, row_len - 1 or 1, row_len}):
                    for largest in (False, True):
                        check(s, x, bits, t, largest, k, f"hook {t} [{rows}, {row_len}]", against_rows=False)
        finally:
            s.set_option("debug_long_rows", 0)
        # the same calls on topk_rows' own launch give the same answers
        bits = random_bits(rng, 7 * 3000, t).reshape(7, 3000)
        x = dev(bits.reshape(-1), t).reshape(7, 3000)
        s.set_option("debug_long_rows", 1)
        a = s.topk_long_rows(x, 100, t, True, True)
        s.set_option("debug_long_rows", 0)
        b = s.topk_rows(x, 100, t, True, True)
        same(host(a[0], t), host(b[0], t), "hook against topk_rows: keys")
        same(a[1].cpu().numpy(), b[1].cpu().numpy(), "hook against topk_rows: indices")


@pytest.mark.parametrize("extra", [0, 1])
def test_capacity_hook_at_n_and_n_plus_1_candidates(g, extra):
    """a row whose smallest top byte holds N (+ extra) keys: with debug_topk_capacity N it stops after level 0, or one level
    later; k lies inside that bucket, so the finisher takes the rest"""
    rng = np.random.default_rng(41 + extra)
    n_cap, rows, row_len = 3000, 4, 50_000
    bits = (rng.integers(1 << 24, 1 << 31, rows * row_len, dtype=np.uint32) | np.uint32(1 << 31)).reshape(rows, row_len)
    for r in range(rows):
        pos = rng.choice(row_len, n_cap + extra, replace=False)
        bits[r, pos] = rng.integers(0, 1 << 24, n_cap + extra, dtype=np.uint32)
        bits[r, pos[:300]] = bits[r, pos[0]]  # ties inside the finisher's candidates
    x = dev(bits.reshape(-1), "u32").reshape(rows, row_len)
    with sorter(g, rows * row_len, "u32") as s:
        s.set_option("debug_topk_capacity", n_cap)
        s.set_option("debug_long_rows", 1)
        try:
            for k in (1, 299, 300, 301, 1500, n_cap, n_cap + extra):
                check(s, x, bits, "u32", False, k, f"capacity {n_cap} + {extra}")
        finally:
            s.set_option("debug_topk_capacity", 0)


# ---- 4. skewed keys, ties across tiles, rows resolved early ------------------------------------------------------------------
def test_skewed_keys_and_ties_across_tiles(g):
    rng = np.random.default_rng(59)
    rows, row_len = 6, 3 * 8192 + 5  # a ragged last tile of 5 keys
    few = rng.integers(0, 3, rows * row_len).astype(np.float32).reshape(rows, row_len)  # three values
    few[1] = 1.0  # all equal
    few[2, -5:] = 7.0  # the largest keys in the ragged last tile
    logits = (rng.standard_normal(rows * row_len) * 3).astype(np.float32).reshape(rows, row_len)
    top = np.float32(np.array([0x40000000, 0x40800000, 0xC0000000], dtype=np.uint32).view(np.float32))
    logits[3] = top[rng.integers(0, 3, row_len)]  # the top byte takes a few values, and so do the others
    with sorter(g, rows * row_len, "f32") as s:
        s.set_option("debug_long_rows", 1)
        for arr in (few, logits):
            bits = arr.view(np.uint32)
            x = dev(bits.reshape(-1), "f32").reshape(rows, row_len)
            for k in (1, 5, 6, 8191, 8192, 8193, 12_000, 16_384, 16_385, 20_000, row_len - 1, row_len):
                for largest in (True, False):
                    check(s, x, bits, "f32", largest, k, "skewed f32")


def test_rows_resolved_at_level_0(g):
    """exactly k keys share the smallest top byte: the row is resolved by the first pick"""
    rng = np.random.default_rng(61)
    rows, row_len, k = 5, 30_000, 777
    bits = rng.integers(1 << 30, 1 << 32, rows * row_len, dtype=np.uint64).astype(np.uint32).reshape(rows, row_len)
    bits |= np.uint32(1 << 31)
    for r in range(rows):
        bits[r, rng.choice(row_len, k, replace=False)] = rng.integers(0, 4, k, dtype=np.uint32)  # ties among them too
    x = dev(bits.reshape(-1), "u32").reshape(rows, row_len)
    with sorter(g, rows * row_len, "u32") as s:
        s.set_option("debug_long_rows", 1)
        for kk in (k - 1, k, k + 1):
            check(s, x, bits, "u32", False, kk, "resolved at level 0")


def test_batch_at_the_path_threshold_is_topk_rows(g):
    """at least as many rows as SMs, or rows of at most 65,536 keys, with k <= C: topk_rows' launch, which needs no workspace"""
    rng = np.random.default_rng(67)
    for rows, row_len in ((SM_COUNT, 70_000), (2 * SM_COUNT, 70_000), (1, 65_536), (8, 32_000)):
        bits = random_bits(rng, rows * row_len, "f32").reshape(rows, row_len)
        x = dev(bits.reshape(-1), "f32").reshape(rows, row_len)
        with g.OneSweepSorter(1, 4, 0) as s:  # no workspace: the split path would refuse the call
            a = s.topk_long_rows(x, 64, "f32", True, True)
            b = s.topk_rows(x, 64, "f32", True, True)
            same(host(a[0], "f32"), host(b[0], "f32"), f"[{rows}, {row_len}]: keys")
            same(a[1].cpu().numpy(), b[1].cpu().numpy(), f"[{rows}, {row_len}]: indices")
            if rows == SM_COUNT:
                with pytest.raises(g.OneSweepError):  # one row fewer takes the split path
                    s.topk_long_rows(x[1:], 64, "f32", True, True)


# ---- 5. errors ------------------------------------------------------------------------------------------------------------
def test_argument_and_workspace_errors(g):
    lib = g.lib
    n = 40_000
    a = torch.zeros(n, dtype=torch.int64, device="cuda")
    b = torch.zeros(n, dtype=torch.int64, device="cuda")
    c = torch.zeros(n, dtype=torch.int32, device="cuda")
    pa, pb, pc = a.data_ptr(), b.data_ptr(), c.data_ptr()

    def call(h, i=pa, o=pb, x=pc, rows=1, row_len=20_000, k=16_385, kb=4, kt=2, largest=1, srt=1):
        return lib.osb200_topk_long_rows(h, i, o, x, rows, row_len, k, kb, kt, largest, srt, None)

    with g.OneSweepSorter(n, 4, 4) as s, g.OneSweepSorter(n, 4, 0) as nov, g.OneSweepSorter(1000, 4, 4) as small, \
            g.OneSweepSorter(n, 8, 4) as wide:
        h = s._h
        assert call(h) == OK
        assert call(h, k=20_000) == OK
        assert call(h, k=20_001) == INVALID_ARG
        assert call(None) == INVALID_ARG
        assert call(h, x=None) == INVALID_ARG
        assert call(h, i=pa + 2) == INVALID_ARG
        assert call(h, o=pa) == INVALID_ARG  # overlapping input and output
        assert call(h, x=pb + 16) == INVALID_ARG  # overlapping outputs
        assert call(nov._h) == INVALID_ARG  # a (4, 0) handle on the split path
        assert call(nov._h, k=64) == OK  # topk_rows' launch: any handle
        assert call(small._h) == SIZE  # n > max_n
        assert call(small._h, k=16_384) == OK
        assert call(h, kb=8, kt=3, k=9000) == INVALID_ARG  # 8-byte keys on a 4-byte handle
        assert call(wide._h, kb=8, kt=3, k=9000) == OK
        assert call(wide._h, kb=2, kt=0, k=20_000) == OK
        for kw in ({"rows": 0}, {"row_len": 0}, {"k": 0}):
            assert call(h, i=None, o=None, x=None, **kw) == OK, kw
        torch.cuda.synchronize()
    with pytest.raises(g.OneSweepError):
        g.topk_long_rows(torch.zeros(2, 10, device="cuda"), 11)


# ---- 6. graphs, streams, the module function --------------------------------------------------------------------------------
def test_graph_capture_and_replay_on_new_data(g):
    rng = np.random.default_rng(71)
    shapes = {"f32": ((4, 60_000), 20_000), "bf16": ((2, 100_000), 50), "i64": ((3, 30_000), 9000)}
    with g.OneSweepSorter(1 << 20, 8, 4) as s:
        bufs = {t: torch.zeros(shape, dtype=TYPES[t][0], device="cuda") for t, (shape, _) in shapes.items()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for t, bb in bufs.items():
                s.topk_long_rows(bb, shapes[t][1], t, True, True)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        outs = {}
        with torch.cuda.graph(graph):
            for t, bb in bufs.items():
                outs[t] = s.topk_long_rows(bb, shapes[t][1], t, True, True)
        for replay in range(3):
            data = {t: random_bits(rng, shape[0] * shape[1], t).reshape(shape) for t, (shape, _) in shapes.items()}
            for t, bb in bufs.items():
                bb.copy_(dev(data[t].reshape(-1), t).reshape(shapes[t][0]))
            graph.replay()
            torch.cuda.synchronize()
            for t, (_, k) in shapes.items():
                want_i = order_of(data[t], t, True)[:, :k]
                same(host(outs[t][0], t), np.take_along_axis(data[t], want_i, axis=-1), f"replay {replay} {t}: keys")
                same(outs[t][1].cpu().numpy().view(np.uint32), want_i, f"replay {replay} {t}: indices")
        del graph


def test_two_streams_with_their_own_handles(g):
    torch.manual_seed(3)
    xs = [torch.randn(8, 128_256, device="cuda"), torch.randn(2, 500_000, device="cuda")]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    with g.OneSweepSorter(1 << 21, 4, 4) as s0, g.OneSweepSorter(1 << 21, 4, 4) as s1:
        torch.cuda.synchronize()
        res = []
        for s, x, st, k in ((s0, xs[0], streams[0], 1024), (s1, xs[1], streams[1], 20_000)):
            with torch.cuda.stream(st):
                for _ in range(3):
                    r = s.topk_long_rows(x, k, "f32", True, True, stream=st)
            res.append(r)
        torch.cuda.synchronize()
        for (v, i), x, k in zip(res, xs, (1024, 20_000)):
            want = torch.sort(x, dim=-1, descending=True, stable=True)
            assert torch.equal(v, want.values[:, :k]) and torch.equal(i.long(), want.indices[:, :k])


def test_module_function(g):
    torch.manual_seed(7)
    for dt in (torch.float32, torch.bfloat16, torch.int64, torch.float16):
        x = (torch.randn(3, 2, 70_000, device="cuda") * 100).to(dt)
        for k, largest in ((50, True), (17_000, False), (70_000, True)):
            if dt == torch.int64 and k == 17_000:
                k = 9000
            v, i = g.topk_long_rows(x, k, largest)
            want = torch.sort(x, dim=-1, descending=largest, stable=True)
            assert v.shape == i.shape == (3, 2, k) and i.dtype == torch.int32
            assert torch.equal(v, want.values[..., :k]) and torch.equal(i.long(), want.indices[..., :k])
    x = torch.randn(16, 300, device="cuda")
    v, i = g.topk_long_rows(x, 30)
    assert torch.equal(v, torch.topk(x, 30, dim=-1).values)


# ---- 7. one row past 2^31 keys -----------------------------------------------------------------------------------------------
def test_bf16_row_past_2pow31(g):
    """one bfloat16 row of 2^31 + 4,099 keys whose k largest lie past position 2^31 (negative int32 positions) and every other
    key is strictly smaller: the answer is known without a sort"""
    n, k = (1 << 31) + 4099, 64
    x = torch.rand(n, dtype=torch.bfloat16, device="cuda")
    planted = 2.0 + torch.arange(k, device="cuda", dtype=torch.float32) / 64
    pos = (1 << 31) + 17 + torch.randperm(4000, device="cuda")[:k].sort().values
    x[pos] = planted.to(torch.bfloat16)[torch.randperm(k, device="cuda")]
    with g.OneSweepSorter(n, 4, 4) as s:
        vals, idx = s.topk_long_rows(x.view(1, n), k, "bf16", True, True)
    want_v, order = torch.sort(x[pos].float(), descending=True, stable=True)
    assert torch.equal(vals[0].float(), want_v)
    assert torch.equal(idx[0].long() & 0xFFFFFFFF, pos[order])
    assert (idx[0] < 0).all()
    del x
    torch.cuda.empty_cache()
