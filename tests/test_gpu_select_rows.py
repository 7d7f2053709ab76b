"""osb200_select_rows, OneSweepSorter.select_rows and the module functions select_rows, kthvalue, median and quantile: the keys
at given ranks of every row's ascending stable sort, and their positions within the row.

The yardstick is the library's own stable row sort (sort_rows, sort_long_rows): the selected values and positions must be its
columns at the ranks, bit for bit, and numpy's stable argsort of the radix images where an input is built on the host.  The
split path (rows above C = 16,384 keys, 8,192 for 64-bit keys) is also reached through the "debug_long_rows" hook, which
sends every row of two or more keys to it, so it is compared with the short path on the same rows.
The test whose name contains "past_2pow" needs about 17 GB: -k "not past_2pow" leaves it out of a quick run.  -m gpu"""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_topk import TYPES, dev, host, order_of, width

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
KEY_TYPE = {"u16": 0, "i16": 1, "f16": 2, "bf16": 3, "u32": 0, "i32": 1, "f32": 2, "u64": 3, "i64": 4, "f64": 5}


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def cap(t):
    return 8192 if width(t) == 64 else 16384


def random_bits(rng, n, t):
    c = TYPES[t][1]
    return rng.integers(0, np.iinfo(c).max, n, dtype=c, endpoint=True)


def typed(rng, n, t):
    """randn * 3 for floats, uniform bits for integers, with some ties"""
    if TYPES[t][3] == "f":
        x = (torch.randn(n, generator=torch.Generator().manual_seed(int(rng.integers(1 << 30))), dtype=torch.float64) * 3)
        return x.to(TYPES[t][0]).view(getattr(torch, np.dtype(TYPES[t][2]).name)).numpy().view(TYPES[t][1])
    bits = random_bits(rng, n, t)
    bits[::5] = bits[0]
    return bits


def spread(row_len, count=16):
    """up to `count` distinct ranks spread over the row, with 0 and row_len - 1"""
    return sorted({round(i * (row_len - 1) / (count - 1)) for i in range(count)}) if row_len > 1 else [0]


def bits_of(x, t):
    return x.contiguous().view(getattr(torch, np.dtype(TYPES[t][2]).name))


def check_against_sort(g, s, x, t, ranks, what, indices=True):
    """select_rows on sorter s against the library's stable row sort of the same rows, bit for bit"""
    sv, si = g.sort_long_rows(x)
    r = torch.tensor(ranks, device=x.device, dtype=torch.int64).expand(*x.shape[:-1], len(ranks))
    want_v, want_i = torch.gather(bits_of(sv, t), -1, r), torch.gather(si, -1, r)
    if indices:
        v, i = s.select_rows(x, ranks, t)
        assert v.shape == i.shape == tuple(x.shape[:-1]) + (len(ranks),) and v.dtype == x.dtype and i.dtype == torch.int32
        assert torch.equal(i, want_i), f"{what}: positions"
    else:
        v = s.select_rows(x, ranks, t, return_indices=False)
    assert torch.equal(bits_of(v, t), want_v), f"{what}: values"


def batch_for(row_len, i):
    b = (1, 8, 64, 1000)[i % 4]
    while b > 1 and b * row_len > (1 << 24):
        b //= 8
    return b


LENGTHS = [1, 2, 31, 256, 257, 2048, 2049, 8192, 8193, 16384, 16385, 65536, 151936]


# ---- 1. every dtype, the lengths around each path's edges, batches ---------------------------------------------------------
@pytest.mark.parametrize("t", list(TYPES))
def test_dtypes_and_lengths(g, t):
    rng = np.random.default_rng(width(t) + KEY_TYPE[t])
    with g.OneSweepSorter(1 << 10, 4, 0) as s:  # far smaller than the inputs: the split path's bound is what counts
        for j, row_len in enumerate(LENGTHS):
            rows = batch_for(row_len, j)
            x = dev(typed(rng, rows * row_len, t), t).reshape(rows, row_len)
            ranks = sorted(set(spread(row_len, 14)) | {(row_len - 1) // 2})
            if row_len > cap(t) and g.select_workspace_words(rows, row_len, len(ranks)) > 1 << 10:
                with g.OneSweepSorter(g.select_workspace_words(rows, row_len, len(ranks)), 4, 0) as big:
                    check_against_sort(g, big, x, t, ranks, f"{t} [{rows}, {row_len}]")
                    check_against_sort(g, big, x, t, ranks, f"{t} [{rows}, {row_len}] values only", indices=False)
            else:
                check_against_sort(g, s, x, t, ranks, f"{t} [{rows}, {row_len}]")
                check_against_sort(g, s, x, t, ranks, f"{t} [{rows}, {row_len}] values only", indices=False)


@pytest.mark.parametrize("rows", [1, 8, 64])
def test_long_rows_in_batches(g, rows):
    torch.manual_seed(rows)
    x = torch.randn(rows, 151_936, device="cuda") * 3
    ranks = spread(151_936)
    with g.OneSweepSorter(g.select_workspace_words(rows, 151_936, 16), 4, 0) as s:
        check_against_sort(g, s, x, "f32", ranks, f"[{rows}, 151936]")


def test_one_row_of_2pow26_float32(g):
    torch.manual_seed(26)
    x = torch.randn(1, 1 << 26, device="cuda") * 3
    ranks = [0, 1, (1 << 25) - 1, 1 << 25, (1 << 26) - 2, (1 << 26) - 1]
    with g.OneSweepSorter(g.select_workspace_words(1, 1 << 26, len(ranks)), 4, 0) as s:
        check_against_sort(g, s, x, "f32", ranks, "one row of 2^26")
    del x
    torch.cuda.empty_cache()


# ---- 2. rank sets ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", ["u32", "f32", "bf16", "i64"])
@pytest.mark.parametrize("row_len", [3000, 40_000])
def test_rank_sets(g, t, row_len):
    rng = np.random.default_rng(row_len + width(t))
    rows = 4
    bits = typed(rng, rows * row_len, t).reshape(rows, row_len)
    bits[:, 100:400] = bits[0, 7]  # a run of equal keys: adjacent ranks fall on it
    x = dev(bits.reshape(-1), t).reshape(rows, row_len)
    order = order_of(bits, t, False)
    with g.OneSweepSorter(1 << 20, 4, 0) as s:
        hit = int(np.flatnonzero(np.take_along_axis(bits, order, -1)[0] == bits[0, 7])[0])
        for ranks in ([0], [row_len - 1], [(row_len - 1) // 2], spread(row_len), [hit, hit + 1, hit + 2, hit + 150]):
            for hook in (0, 1):
                s.set_option("debug_long_rows", hook)
                v, i = s.select_rows(x, ranks, t)
                want_i = order[:, ranks]
                assert np.array_equal(i.cpu().numpy().astype(np.int64), want_i), f"{t} {row_len} {ranks} hook={hook}: positions"
                assert np.array_equal(host(v, t), np.take_along_axis(bits, want_i, -1)), f"{t} {row_len} {ranks} hook={hook}: values"


@pytest.mark.parametrize("t", ["u16", "u32", "u64"])
def test_prefixes_that_part_at_the_last_level(g, t):
    """keys that share every digit but the last: 16 ranks stay in one group for D - 1 levels and part at the last one"""
    rng = np.random.default_rng(5)
    c = TYPES[t][1]
    row_len = 20_000
    high = c(0xA5) << c(8 * (width(t) // 8 - 1))
    bits = (high | rng.integers(0, 256, row_len).astype(c)).reshape(1, row_len)
    x = dev(bits.reshape(-1), t).reshape(1, row_len)
    order = order_of(bits, t, False)
    ranks = spread(row_len)
    with g.OneSweepSorter(1 << 16, 4, 0) as s:
        for hook in (0, 1):
            s.set_option("debug_long_rows", hook)
            v, i = s.select_rows(x, ranks, t)
            assert np.array_equal(i.cpu().numpy().astype(np.int64), order[:, ranks]), f"{t} hook={hook}"
            assert np.array_equal(host(v, t), np.take_along_axis(bits, order[:, ranks], -1))


# ---- 3. inputs ------------------------------------------------------------------------------------------------------------
def structured(rng, t, rows, row_len):
    c = TYPES[t][1]
    u = random_bits(rng, rows * row_len, t).reshape(rows, row_len)
    top = c(0x3C) << c(8 * (width(t) // 8 - 1))
    return {
        "uniform": u,
        "all_equal": np.full((rows, row_len), u[0, 0], dtype=c),
        "two_values": np.where(rng.random((rows, row_len)) < 0.3, u[0, 0], u[0, 1]).astype(c),
        "constant_top_byte": (u >> c(8)) | top if width(t) > 8 else u,
        "sorted": np.sort(u, axis=-1),
        "reversed": np.sort(u, axis=-1)[:, ::-1].copy(),
    }


@pytest.mark.parametrize("t", ["u16", "i32", "f32", "u64", "f64"])
@pytest.mark.parametrize("row_len", [200, 9000, 70_000])
def test_structured_inputs(g, t, row_len):
    rng = np.random.default_rng(row_len)
    rows = 3
    ranks = spread(row_len)
    with g.OneSweepSorter(1 << 20, 4, 0) as s:
        for name, bits in structured(rng, t, rows, row_len).items():
            x = dev(bits.reshape(-1), t).reshape(rows, row_len)
            order = order_of(bits, t, False)
            for hook in (0, 1):
                s.set_option("debug_long_rows", hook)
                v, i = s.select_rows(x, ranks, t)
                gi = i.cpu().numpy().astype(np.int64)
                assert np.array_equal(gi, order[:, ranks]), f"{name} {t} {row_len} hook={hook}: positions"
                assert np.array_equal(host(v, t), np.take_along_axis(bits, order[:, ranks], -1)), f"{name}: values"
                if name == "all_equal":
                    assert np.array_equal(gi, np.broadcast_to(ranks, gi.shape))


SPECIALS = {  # +0, -0, +inf, -inf, +NaN, -NaN, 1, -1
    "f16": [0x0000, 0x8000, 0x7C00, 0xFC00, 0x7E00, 0xFE00, 0x3C00, 0xBC00],
    "bf16": [0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0xFFC0, 0x3F80, 0xBF80],
    "f32": [0x0, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x3F800000, 0xBF800000],
    "f64": [0x0, 1 << 63, 0x7FF0 << 48, 0xFFF0 << 48, 0x7FF8 << 48, 0xFFF8 << 48, 0x3FF0 << 48, 0xBFF0 << 48],
}


@pytest.mark.parametrize("t", list(SPECIALS))
def test_zeros_infinities_and_nans(g, t):
    """the library's total order: -NaN < -inf < .. < -0.0 < +0.0 < .. < +inf < +NaN, stable among equal bits"""
    rng = np.random.default_rng(9)
    sp = np.array(SPECIALS[t], dtype=TYPES[t][1])
    with g.OneSweepSorter(1 << 20, 4, 0) as s:
        for row_len in (300, 30_000):
            bits = sp[rng.integers(0, len(sp), 2 * row_len)].reshape(2, row_len)
            x = dev(bits.reshape(-1), t).reshape(2, row_len)
            order = order_of(bits, t, False)
            ranks = spread(row_len)
            for hook in (0, 1):
                s.set_option("debug_long_rows", hook)
                v, i = s.select_rows(x, ranks, t)
                assert np.array_equal(i.cpu().numpy().astype(np.int64), order[:, ranks]), f"{t} {row_len} hook={hook}"
                assert np.array_equal(host(v, t), np.take_along_axis(bits, order[:, ranks], -1))
                check_against_sort(g, s, x, t, ranks, f"{t} specials {row_len} hook={hook}")


# ---- 4. both paths --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", list(TYPES))
def test_split_path_equals_short_path(g, t):
    rng = np.random.default_rng(KEY_TYPE[t] + 40)
    with g.OneSweepSorter(1 << 22, 4, 0) as s:
        for row_len in (2, 3, 33, 256, 1000, 2049, cap(t)):
            rows = 37
            x = dev(typed(rng, rows * row_len, t), t).reshape(rows, row_len)
            ranks = spread(row_len)
            s.set_option("debug_long_rows", 0)
            v0, i0 = s.select_rows(x, ranks, t)
            s.set_option("debug_rows_block", 1)
            v1, i1 = s.select_rows(x, ranks, t)
            s.set_option("debug_rows_block", 0)
            s.set_option("debug_long_rows", 1)
            v2, i2 = s.select_rows(x, ranks, t)
            w2 = s.select_rows(x, ranks, t, return_indices=False)
            s.set_option("debug_long_rows", 0)
            for what, v, i in (("block path", v1, i1), ("split path", v2, i2)):
                assert torch.equal(i, i0), f"{t} {row_len} {what}: positions"
                assert torch.equal(bits_of(v, t), bits_of(v0, t)), f"{t} {row_len} {what}: values"
            assert torch.equal(bits_of(w2, t), bits_of(v0, t))


# ---- 5. errors ------------------------------------------------------------------------------------------------------------
def call(g, h, x, out, idx, rows, row_len, ranks, kb, kt):
    arr = (ctypes.c_uint32 * max(len(ranks), 1))(*ranks)
    return g.lib.osb200_select_rows(h, x, out, idx, rows, row_len, arr if ranks is not None else None, len(ranks), kb, kt,
                                    torch.cuda.current_stream().cuda_stream)


def test_argument_errors_their_order_and_no_work(g):
    rows, row_len = 4, 20_000
    x = torch.randn(rows, row_len, device="cuda")
    out = torch.full((rows, 16), 7.0, device="cuda")
    idx = torch.full((rows, 16), 7, dtype=torch.int32, device="cuda")
    X, O, I = x.data_ptr(), out.data_ptr(), idx.data_ptr()
    with g.OneSweepSorter(1 << 10, 4, 0) as s:
        h = s._h
        F = KEY_TYPE["f32"]
        cases = {
            "null handle": (None, X, O, I, rows, row_len, [1], 4, F, INVALID_ARG),
            "bad key pair": (h, X, O, I, rows, row_len, [1], 4, KEY_TYPE["f64"], INVALID_ARG),
            "bad key pair before the no-op": (h, X, O, I, 0, row_len, [1], 3, F, INVALID_ARG),
            "no rows: a no-op before the arrays": (h, None, None, None, 0, row_len, [1], 4, F, OK),
            "no rows: a no-op before the ranks": (h, X, O, I, 0, row_len, [5, 1], 4, F, OK),
            "null input": (h, None, O, I, rows, row_len, [1], 4, F, INVALID_ARG),
            "null output": (h, X, None, I, rows, row_len, [1], 4, F, INVALID_ARG),
            "misaligned input": (h, X + 2, O, I, rows, row_len, [1], 4, F, INVALID_ARG),
            "misaligned indices": (h, X, O, I + 2, rows, row_len, [1], 4, F, INVALID_ARG),
            "sizes overflow": (h, X, O, I, 1 << 62, 1 << 8, [1], 4, F, INVALID_ARG),
            "output overlaps input": (h, X, X + 64, I, rows, row_len, [1], 4, F, INVALID_ARG),
            "indices overlap output": (h, X, O, O, rows, row_len, [1], 4, F, INVALID_ARG),
            "no ranks": (h, X, O, I, rows, row_len, [], 4, F, INVALID_ARG),
            "17 ranks": (h, X, O, I, rows, row_len, list(range(17)), 4, F, INVALID_ARG),
            "not increasing": (h, X, O, I, rows, row_len, [3, 3], 4, F, INVALID_ARG),
            "decreasing": (h, X, O, I, rows, row_len, [4, 3], 4, F, INVALID_ARG),
            "rank == row_len": (h, X, O, I, rows, row_len, [row_len], 4, F, INVALID_ARG),
            "bad ranks before the workspace": (h, X, O, I, rows, row_len, list(range(15)) + [row_len], 4, F, INVALID_ARG),
            "workspace too small": (h, X, O, I, rows, row_len, list(range(16)), 4, F, SIZE),
        }
        for what, (hh, xx, oo, ii, r, L, ranks, kb, kt, want) in cases.items():
            assert call(g, hh, xx, oo, ii, r, L, ranks, kb, kt) == want, what
        # a null rank array
        assert g.lib.osb200_select_rows(h, X, O, I, rows, row_len, None, 1, 4, F, None) == INVALID_ARG
        torch.cuda.synchronize()
        assert bool((out == 7.0).all()) and bool((idx == 7).all()), "a call that failed wrote its outputs"
        # a handle far smaller than n where the bound fits
        assert call(g, h, X, O, I, 1, row_len, [0, row_len // 2, row_len - 1], 4, F) == OK
        torch.cuda.synchronize()
        want = torch.sort(x[0], stable=True)
        assert torch.equal(out[0, :3], want.values[[0, row_len // 2, row_len - 1]])
        assert torch.equal(idx[0, :3].long(), want.indices[[0, row_len // 2, row_len - 1]])


def test_workspace_bound_is_exact(g):
    rows, row_len, ranks = 3, 50_000, [0, 7, 1000, 49_999]
    torch.manual_seed(1)
    x = torch.randn(rows, row_len, device="cuda")
    for indices in (True, False):
        need = g.select_workspace_words(rows, row_len, len(ranks), indices)
        with g.OneSweepSorter(need - 1, 4, 0) as s:
            with pytest.raises(g.OneSweepError, match="status -2"):
                s.select_rows(x, ranks, "f32", indices)
        with g.OneSweepSorter(need, 4, 0) as s:
            check_against_sort(g, s, x, "f32", ranks, f"exact bound indices={indices}", indices)
    # the hook on short rows needs the room too
    with g.OneSweepSorter(1 << 10, 4, 0) as s:
        s.set_option("debug_long_rows", 1)
        with pytest.raises(g.OneSweepError, match="status -2"):
            s.select_rows(torch.randn(100, 64, device="cuda"), [1, 2], "f32")


def test_row_len_one(g):
    x = torch.arange(12, dtype=torch.int64, device="cuda").reshape(12, 1)
    with g.OneSweepSorter(16, 4, 0) as s:
        for hook in (0, 1):
            s.set_option("debug_long_rows", hook)
            v, i = s.select_rows(x, [0], "i64")
            assert torch.equal(v, x) and bool((i == 0).all())


# ---- 6. graphs and shared handles ---------------------------------------------------------------------------------------
def test_graph_capture_and_replay_on_new_data(g):
    shapes = {"f32": ((4, 60_000), [0, 5, 30_000, 59_999]), "bf16": ((64, 500), [0, 249, 499]),
              "i64": ((3, 10_000), [1, 2, 3, 9999])}
    with g.OneSweepSorter(1 << 20, 4, 0) as s:
        bufs = {t: torch.zeros(shape, dtype=TYPES[t][0], device="cuda") for t, (shape, _) in shapes.items()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for t, bb in bufs.items():
                s.select_rows(bb, shapes[t][1], t)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        outs = {}
        with torch.cuda.graph(graph):
            for t, bb in bufs.items():
                outs[t] = s.select_rows(bb, shapes[t][1], t)
        rng = np.random.default_rng(3)
        for replay in range(3):
            data = {t: random_bits(rng, shape[0] * shape[1], t).reshape(shape) for t, (shape, _) in shapes.items()}
            for t, bb in bufs.items():
                bb.copy_(dev(data[t].reshape(-1), t).reshape(shapes[t][0]))
            graph.replay()
            torch.cuda.synchronize()
            for t, (_, ranks) in shapes.items():
                want_i = order_of(data[t], t, False)[:, ranks]
                assert np.array_equal(outs[t][1].cpu().numpy().astype(np.int64), want_i), f"replay {replay} {t}: positions"
                assert np.array_equal(host(outs[t][0], t), np.take_along_axis(data[t], want_i, -1)), f"replay {replay} {t}"
        del graph


def test_interleaved_with_long_sorts_on_one_handle(g):
    """a select between sort_long_rows and topk_long_rows on one handle and stream reads nothing they left behind"""
    torch.manual_seed(7)
    a = torch.randn(8, 100_000, device="cuda")
    b = torch.randn(2, 300_000, device="cuda")
    ranks = [0, 10, 50_000, 99_999]
    with g.OneSweepSorter(1 << 21, 4, 4) as s:
        want = torch.sort(a, dim=-1, stable=True)
        for _ in range(2):
            s.sort_long_rows(b, "f32")
            v, i = s.select_rows(a, ranks, "f32")
            s.topk_long_rows(b, 20_000, "f32")
            v2, i2 = s.select_rows(a, ranks, "f32")
            for vv, ii in ((v, i), (v2, i2)):
                assert torch.equal(vv, want.values[:, ranks]) and torch.equal(ii.long(), want.indices[:, ranks])


# ---- 7. against torch ---------------------------------------------------------------------------------------------------
def unique_in_row(x, v):
    return (x == v.unsqueeze(-1)).sum(-1) == 1


def stable_rule(x, v, i, k0):
    """positions obey the stable-sort rule: x[i] == v and exactly k0 - count(x < v) keys equal to v come before i"""
    assert torch.equal(torch.gather(x, -1, i.long().unsqueeze(-1)).squeeze(-1), v)
    below = (x < v.unsqueeze(-1)).sum(-1)
    pos = torch.arange(x.shape[-1], device=x.device)
    before = ((x == v.unsqueeze(-1)) & (pos < i.long().unsqueeze(-1))).sum(-1)
    assert torch.equal(below + before, torch.full_like(below, k0))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16, torch.int32, torch.int64, torch.int16])
@pytest.mark.parametrize("shape", [(1000, 64), (16, 3000), (4, 100_000)])
def test_kthvalue_and_median_against_torch(g, dtype, shape):
    torch.manual_seed(shape[-1])
    if dtype.is_floating_point:
        x = (torch.randn(shape, device="cuda", dtype=torch.float64) * 3).to(dtype)
        x = torch.where(x == 0, torch.ones_like(x), x)  # no -0.0
    else:
        x = torch.randint(-50, 50, shape, device="cuda").to(dtype)
    L = shape[-1]
    for k in (1, L // 3 + 1, L):
        v, i = g.kthvalue(x, k)
        tv, ti = torch.kthvalue(x, k)
        assert torch.equal(v, tv), f"kthvalue k={k}"
        u = unique_in_row(x, v)
        assert torch.equal(i.long()[u], ti[u])
        stable_rule(x, v, i, k - 1)
        vk, ik = g.kthvalue(x, k, keepdim=True)
        assert vk.shape == ik.shape == torch.kthvalue(x, k, keepdim=True).values.shape
    v, i = g.median(x, dim=-1)
    tv, ti = torch.median(x, dim=-1)
    assert torch.equal(v, tv)
    stable_rule(x, v, i, (L - 1) // 2)
    assert torch.equal(g.median(x), torch.median(x))
    assert g.median(x).shape == ()
    assert torch.equal(g.kthvalue(x, 5, dim=None)[0], torch.kthvalue(x.reshape(-1), 5)[0])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("interpolation", ["linear", "lower", "higher", "midpoint", "nearest"])
def test_quantile_against_torch(g, dtype, interpolation):
    torch.manual_seed(11)
    qs = [0.0, 1.0, 0.5, 0.25, 0.999, 1e-3, torch.linspace(0, 1, 37, dtype=dtype)]
    for shape in [(64, 1000), (3, 40_000), (5000,)]:
        x = (torch.randn(shape, device="cuda", dtype=dtype) * 3)
        x[x == 0] = 1
        for q in qs:
            for dim in (None, -1):
                for keepdim in (False, True):
                    want = torch.quantile(x, q if isinstance(q, float) else q.cuda(), dim=dim, keepdim=keepdim,
                                          interpolation=interpolation)
                    got = g.quantile(x, q, dim=dim, keepdim=keepdim, interpolation=interpolation)
                    assert got.shape == want.shape, (shape, q, dim, keepdim)
                    assert torch.equal(got, want), (shape, q if isinstance(q, float) else "1-D", dim, keepdim)
    # NaN rows, as torch
    x = torch.randn(6, 5000, device="cuda", dtype=dtype)
    x[1, 17] = float("nan")
    x[4, 3] = float("nan")
    q = torch.tensor([0.1, 0.5, 0.9], dtype=dtype)
    want = torch.quantile(x, q.cuda(), dim=-1, interpolation=interpolation)
    assert torch.equal(torch.isnan(want[1]), torch.tensor([False, True, False, False, True, False], device="cuda"))
    assert torch.allclose(g.quantile(x, q, dim=-1, interpolation=interpolation), want, rtol=0, atol=0, equal_nan=True)
    # a NaN with the sign bit set sorts first in this library's order, and its row is NaN too
    x[4, 3] = -float("nan")
    got = g.quantile(x, q, dim=-1, interpolation=interpolation)
    assert torch.equal(torch.isnan(got), torch.isnan(want))


def test_quantile_argument_errors(g):
    x = torch.randn(10, 20, device="cuda")
    with pytest.raises(ValueError):
        g.quantile(x, torch.tensor([0.5], device="cuda"))
    with pytest.raises(ValueError):
        g.quantile(x, 1.5)
    with pytest.raises(ValueError):
        g.quantile(x, 0.5, dim=0)
    with pytest.raises(TypeError):
        g.quantile(x.to(torch.int32), 0.5)
    with pytest.raises(ValueError):
        g.kthvalue(x, 21)
    with pytest.raises(ValueError):
        g.median(x, dim=0)


def test_quantile_above_2pow24(g):
    torch.manual_seed(24)
    n = (1 << 24) + 4099
    x = torch.randn(n, device="cuda") * 3
    x[x == 0] = 1
    q = torch.tensor([0.0, 0.01, 0.5, 0.99, 0.999, 1.0])
    with pytest.raises(RuntimeError):
        torch.quantile(x, q.cuda())
    srt = torch.sort(x).values
    pos = q * (n - 1)  # ATen's formula, in x's dtype
    below = pos.long().clamp(0, n - 1)
    above = pos.ceil().long().clamp(0, n - 1)
    want = torch.lerp(srt[below.cuda()], srt[above.cuda()], (pos - below.float()).cuda())
    assert torch.equal(g.quantile(x, q), want)
    # more than 16 distinct ranks, over several calls
    q2 = torch.linspace(0, 1, 41)
    pos = q2 * (n - 1)
    below = pos.long().clamp(0, n - 1)
    above = pos.ceil().long().clamp(0, n - 1)
    want = torch.lerp(srt[below.cuda()], srt[above.cuda()], (pos - below.float()).cuda())
    assert torch.equal(g.quantile(x, q2), want)


def test_module_sorter_grows_to_the_bound_not_to_numel(g):
    torch.manual_seed(2)
    x = torch.randn(1 << 22, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    assert torch.equal(g.median(x, stream=side), torch.median(x))
    s = g.onesweep._CACHE[(0, 4, 4, side.cuda_stream)]
    assert s.max_n < x.numel() and s.max_n >= g.select_workspace_words(1, x.numel(), 1)


# ---- 8. past 2^32 elements ----------------------------------------------------------------------------------------------
def test_bf16_rows_past_2pow32(g):
    rows, row_len = 2, (1 << 31) + 12_345
    x = torch.randint(-1000, 1000, (rows, row_len), device="cuda", dtype=torch.int16).to(torch.bfloat16)
    ranks = [0, 123_456_789, row_len // 2, row_len - 1]
    with g.OneSweepSorter(g.select_workspace_words(rows, row_len, len(ranks)), 4, 0) as s:
        v, i = s.select_rows(x, ranks, "bf16")
    for r in range(rows):
        row = x[r]
        for j, k0 in enumerate(ranks):
            vv, ii = v[r, j], int(i[r, j].item()) & 0xFFFFFFFF
            below = int((row < vv).sum())
            eq = int((row == vv).sum())
            assert below <= k0 < below + eq
            assert bool(row[ii] == vv)
            assert int((row[:ii] == vv).sum()) == k0 - below
