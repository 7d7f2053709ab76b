"""osb200_select_segments, OneSweepSorter.select_segments and the module functions select_segments, median_segments and
quantile_segments: the keys at given per-segment ranks of every ragged segment's ascending stable sort, and their positions
within the segment.

The yardstick is the library's own stable segment sort (sort_long_segments) gathered at offsets[s] + rank, bit for bit for
values and positions, and numpy's stable argsort of the radix images where the input is built on the host.  The three paths
-- warp class, block class, split path -- are compared on the same input through the "debug_rows_block" and
"debug_long_rows" hooks.  The test whose name contains "past_2pow" needs about 9 GB: -k "not past_2pow" leaves it out.  -m gpu"""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_topk import TYPES, dev, host, width
from tests.test_gpu_topk import radix as radix_images

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
KEY_TYPE = {"u16": 0, "i16": 1, "f16": 2, "bf16": 3, "u32": 0, "i32": 1, "f32": 2, "u64": 3, "i64": 4, "f64": 5}
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def cap(t):
    return 8192 if width(t) == 64 else 16384


def pad_bits(t):
    """the decoded all-ones radix image: the maximum of an unsigned type, 0x7F..F (INT_MAX, or a NaN) otherwise"""
    w = width(t)
    return TYPES[t][1]((1 << w) - 1 if TYPES[t][3] == "u" else (1 << (w - 1)) - 1)


def keys_for(rng, n, t, kind="random"):
    c = TYPES[t][1]
    if kind == "random":
        if TYPES[t][3] == "f":
            x = torch.randn(n, generator=torch.Generator().manual_seed(int(rng.integers(1 << 30))), dtype=torch.float64) * 3
            return x.to(TYPES[t][0]).view(getattr(torch, np.dtype(TYPES[t][2]).name)).numpy().view(c)
        bits = rng.integers(0, np.iinfo(c).max, n, dtype=c, endpoint=True)
        bits[::7] = bits[0]
        return bits
    u = rng.integers(0, np.iinfo(c).max, n, dtype=c, endpoint=True)
    top = c(0x5A) << c(width(t) - 8)
    if kind == "equal":
        return np.full(n, u[0] if n else 0, dtype=c)
    if kind == "two":
        return np.where(rng.integers(0, 2, n) == 1, u[0], u[1] if n > 1 else 0).astype(c)
    if kind == "top_byte":
        return (u >> c(8)) | top
    if kind == "sorted":
        return np.sort(u)
    if kind == "reversed":
        return np.sort(u)[::-1].copy()
    raise ValueError(kind)


def specials(t):
    """float bit patterns of +-0, +-inf and NaNs of both signs"""
    w = width(t)
    if TYPES[t][3] != "f":
        return []
    f = {"f16": np.float16, "bf16": None, "f32": np.float32, "f64": np.float64}[t]
    if f is None:
        vals = [0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0xFFC0, 0x7F81, 0x3F80]
    else:
        vals = [int(np.array(v, dtype=f).view(TYPES[t][1])) for v in (0.0, -0.0, np.inf, -np.inf, 1.0)]
        vals += [(1 << (w - 1)) - 1, (1 << w) - 1, ((1 << (w - 1)) - 1) ^ 1]  # NaNs of both signs
    return vals


def reference(bits, off, ranks2d, t, max_len):
    """values (bits) and positions of the oracle: numpy's stable argsort of each valid segment's radix images"""
    img = radix_images(bits[None, :], t, False)[0] if bits.size else np.zeros(0, np.uint64)
    S, R = ranks2d.shape
    vals = np.full((S, R), pad_bits(t), dtype=TYPES[t][1])
    pos = np.full((S, R), NONE, dtype=np.uint64)
    for s in range(S):
        lo, hi = int(off[s]), int(off[s + 1])
        if not (lo <= hi <= bits.size and hi - lo <= max_len):
            continue
        r = ranks2d[s].astype(np.uint64)
        if np.any(r[1:] < r[:-1]):
            continue
        L = hi - lo
        ok = r < L
        if not ok.any():
            continue
        order = np.argsort(img[lo:hi], kind="stable")
        p = order[r[ok].astype(np.int64)]
        vals[s, ok] = bits[lo:hi][p]
        pos[s, ok] = p
    return vals, pos


def run(s, x, offs, ranks, t, max_len, indices=True):
    """one osb200_select_segments call on sorter s with uint32 ranks [S, R] (numpy): (values bits, positions) on the host"""
    S, R = ranks.shape
    rk = torch.from_numpy(ranks.astype(np.uint32).view(np.int32)).cuda()
    v, i = s.select_segments(x, offs, rk, t, return_indices=indices, max_segment_len=max_len) if indices else (
        s.select_segments(x, offs, rk, t, return_indices=False, max_segment_len=max_len), None)
    vb = host(v, t).reshape(S, R)
    ib = i.cpu().numpy().view(np.uint32).astype(np.uint64).reshape(S, R) if indices else None
    return vb, ib


def check(g, s, bits, off, ranks, t, max_len, what, sort_yardstick=True):
    x = dev(bits, t)
    offs = torch.from_numpy(np.asarray(off, dtype=np.int64)).cuda()
    wv, wp = reference(bits, off, ranks, t, max_len)
    v, p = run(s, x, offs, ranks, t, max_len)
    assert np.array_equal(v, wv), f"{what}: values differ at {np.argwhere(v != wv)[:5].tolist()}"
    assert np.array_equal(p, wp), f"{what}: positions differ at {np.argwhere(p != wp)[:5].tolist()}"
    v2, _ = run(s, x, offs, ranks, t, max_len, indices=False)
    assert np.array_equal(v2, wv), f"{what}: values-only call differs"
    if sort_yardstick and len(off) > 1 and np.all(np.diff(off) >= 0) and off[-1] <= bits.size:
        # sort_long_segments gathered at offsets[s] + rank
        sv, si = g.sort_long_segments(x, offs, max_segment_len=max(int(np.diff(off).max()), 1))
        svb, sib = host(sv, t), si.cpu().numpy().view(np.uint32)
        for s_ in range(len(off) - 1):
            lo, L = int(off[s_]), int(off[s_ + 1] - off[s_])
            if L > max_len or np.any(np.diff(ranks[s_].astype(np.int64)) < 0):
                continue
            for j, r in enumerate(ranks[s_]):
                if r < L:
                    assert v[s_, j] == svb[lo + r] and p[s_, j] == sib[lo + r], f"{what}: segment {s_} rank {r} vs sort_long_segments"
    return v, p


def offsets_of(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


def random_ranks(rng, lengths, R, past=True):
    """R non-decreasing ranks per segment, some at or past the length and some repeated"""
    out = np.zeros((len(lengths), R), dtype=np.uint64)
    for s, L in enumerate(lengths):
        hi = int(L) + (3 if past else 0)
        r = np.sort(rng.integers(0, max(hi, 1), R))
        out[s] = r
    return out


@pytest.fixture(scope="module")
def sorter(g):
    s = g.OneSweepSorter(1 << 23, 4, 4)
    yield s
    s.close()


def edge_lengths(t):
    c = cap(t)
    return [0, 1, 2, 31, 256, 257, 2048, 2049, c, c + 1, 65_536, 151_936]


@pytest.mark.parametrize("t", list(TYPES))
def test_every_dtype_and_edge_length(g, sorter, t):
    rng = np.random.default_rng(width(t) + len(t))
    lengths = np.array(edge_lengths(t))
    rng.shuffle(lengths)
    bits = keys_for(rng, int(lengths.sum()), t)
    off = offsets_of(lengths)
    for R in (1, 16):
        ranks = random_ranks(rng, lengths, R)
        check(g, sorter, bits, off, ranks, t, int(lengths.max()), f"{t} R={R}")
    # median of every segment
    med = np.array([[max(L - 1, 0) // 2] for L in lengths], dtype=np.uint64)
    check(g, sorter, bits, off, med, t, int(lengths.max()), f"{t} median")


@pytest.mark.parametrize("t", ["f32", "i64", "bf16"])
def test_log_uniform_empty_and_tile_edges(g, sorter, t):
    rng = np.random.default_rng(7)
    lengths = np.exp(rng.uniform(0, np.log(1 << 17), 120)).astype(np.int64)
    lengths[rng.integers(0, 120, 30)] = 0
    lengths = np.concatenate([lengths, [8192, 8193, 2 * 8192, 2 * 8192 + 1, 16 * 8192, 16 * 8192 + 1, 0, 0]])
    bits = keys_for(rng, int(lengths.sum()), t)
    off = offsets_of(lengths)
    check(g, sorter, bits, off, random_ranks(rng, lengths, 16), t, int(lengths.max()), f"{t} log-uniform")
    # a loose bound above the largest segment, and a short-path bound with the long segments then padding
    check(g, sorter, bits, off, random_ranks(rng, lengths, 5), t, 1 << 20, f"{t} loose bound", sort_yardstick=False)
    check(g, sorter, bits, off, random_ranks(rng, lengths, 5), t, cap(t), f"{t} short-path bound", sort_yardstick=False)


@pytest.mark.parametrize("t", ["u32", "f64", "i16"])
def test_rank_sets(g, sorter, t):
    rng = np.random.default_rng(11)
    lengths = np.array([5, 300, 3000, 20_000, 0, 40_000, 1])
    bits = keys_for(rng, int(lengths.sum()), t, "two")  # ranks fall in runs of equal keys
    off = offsets_of(lengths)
    S = len(lengths)
    ranks = np.zeros((S, 16), dtype=np.uint64)
    ranks[0] = [0, 0, 1, 1, 2, 4, 4, 5, 5, 6, NONE, NONE, NONE, NONE, NONE, NONE]  # duplicates, past the length
    ranks[1] = np.full(16, NONE)  # all 0xFFFFFFFF
    ranks[2] = np.arange(16)[::-1]  # decreasing: the whole row is padding
    ranks[3] = np.sort(rng.integers(0, 20_000, 16))
    ranks[4] = np.zeros(16)
    ranks[5] = np.full(16, 39_999)
    ranks[6] = np.zeros(16)
    v, p = check(g, sorter, bits, off, ranks, t, 40_000, f"{t} rank sets")
    assert np.all(p[1] == NONE) and np.all(p[2] == NONE) and np.all(p[4] == NONE)
    # one rank per segment, differing per segment
    check(g, sorter, bits, off, np.array([[L // 3] for L in lengths], dtype=np.uint64), t, 40_000, f"{t} one rank")


@pytest.mark.parametrize("t", ["f32", "u64", "f16"])
def test_three_paths_agree(g, t):
    rng = np.random.default_rng(5)
    lengths = np.array([0, 1, 2, 3, 31, 100, 256, 257, 1000, 2048, 2049, 5000, cap(t), 1])
    bits = keys_for(rng, int(lengths.sum()), t)
    off = offsets_of(lengths)
    ranks = random_ranks(rng, lengths, 16)
    x, offs = dev(bits, t), torch.from_numpy(off).cuda()
    results = []
    for hook in (None, "debug_rows_block", "debug_long_rows"):
        with g.OneSweepSorter(1 << 22, 4, 4) as s:
            if hook:
                s.set_option(hook, 1)
            results.append(run(s, x, offs, ranks, t, cap(t)))
    wv, wp = reference(bits, off, ranks, t, cap(t))
    for (v, p), path in zip(results, ("warp/block", "block", "split")):
        assert np.array_equal(v, wv) and np.array_equal(p, wp), f"{t}: the {path} path differs"


@pytest.mark.parametrize("t", ["f32", "i64"])
def test_untrusted_offsets_and_guards(g, sorter, t):
    rng = np.random.default_rng(3)
    n = 100_000
    bits = keys_for(rng, n, t)
    off = np.array([0, 40_000, 10, 30_000, 30_000, 120_000, 50_000, 70_000, 99_990, n, 5, 5 + 20_000], dtype=np.int64)
    S, R = len(off) - 1, 7
    ranks = random_ranks(rng, np.maximum(np.diff(off), 0), R)
    x, offs = dev(bits, t), torch.from_numpy(off).cuda()
    G = 37
    for max_len in (cap(t), 25_000, 1 << 20):
        vbytes = np.dtype(TYPES[t][1]).itemsize
        vals = torch.full((S * R + 2 * G,), 0x3C, dtype={2: torch.int16, 4: torch.int32, 8: torch.int64}[vbytes], device="cuda")
        idx = torch.full((S * R + 2 * G,), 0x1234567, dtype=torch.int32, device="cuda")
        rk = torch.from_numpy(ranks.astype(np.uint32).view(np.int32)).cuda()
        st = g.lib.osb200_select_segments(sorter._h, x.data_ptr(), vals[G:].data_ptr(), idx[G:].data_ptr(), n, offs.data_ptr(), S,
                                          max_len, rk.data_ptr(), R, vbytes, KEY_TYPE[t], None)
        torch.cuda.synchronize()
        assert st == OK
        assert torch.all(vals[:G] == 0x3C) and torch.all(vals[G + S * R:] == 0x3C), "value guard words overwritten"
        assert torch.all(idx[:G] == 0x1234567) and torch.all(idx[G + S * R:] == 0x1234567), "index guard words overwritten"
        wv, wp = reference(bits, off, ranks, t, max_len)
        got_v = vals[G:G + S * R].cpu().numpy().view(TYPES[t][1]).reshape(S, R)
        got_p = idx[G:G + S * R].cpu().numpy().view(np.uint32).astype(np.uint64).reshape(S, R)
        assert np.array_equal(got_v, wv) and np.array_equal(got_p, wp), f"{t} max_len={max_len}"
    # valid segments that overlap past the long path's bounds (the whole input, eight times): padding or the true columns
    off = np.array([0, n] * 8 + [0], dtype=np.int64)
    offs, S = torch.from_numpy(off).cuda(), len(off) - 1
    ranks = np.tile(np.array([[0, 5, 50_000, n - 1]], dtype=np.uint64), (S, 1))
    v, p = run(sorter, x, offs, ranks, t, 1 << 20)
    wv, wp = reference(bits, off, ranks, t, 1 << 20)
    padded = p == NONE
    assert np.array_equal(v[~padded], wv[~padded]) and np.array_equal(p[~padded], wp[~padded])
    assert np.all(v[padded] == pad_bits(t))


@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("kind", ["equal", "two", "top_byte", "sorted", "reversed", "specials"])
def test_structured_inputs(g, sorter, t, kind):
    rng = np.random.default_rng(17)
    lengths = np.array([3, 200, 1500, cap(t) + 5, 40_000])
    n = int(lengths.sum())
    if kind == "specials":
        sp = specials(t)
        if not sp:
            pytest.skip("integer type")
        bits = np.array(sp, dtype=TYPES[t][1])[rng.integers(0, len(sp), n)]
    else:
        bits = keys_for(rng, n, t, kind)
    check(g, sorter, bits, offsets_of(lengths), random_ranks(rng, lengths, 16), t, 40_000, f"{t} {kind}")


def test_graph_replays_with_new_keys_and_ranks(g):
    rng = np.random.default_rng(23)
    t = "f32"
    lengths = np.array([10, 300, 5000, 30_000, 0, 70_000])
    off = offsets_of(lengths)
    S, R, n = len(lengths), 9, int(lengths.sum())
    x = dev(keys_for(rng, n, t), t)
    offs = torch.from_numpy(off).cuda()
    rk = torch.zeros((S, R), dtype=torch.int32, device="cuda")
    with g.OneSweepSorter(1 << 20, 4, 4) as s:
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            s.select_segments(x, offs, rk, t, True, 70_000, stream)  # warm up
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            v, i = s.select_segments(x, offs, rk, t, True, 70_000, stream)
        for rep in range(3):
            bits = keys_for(rng, n, t)
            ranks = random_ranks(rng, lengths, R)
            x.copy_(dev(bits, t))
            rk.copy_(torch.from_numpy(ranks.astype(np.uint32).view(np.int32)))
            graph.replay()
            torch.cuda.synchronize()
            wv, wp = reference(bits, off, ranks, t, 70_000)
            assert np.array_equal(host(v, t).reshape(S, R), wv), f"replay {rep}: values"
            assert np.array_equal(i.cpu().numpy().view(np.uint32).astype(np.uint64).reshape(S, R), wp), f"replay {rep}: positions"
        del graph


def test_argument_errors_and_their_order(g):
    fn = g.lib.osb200_select_segments
    S, R, n = 4, 3, 1000
    x = torch.zeros(n, dtype=torch.int32, device="cuda")
    off = torch.tensor([0, 10, 20, 30, n], dtype=torch.int64, device="cuda")
    rk = torch.zeros((S, R), dtype=torch.int32, device="cuda")
    out = torch.full((S * R,), 7, dtype=torch.int32, device="cuda")
    idx = torch.full((S * R,), 7, dtype=torch.int32, device="cuda")
    with g.OneSweepSorter(1 << 12, 4, 4) as s:
        h = s._h

        def call(h=h, xp=x.data_ptr(), op=out.data_ptr(), ip=idx.data_ptr(), nn=n, fp=off.data_ptr(), ss=S, ml=100, rp=rk.data_ptr(),
                 r=R, kb=4, kt=2):
            return fn(h, xp, op, ip, nn, fp, ss, ml, rp, r, kb, kt, None)

        assert call(h=None) == INVALID_ARG
        assert call(kb=3) == INVALID_ARG and call(kt=9) == INVALID_ARG
        assert call(ss=0, r=0) == OK  # no segments: a no-op before anything else
        assert call(op=None) == INVALID_ARG and call(fp=None) == INVALID_ARG and call(rp=None) == INVALID_ARG
        assert call(xp=None) == INVALID_ARG
        assert call(op=out.data_ptr() + 2) == INVALID_ARG  # misaligned
        assert call(ip=out.data_ptr()) == INVALID_ARG  # the outputs overlap
        assert call(rp=x.data_ptr()) == INVALID_ARG and call(rp=off.data_ptr()) == INVALID_ARG  # read arrays overlap
        assert call(op=x.data_ptr()) == INVALID_ARG
        assert call(r=0) == INVALID_ARG and call(r=17) == INVALID_ARG
        assert call(r=17, op=None) == INVALID_ARG
        torch.cuda.synchronize()
        assert torch.all(out == 7) and torch.all(idx == 7), "a refused call wrote its outputs"
        assert call() == OK
        assert call(xp=None, nn=0) == OK  # no keys: every segment is empty, every column padding
        torch.cuda.synchronize()
        assert torch.all(out == 0x7FFFFFFF) and torch.all(idx == -1)
    # the long path's bound: a handle without payloads is refused, one below the bound gives OSB200_ERR_SIZE
    n = 1 << 16
    x = torch.zeros(n, dtype=torch.int32, device="cuda")
    off = torch.tensor([0, 20_000, n], dtype=torch.int64, device="cuda")
    rk = torch.zeros((2, 16), dtype=torch.int32, device="cuda")
    out = torch.empty(32, dtype=torch.int32, device="cuda")
    idx = torch.empty(32, dtype=torch.int32, device="cuda")
    words = g.select_segments_workspace(n, 2, 16, 4, True)
    with g.OneSweepSorter(1 << 12, 4, 0) as s:
        assert fn(s._h, x.data_ptr(), out.data_ptr(), idx.data_ptr(), n, off.data_ptr(), 2, 50_000, rk.data_ptr(), 16, 4, 2, None) == INVALID_ARG
    with g.OneSweepSorter(words - 1, 4, 4) as s:
        assert fn(s._h, x.data_ptr(), out.data_ptr(), idx.data_ptr(), n, off.data_ptr(), 2, 50_000, rk.data_ptr(), 16, 4, 2, None) == SIZE
        # the short path needs no payloads: the same handle takes max_segment_len <= C
        assert fn(s._h, x.data_ptr(), out.data_ptr(), idx.data_ptr(), n, off.data_ptr(), 2, 16384, rk.data_ptr(), 16, 4, 2, None) == OK
    with g.OneSweepSorter(words, 4, 4) as s:
        assert fn(s._h, x.data_ptr(), out.data_ptr(), idx.data_ptr(), n, off.data_ptr(), 2, 50_000, rk.data_ptr(), 16, 4, 2, None) == OK
    torch.cuda.synchronize()


@pytest.mark.parametrize("t", ["f32", "u64"])
def test_loose_bound_on_small_inputs(g, t):
    """max_segment_len above C on fewer than C + 1 keys (and on none): the call is clamped to n and answers on any handle"""
    rng = np.random.default_rng(31)
    lengths = np.array([0, 1, 5, 300, 2000, 4000])
    bits = keys_for(rng, int(lengths.sum()), t)
    off = offsets_of(lengths)
    ranks = random_ranks(rng, lengths, 16)
    x, offs = dev(bits, t), torch.from_numpy(off).cuda()
    wv, wp = reference(bits, off, ranks, t, 1 << 17)
    for vb in (4, 0):  # payloads or none: the long path is not taken
        with g.OneSweepSorter(len(lengths), 4, vb) as s:
            for max_len in (1 << 17, 0xFFFFFFFF):
                v, p = run(s, x, offs, ranks, t, max_len)
                assert np.array_equal(v, wv) and np.array_equal(p, wp), (vb, max_len)
    # the test hook sends every segment of two or more keys down the long path; one key is not one
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        s.set_option("debug_long_rows", 1)
        v, p = run(s, x, offs, ranks, t, 1 << 17)
        assert np.array_equal(v, wv) and np.array_equal(p, wp)
        one = torch.from_numpy(np.array([0, 1], dtype=np.int64)).cuda()
        v, p = run(s, x[:1], one, np.array([[0, 1]], dtype=np.uint64), t, 1 << 17)
        assert v[0, 0] == bits[0] and p[0, 0] == 0 and p[0, 1] == NONE
    # no keys at all: every column padding
    empty = torch.zeros(3, dtype=torch.int64, device="cuda")
    with g.OneSweepSorter(4, 4, 4) as s:
        v, p = run(s, x[:0], empty, np.zeros((2, 3), dtype=np.uint64), t, 1 << 20)
    assert np.all(p == NONE) and np.all(v == pad_bits(t))
    # the module functions with max_segment_len given, eagerly and under stream capture
    xf = torch.randn(int(lengths.sum()), device="cuda")
    q = g.quantile_segments(xf, offs, 0.5, max_segment_len=20_000)
    m, mi = g.median_segments(xf, offs, max_segment_len=1 << 17)
    for s_ in range(1, len(lengths)):
        seg = xf[int(off[s_]):int(off[s_ + 1])].cpu()
        assert q[s_].item() == torch.quantile(seg, 0.5).item()
        assert m[s_].item() == torch.sort(seg, stable=True)[0][(seg.numel() - 1) // 2].item()
    assert q[0].isnan() and mi[0].item() == -1
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        g.median_segments(xf, offs, max_segment_len=1 << 17, stream=stream)
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        mg, _ = g.median_segments(xf, offs, max_segment_len=1 << 17, stream=stream)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(mg.view(torch.int32), m.view(torch.int32))
    del graph


def test_rank_arguments_of_the_python_layer(g):
    x = torch.randn(100, device="cuda")
    offs = torch.tensor([0, 40, 100], dtype=torch.int64, device="cuda")
    with pytest.raises(TypeError):
        g.select_segments(x, offs, torch.zeros((2, 1), dtype=torch.int64))  # a CPU tensor is not a sequence of shared ranks
    with g.OneSweepSorter(16, 4, 4) as s:
        with pytest.raises(TypeError):
            s.select_segments(x, offs, torch.zeros((2, 1), dtype=torch.int64), "f32")
    v, i = g.select_segments(x, offs, (r for r in (0, 5, 39)))  # a generator is read once
    assert v.shape == (2, 3)
    want = torch.sort(x[:40].cpu(), stable=True)
    assert i[0].tolist() == want[1][[0, 5, 39]].tolist()
    # out-of-range tensor ranks take no part
    v, i = g.select_segments(x, offs, torch.tensor([[0, 1 << 40], [-1, -1]], device="cuda"))
    assert i[0, 1].item() == -1 and i[1].tolist() == [-1, -1]


def test_segment_count_is_checked_against_the_handle(g):
    fn = g.lib.osb200_select_segments
    S = 100
    x = torch.zeros(1000, dtype=torch.int32, device="cuda")
    off = torch.arange(S + 1, dtype=torch.int64, device="cuda")
    rk = torch.zeros((S, 1), dtype=torch.int32, device="cuda")
    out = torch.empty(S, dtype=torch.int32, device="cuda")
    with g.OneSweepSorter(S - 1, 4, 4) as s:
        assert fn(s._h, x.data_ptr(), out.data_ptr(), None, 1000, off.data_ptr(), S, 1, rk.data_ptr(), 1, 4, 2, None) == SIZE
    with g.OneSweepSorter(S, 4, 4) as s:
        assert fn(s._h, x.data_ptr(), out.data_ptr(), None, 1000, off.data_ptr(), S, 1, rk.data_ptr(), 1, 4, 2, None) == OK
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_median_and_quantile_segments_match_torch(g, dtype):
    rng = np.random.default_rng(29)
    lengths = np.array([0, 1, 2, 3, 7, 100, 257, 3000, 20_000, 0, 50_000, 5])
    off = offsets_of(lengths)
    n = int(lengths.sum())
    x = (torch.randn(n, dtype=torch.float64, generator=torch.Generator().manual_seed(1)) * 3).to(dtype)
    x[int(off[3]) + 1] = float("nan")  # a NaN segment
    x[int(off[5]) + 10] = x[int(off[5]) + 11]  # ties
    xc, offs = x.cuda(), torch.from_numpy(off).cuda()
    mv, mi = g.median_segments(xc, offs)
    for s in range(len(lengths)):
        seg = x[off[s]:off[s + 1]]
        if seg.numel() == 0:
            assert mi[s].item() == -1
            continue
        if seg.isnan().any():
            continue  # torch.median returns a NaN there; this library orders NaNs by their bits
        tv, _ = torch.sort(seg, stable=True)
        assert mv[s].item() == tv[(seg.numel() - 1) // 2].item()
        assert seg[mi[s].item()].item() == mv[s].item()
    qs = [0.0, 0.01, 0.25, 0.5, 0.75, 0.99, 1.0]
    for interp in ("linear", "lower", "higher", "midpoint", "nearest"):
        got = g.quantile_segments(xc, offs, qs, interpolation=interp)
        got1 = g.quantile_segments(xc, offs, 0.3, interpolation=interp, max_segment_len=int(lengths.max()))
        assert got.shape == (len(qs), len(lengths)) and got1.shape == (len(lengths),)
        for s in range(len(lengths)):
            seg = x[off[s]:off[s + 1]]
            if seg.numel() == 0:
                assert got[:, s].isnan().all() and got1[s].isnan()
                continue
            want = torch.quantile(seg, torch.tensor(qs, dtype=dtype), interpolation=interp)
            w1 = torch.quantile(seg, 0.3, interpolation=interp)
            assert torch.equal(got[:, s].cpu().isnan(), want.isnan()), (interp, s)
            ok = ~want.isnan()
            assert torch.equal(got[:, s].cpu()[ok], want[ok]), (interp, s)
            assert (got1[s].isnan().item() and w1.isnan().item()) or got1[s].item() == w1.item(), (interp, s)
    # the module select_segments with shared ranks
    v, i = g.select_segments(xc, offs, [0, 2])
    assert v.shape == (len(lengths), 2) and i.dtype == torch.int32


def test_segment_straddling_past_2pow(g):
    t = "i16"
    n = (1 << 32) + (1 << 20)
    mid = 1 << 32
    off = np.array([0, mid - (1 << 19), mid + (1 << 19) + 3, n], dtype=np.int64)
    x = torch.randint(-3000, 3000, (n,), dtype=torch.int16, device="cuda")
    offs = torch.from_numpy(off).cuda()
    L = int(off[2] - off[1])
    ranks = np.array([[0, 1, L // 4, L // 2, L - 2, L - 1, L]] * 3, dtype=np.uint64)
    rk = torch.from_numpy(ranks.astype(np.uint32).view(np.int32)).cuda()
    with g.OneSweepSorter(1 << 22, 4, 4) as s:
        v, i = s.select_segments(x, offs, rk, t, True, n)
    seg = x[int(off[1]):int(off[2])]
    bits = host(seg, t)
    wv, wp = reference(bits, np.array([0, L]), ranks[1:2], t, L)
    assert np.array_equal(host(v[1], t), wv[0]) and np.array_equal(i[1].cpu().numpy().view(np.uint32).astype(np.uint64), wp[0])
    del x
    torch.cuda.empty_cache()
