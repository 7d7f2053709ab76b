"""osb200_sort_segments, OneSweepSorter.sort_segments and gpusorting_b200.sort_segments: every segment [off[s], off[s+1]) of
a 1-D array sorted stable into the same positions, for 16-, 32- and 64-bit keys, with int32 indices within the segment.

The oracle is numpy's per-segment stable sort: lexsort on (radix image, segment id), the radix image as in the row sort's
tests (descending is the complement, so ties keep their order).  Keys and indices are compared bit for bit.  Most cases
call the C entry point on outputs filled with a sentinel and framed by guard regions, so they also prove what is NOT
written: positions outside every segment, segments longer than max_segment_len, segments whose offsets decrease or pass n,
and anything outside [0, n).  -m gpu"""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_rows import KEY_TYPE, TYPES, dev, host, radix, random_bits, same, typed_input

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
GUARD = 64
SENTINEL_IDX = 0xDEADBEEF


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def rank_mode_sorter(g, rank_mode, max_n=1 << 12):
    """a (4, 4) sorter in the given rank mode; its max_n bounds the segments per call"""
    s = g.OneSweepSorter(max_n, 4, 4)
    if rank_mode == 0 and not s.info("atomic_order_ok"):
        s.close()
        pytest.skip("the atomic rank mode failed its self-test on this device")
    s.set_option("rank_mode", rank_mode)
    return s


def width(t):
    return np.dtype(TYPES[t][1]).itemsize * 8


def cap(t):
    return 8192 if width(t) == 64 else 16384


def edge_lengths(t):
    """every class edge: empty, one key, the warp path's buckets, the block classes and the cap"""
    c = cap(t)
    return [0, 1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049, c - 1, c]


def offsets_of(lengths, start=0):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64) + start


def oracle(bits, off, n, max_len, t, descending, base_keys, base_idx):
    """expected keys and indices: base_* everywhere, each valid segment sorted stable in place"""
    keys, idx = base_keys.copy(), base_idx.copy()
    lo, hi = off[:-1].view(np.uint64), off[1:].view(np.uint64)  # the offsets are unsigned to the library
    ok = (lo <= hi) & (hi <= n) & (hi - lo <= max_len)
    L = np.where(ok, hi - lo, 0).astype(np.int64)
    lo = np.where(ok, lo, 0).astype(np.int64)
    seg = np.repeat(np.arange(L.size), L)
    start = np.repeat(lo, L)
    pos = start + (np.arange(int(L.sum())) - np.repeat(np.cumsum(L) - L, L))
    k = bits[pos]
    order = np.lexsort((radix(k, t, descending), seg))
    keys[pos] = k[order]
    idx[pos] = (pos - start)[order].astype(np.uint32)
    return keys, idx


def sentinel_bits(t):
    return np.array([0x5A5A5A5A5A5A5A5A & ((1 << width(t)) - 1)], dtype=TYPES[t][1])[0]


class Framed:
    """a device array of n elements framed by GUARD elements on each side, all set from host `fill`"""

    def __init__(self, fill, t_or_idx):
        self.t = t_or_idx
        self.n = fill.size - 2 * GUARD
        if t_or_idx == "idx":
            self.buf = torch.from_numpy(fill.view(np.int32).copy()).cuda()
        else:
            self.buf = dev(fill, t_or_idx)
        self.ptr = self.buf.data_ptr() + GUARD * self.buf.element_size()

    def host(self):
        return self.buf.cpu().numpy().view(np.uint32) if self.t == "idx" else host(self.buf, self.t)


def framed_keys(bits, t, fill=None):
    frame = np.full(bits.size + 2 * GUARD, sentinel_bits(t), dtype=TYPES[t][1])
    frame[GUARD:GUARD + bits.size] = bits if fill is None else fill
    return Framed(frame, t)


def framed_idx(n):
    return Framed(np.full(n + 2 * GUARD, SENTINEL_IDX, dtype=np.uint32), "idx")


def call(s, keys_in, keys_out, idx, n, off_t, segs, max_len, t, descending, stream=None):
    from gpusorting_b200 import lib

    kb = width(t) // 8
    st = lib.osb200_sort_segments(s._h, keys_in, keys_out, idx, n, off_t.data_ptr() if off_t is not None else None, segs,
                                    max_len, kb, KEY_TYPE[t], 1 if descending else 0,
                                    int((stream or torch.cuda.current_stream()).cuda_stream))
    return st


def run_framed(s, bits, off, t, descending, max_len=None, indices=True, inplace=False, n=None):
    """one call on sentinel-filled, guarded outputs; checks every element (guards included) against the oracle"""
    n = bits.size if n is None else n
    max_len = cap(t) if max_len is None else max_len
    off_t = torch.from_numpy(off).cuda()
    src = framed_keys(bits, t)
    out = src if inplace else framed_keys(bits, t, np.full(bits.size, sentinel_bits(t), dtype=TYPES[t][1]))
    ix = framed_idx(bits.size) if indices else None
    st = call(s, src.ptr, out.ptr, ix.ptr if ix else None, n, off_t, off.size - 1, max_len, t, descending)
    assert st == OK, st
    torch.cuda.synchronize()
    base = bits if inplace else np.full(bits.size, sentinel_bits(t), dtype=TYPES[t][1])
    want_k, want_i = oracle(bits, off, n, max_len, t, descending, base,
                            np.full(bits.size, SENTINEL_IDX, dtype=np.uint32))
    gk = out.host()
    same(gk[:GUARD], np.full(GUARD, sentinel_bits(t), dtype=TYPES[t][1]), "guard before the keys")
    same(gk[-GUARD:], np.full(GUARD, sentinel_bits(t), dtype=TYPES[t][1]), "guard after the keys")
    same(gk[GUARD:-GUARD], want_k, "keys")
    if not inplace:
        same(src.host()[GUARD:-GUARD], bits, "input modified")
    if ix:
        gi = ix.host()
        same(gi[:GUARD], np.full(GUARD, SENTINEL_IDX, dtype=np.uint32), "guard before the indices")
        same(gi[-GUARD:], np.full(GUARD, SENTINEL_IDX, dtype=np.uint32), "guard after the indices")
        same(gi[GUARD:-GUARD], want_i, "indices")


def shuffled_edges(rng, t, extra=300):
    """every class edge, twice, among random lengths (most of them short), in a random order"""
    L = np.concatenate([edge_lengths(t) * 2, rng.integers(0, 300, extra), rng.integers(0, cap(t) + 1, 6)])
    return L[rng.permutation(L.size)]


# ---- 1. every dtype, both orders, both rank modes, lengths at every class edge ----------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_types_orders_and_class_edges(g, rank_mode, t, descending):
    rng = np.random.default_rng(list(TYPES).index(t) * 4 + descending * 2 + rank_mode)
    L = shuffled_edges(rng, t)
    off = offsets_of(L)
    bits = typed_input(rng, int(off[-1]), t)
    with rank_mode_sorter(g, rank_mode) as s:
        run_framed(s, bits, off, t, descending, indices=False)
        run_framed(s, bits, off, t, descending, indices=True)


# ---- 2. low-entropy keys: stability ---------------------------------------------------------------------------------
@pytest.mark.parametrize("t", ["i16", "f32", "u64"])
def test_low_entropy_stability(g, t):
    rng = np.random.default_rng(5)
    L = shuffled_edges(rng, t)
    off = offsets_of(L)
    bits = random_bits(rng, 3, t)[rng.integers(0, 3, int(off[-1]))]
    with g.OneSweepSorter(1 << 12, 4, 4) as s:
        for descending in (False, True):
            run_framed(s, bits, off, t, descending)


# ---- 3. in place with indices: each segment is sorted by exactly one kernel ------------------------------------------------
@pytest.mark.parametrize("t", ["bf16", "u32", "i64"])
def test_in_place_sorted_exactly_once(g, t):
    """a segment sorted twice in place would end with the identity as its indices"""
    rng = np.random.default_rng(7)
    L = shuffled_edges(rng, t)
    off = offsets_of(L)
    bits = typed_input(rng, int(off[-1]), t)
    for rank_mode in (0, 1):
        with rank_mode_sorter(g, rank_mode) as s:
            run_framed(s, bits, off, t, True, inplace=True)
            run_framed(s, bits, off, t, False, inplace=True, indices=False)


# ---- 4. equal lengths: the same output as sort_rows and osb200_segmented_sort_u32 -----------------------------------------
@pytest.mark.parametrize("t", ["f16", "u32", "f32", "f64"])
def test_equal_lengths_match_sort_rows(g, t):
    rng = np.random.default_rng(9)
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        for L in (1, 32, 200, 256, 257, 2048, 4096, cap(t)):
            rows = max(3, 60_000 // L)
            bits = typed_input(rng, rows * L, t)
            x = dev(bits, t)
            off = torch.arange(rows + 1, dtype=torch.int64, device="cuda") * L
            for descending in (False, True):
                rk, ri = s.sort_rows(x.view(rows, L), t, descending)
                sk, si = s.sort_segments(x, off, t, descending)
                same(host(sk, t), host(rk, t).reshape(-1), f"keys, rows of {L}")
                same(si.cpu().numpy(), ri.cpu().numpy().reshape(-1), f"indices, rows of {L}")
            if t == "u32":
                keys = x.clone()
                pay = torch.arange(rows * L, dtype=torch.int32, device="cuda")
                s.segmented_sort(keys, off, pay, max_segment_len=L)
                sk, si = s.sort_segments(x, off, t)
                same(host(sk, t), host(keys, t), f"segmented_sort_u32 keys, rows of {L}")
                same(si.cpu().numpy(), (pay - off[:-1].repeat_interleave(L).int()).cpu().numpy(),
                     f"segmented_sort_u32 payloads, rows of {L}")


# ---- 5. what is not written ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", ["u16", "f32", "f64"])
def test_nothing_written_outside_valid_segments(g, t):
    rng = np.random.default_rng(11)
    c = cap(t)
    with g.OneSweepSorter(1 << 12, 4, 4) as s:
        # off[0] > 0, a gap, empty segments, and positions after off[-1]
        L = np.array([5, 0, 0, 300, 1, 0, 3000, 40])
        off = offsets_of(L, start=17)
        n = int(off[-1]) + 29
        bits = typed_input(rng, n, t)
        run_framed(s, bits, off, t, False)
        run_framed(s, bits, off, t, True, inplace=True)
        # segments longer than max_segment_len, for bounds in every class
        L = shuffled_edges(rng, t, extra=100)
        off = offsets_of(L)
        bits = typed_input(rng, int(off[-1]), t)
        for bound in (1, 2, 33, 256, 257, 2048, 2049, c - 1):
            run_framed(s, bits, off, t, False, max_len=bound)
            run_framed(s, bits, off, t, True, max_len=bound, inplace=True)
        # decreasing offsets and offsets past n: those segments are skipped (their neighbours that are valid are sorted),
        # and nothing outside [0, n) is touched
        n = 5000
        bits = typed_input(rng, n, t)
        # valid: [0, 100), [150, 200), [3000, 3200), [3300, 3400), [4200, n); the rest pass n or decrease (-5 is 2^64 - 5)
        off = np.array([0, 100, n + 50, 150, 200, n + 7, 3000, 3200, 2 ** 62, 3300, 3400, -5, 4200, 4200, n], dtype=np.int64)
        run_framed(s, bits, off, t, False, max_len=c)
        run_framed(s, bits, off, t, True, max_len=c, inplace=True)
        # 2^20 segments of 0-8 keys
        L = rng.integers(0, 9, 1 << 20)
        off = offsets_of(L)
        bits = typed_input(rng, int(off[-1]), t)
    with g.OneSweepSorter(1 << 20, 4, 4) as s:
        run_framed(s, bits, off, t, True)
        run_framed(s, bits, off, t, False, inplace=True, indices=False)


# ---- 6. argument errors -----------------------------------------------------------------------------------------------------
def test_argument_errors(g):
    t = "f32"
    with g.OneSweepSorter(1000, 4, 0) as s:
        n = 64
        # room for every size the calls below state (8-byte keys; 1,001 segments), so no range reaches another allocation
        x = torch.zeros(2 * n + 16, dtype=torch.float32, device="cuda")
        y = torch.zeros(2 * n + 16, dtype=torch.float32, device="cuda")
        ix = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
        off = torch.zeros(1100, dtype=torch.int64, device="cuda")
        off[:3] = torch.tensor([0, 10, n])
        p, q, r = x.data_ptr(), y.data_ptr(), ix.data_ptr()

        def go(keys_in=p, keys_out=q, idx=r, nn=n, offs=off.data_ptr(), segs=2, max_len=64, kb=4, kt=KEY_TYPE[t]):
            return g.lib.osb200_sort_segments(s._h, keys_in, keys_out, idx, nn, offs, segs, max_len, kb, kt, 0, None)

        assert go() == OK
        assert go(keys_out=p) == OK  # in place
        assert go(idx=None) == OK
        assert g.lib.osb200_sort_segments(None, p, q, r, n, off.data_ptr(), 2, 64, 4, 2, 0, None) == INVALID_ARG
        assert go(keys_in=None) == INVALID_ARG
        assert go(keys_out=None) == INVALID_ARG
        assert go(offs=None) == INVALID_ARG
        assert go(keys_in=p + 2) == INVALID_ARG  # misaligned keys
        assert go(keys_out=q + 1) == INVALID_ARG
        assert go(idx=r + 2) == INVALID_ARG
        assert go(offs=off.data_ptr() + 4) == INVALID_ARG  # offsets are 8-byte aligned
        assert go(keys_out=p + 4) == INVALID_ARG  # overlaps the input
        assert go(idx=p + 4) == INVALID_ARG
        assert go(idx=q) == INVALID_ARG
        assert go(keys_out=off.data_ptr()) == INVALID_ARG  # writes over the offsets
        assert go(kb=3) == INVALID_ARG
        assert go(kt=KEY_TYPE["f64"]) == INVALID_ARG  # a type of another width
        assert go(kb=2, kt=7) == INVALID_ARG
        assert go(max_len=16385) == SIZE
        assert go(kb=8, kt=KEY_TYPE["f64"], max_len=8193) == SIZE
        assert go(segs=1001) == SIZE  # more segments than the handle's max_n
        # no-ops: nothing is validated past the key type and nothing is launched
        assert go(max_len=0, keys_in=None) == OK
        assert go(segs=0, offs=None) == OK
        assert go(nn=0, keys_out=None) == OK
        torch.cuda.synchronize()
    with g.OneSweepSorter(1 << 16, 8, 0) as s:  # any handle will do
        x = torch.randn(5000, dtype=torch.float64, device="cuda")
        off = torch.tensor([0, 3000, 5000], dtype=torch.int64, device="cuda")
        v, i = s.sort_segments(x, off, "f64")
        want = torch.cat([torch.sort(x[:3000], stable=True)[0], torch.sort(x[3000:], stable=True)[0]])
        assert torch.equal(v, want)
    with pytest.raises(TypeError):
        g.sort_segments(torch.zeros(10, dtype=torch.int8, device="cuda"), torch.tensor([0, 10], device="cuda"))


# ---- 7. CUDA graphs and a side stream ---------------------------------------------------------------------------------
def test_graph_capture_and_side_stream(g):
    t = "bf16"
    rng = np.random.default_rng(13)
    L = shuffled_edges(rng, t)
    off_np = offsets_of(L)
    n = int(off_np[-1])
    off = torch.from_numpy(off_np).cuda()
    x = dev(typed_input(rng, n, t), t)
    with g.OneSweepSorter(1 << 12, 4, 4) as s:
        s.sort_segments(x, off, t, max_segment_len=cap(t))  # warm-up: occupancy queries are made outside the capture
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                vals, idx = s.sort_segments(x, off, t, descending=True, max_segment_len=cap(t), stream=side)
        for seed in range(3):
            bits = typed_input(np.random.default_rng(100 + seed), n, t)
            x.copy_(dev(bits, t))
            graph.replay()
            torch.cuda.synchronize()
            want_k, want_i = oracle(bits, off_np, n, cap(t), t, True, np.zeros(n, TYPES[t][1]), np.zeros(n, np.uint32))
            same(host(vals, t), want_k, f"replay {seed}: keys")
            same(idx.cpu().numpy().view(np.uint32), want_i, f"replay {seed}: indices")
        # eager on a side stream, through the module-level call (its own cached sorter per stream)
        bits = typed_input(rng, n, t)
        x2 = dev(bits, t)
        with torch.cuda.stream(side):
            side.wait_stream(torch.cuda.default_stream())
            v2, i2 = g.sort_segments(x2, off, stream=side)
        side.synchronize()
        want_k, want_i = oracle(bits, off_np, n, cap(t), t, False, np.zeros(n, TYPES[t][1]), np.zeros(n, np.uint32))
        same(host(v2, t), want_k, "side stream: keys")
        same(i2.cpu().numpy().view(np.uint32), want_i, "side stream: indices")


# ---- 8. past 2^32 elements -----------------------------------------------------------------------------------------------
def test_keys16_segments_past_2pow32(g):
    """int16 segments that lie beyond element 2^32, in place with indices; positions before and after them untouched"""
    n = (1 << 32) + 200_000
    need = n * 2 + n * 4 + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need + (4 << 30):
        pytest.skip(f"needs {(need + (4 << 30)) / 2**30:.1f} GiB free, {free / 2**30:.1f} GiB are")
    t = "i16"
    rng = np.random.default_rng(17)
    L = shuffled_edges(rng, t, extra=40)
    start = (1 << 32) - 3000  # the first segment straddles 2^32
    off_np = offsets_of(L, start=start)
    end = int(off_np[-1])
    assert end <= n
    x = torch.empty(n, dtype=torch.int16, device="cuda")
    ix = torch.empty(n, dtype=torch.int32, device="cuda")
    lo, hi = start - 1000, min(n, end + 1000)
    bits = typed_input(rng, hi - lo, t)
    x[lo:hi] = dev(bits, t)
    ix[lo:hi] = -1
    off = torch.from_numpy(off_np).cuda()
    with g.OneSweepSorter(1 << 12, 4, 4) as s:
        assert call(s, x.data_ptr(), x.data_ptr(), ix.data_ptr(), n, off, off_np.size - 1, cap(t), t, False) == OK
        torch.cuda.synchronize()
    want_k, want_i = oracle(bits, off_np - lo, hi - lo, cap(t), t, False, bits, np.full(hi - lo, 0xFFFFFFFF, np.uint32))
    same(host(x[lo:hi], t), want_k, "keys past 2^32")
    same(ix[lo:hi].cpu().numpy().view(np.uint32), want_i, "indices past 2^32")
    del x, ix
    torch.cuda.empty_cache()


# ---- 9. 2^26 keys in ragged segments against the torch composite ----------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.int64])
def test_large_ragged_matches_torch(g, dtype):
    """values and indices equal a stable sort by key followed by a stable sort by segment id (no NaN or -0.0 here)"""
    n = 1 << 26
    gen = torch.Generator(device="cuda").manual_seed(19)
    lengths = torch.exp(torch.rand(n // 1000, device="cuda", generator=gen) * np.log(16384 if dtype != torch.int64 else 8192))
    lengths = lengths.long().clamp(1)
    lengths = lengths[: int((lengths.cumsum(0) <= n).sum())]
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), lengths.cumsum(0)])
    m = int(off[-1])
    if dtype == torch.int64:
        x = torch.randint(-(1 << 40), 1 << 40, (m,), device="cuda", generator=gen)
    else:
        x = (torch.randn(m, device="cuda", generator=gen) * 100).round().to(dtype)  # ties
        x = torch.where(x == 0, torch.ones_like(x), x)  # no -0.0
    seg = torch.repeat_interleave(torch.arange(lengths.numel(), device="cuda"), lengths)
    for descending in (False, True):
        v1, o1 = torch.sort(x, stable=True, descending=descending)
        _, o2 = torch.sort(seg[o1], stable=True)
        perm = o1[o2]
        want_v, want_i = x[perm], perm - off[:-1].repeat_interleave(lengths)
        v, i = g.sort_segments(x, off, descending=descending, max_segment_len=int(lengths.max()))
        assert torch.equal(v.view(torch.int16 if dtype == torch.bfloat16 else v.dtype),
                           want_v.view(torch.int16 if dtype == torch.bfloat16 else want_v.dtype))
        assert torch.equal(i.long(), want_i)
