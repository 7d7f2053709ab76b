"""osb200_sort_long_segments, OneSweepSorter.sort_long_segments and gpusorting_b200.sort_long_segments: osb200_sort_segments
for segments of any length.  Segments above the segment sort's limit C (16,384 keys, 8,192 for 64-bit keys) are sorted over
tiles of T = 8,192 keys with per-segment tile counts; the shorter ones by the segment sort's classes.

Every case compares keys and indices bit for bit with the numpy oracle of test_gpu_sort_segments.  Most go through the C
entry on sentinel-filled, guard-framed outputs, so they also prove what is not written: gaps between segments, segments
longer than max_segment_len, segments whose offsets decrease or pass n, and anything outside [0, n).  The plan cases assert
the executed passes of the handle's last plan: the GlobalHistogram counts all n keys, long segments or not.  -m gpu; the
past_2pow test needs about 40 GiB of free device memory."""
import gc

import numpy as np
import pytest
import torch

from tests.test_gpu_rows import KEY_TYPE, TYPES, dev, host, radix, random_bits, same, specials, typed_input, width
from tests.test_gpu_sort_segments import (GUARD, SENTINEL_IDX, edge_lengths, framed_idx, framed_keys, offsets_of, oracle,
                                          sentinel_bits, shuffled_edges)

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
T = 8192  # the long path's tile


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


@pytest.fixture(scope="module", autouse=True)
def release_device_memory():
    """hands the cached blocks of this module's large tensors back to the device when it ends, for the tests after it"""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def cap(t):
    return 8192 if width(t) == 64 else 16384


def sorter(g, t, max_n, rank_mode=None, indices=True):
    """a sorter whose workspace takes segments of t: (4, 4) for 16- and 32-bit keys, (8, 4) for 64-bit keys"""
    s = g.OneSweepSorter(max_n, 8 if width(t) == 64 else 4, 4 if indices else 0)
    if rank_mode is not None:
        if rank_mode == 0 and not s.info("atomic_order_ok"):
            s.close()
            pytest.skip("the atomic rank mode failed its self-test on this device")
        s.set_option("rank_mode", rank_mode)
    return s


def executed(bits, t):
    """the passes the plan runs: the digit places on which the n keys of the call are not all equal"""
    img = radix(bits.reshape(-1), t)
    return sum(int(np.unique((img >> img.dtype.type(8 * p)) & img.dtype.type(255)).size > 1) for p in range(width(t) // 8))


def call(s, keys_in, keys_out, idx, n, off_t, segs, max_len, t, descending, stream=None, entry="osb200_sort_long_segments"):
    from gpusorting_b200 import lib

    return getattr(lib, entry)(s._h, keys_in, keys_out, idx, n, off_t.data_ptr() if off_t is not None else None, segs, max_len,
                               width(t) // 8, KEY_TYPE[t], 1 if descending else 0,
                               int((stream or torch.cuda.current_stream()).cuda_stream))


def run_framed(s, bits, off, t, descending, max_len, indices=True, inplace=False, plan=None, entry="osb200_sort_long_segments"):
    """one call on sentinel-filled, guarded outputs; checks every element (guards included) against the oracle and, with
    plan, the executed pass count.  Returns the outputs' host copies."""
    n = bits.size
    off_t = torch.from_numpy(off).cuda()
    src = framed_keys(bits, t)
    out = src if inplace else framed_keys(bits, t, np.full(n, sentinel_bits(t), dtype=TYPES[t][1]))
    ix = framed_idx(n) if indices else None
    st = call(s, src.ptr, out.ptr, ix.ptr if ix else None, n, off_t, off.size - 1, max_len, t, descending, entry=entry)
    assert st == OK, st
    torch.cuda.synchronize()
    base = bits if inplace else np.full(n, sentinel_bits(t), dtype=TYPES[t][1])
    want_k, want_i = oracle(bits, off, n, max_len, t, descending, base, np.full(n, SENTINEL_IDX, dtype=np.uint32))
    gk = out.host()
    guard_k = np.full(GUARD, sentinel_bits(t), dtype=TYPES[t][1])
    same(gk[:GUARD], guard_k, "guard before the keys")
    same(gk[-GUARD:], guard_k, "guard after the keys")
    same(gk[GUARD:-GUARD], want_k, "keys")
    if not inplace:
        same(src.host()[GUARD:-GUARD], bits, "input modified")
    gi = None
    if ix:
        gi = ix.host()
        guard_i = np.full(GUARD, SENTINEL_IDX, dtype=np.uint32)
        same(gi[:GUARD], guard_i, "guard before the indices")
        same(gi[-GUARD:], guard_i, "guard after the indices")
        gi = gi[GUARD:-GUARD]
        same(gi, want_i, "indices")
    if plan is not None:
        assert s.info("last_executed_passes") == plan
    return gk[GUARD:-GUARD], gi


def ragged_offsets(rng, lens, max_len, start=5):
    """offsets of `lens` in a random order after `start` keys that no segment covers, with a skipped segment longer than
    max_len, a segment whose offsets decrease back into it, and a last segment that passes n.  Returns (offsets, n)."""
    lens = [int(x) for x in np.asarray(lens)[rng.permutation(len(lens))]]
    off, cur = [start], start
    for i, L in enumerate(lens):
        if i == len(lens) // 2:
            cur += max_len + 1 + int(rng.integers(0, 40))  # too long: a gap
            off.append(cur)
            cur -= int(rng.integers(1, 30))                 # decreasing: not written, and the next one starts inside the gap
            off.append(cur)
        cur += L
        off.append(cur)
    n = cur + 3
    off.append(n + 1)  # passes n
    return np.array(off, dtype=np.int64), n


def long_mix(t):
    c = cap(t)
    return [0, 0, 1, 1, 2, 3, 100, 256, 257, 2047, 3000, c, c + 1, c + 2, T - 1, 2 * T - 1, 2 * T + 1, 3 * T, 16 * T, 16 * T + 1]


# ---- 1. every dtype, both orders, both rank modes, a mix of every class and the tile and chunk edges ------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_types_orders_and_lengths(g, rank_mode, t, descending):
    rng = np.random.default_rng(list(TYPES).index(t) * 4 + descending * 2 + rank_mode)
    max_len = 16 * T + 1
    off, n = ragged_offsets(rng, long_mix(t) + list(rng.integers(0, 300, 40)), max_len)
    bits = typed_input(rng, n, t)
    with sorter(g, t, n, rank_mode) as s:
        run_framed(s, bits, off, t, descending, max_len, indices=False)
        run_framed(s, bits, off, t, descending, max_len, indices=True, plan=executed(bits, t))


@pytest.mark.parametrize("t", ["u16", "f32", "i64"])
def test_lengths_around_2pow20(g, t):
    rng = np.random.default_rng(11)
    lens = [(1 << 20) - 1, 1 << 20, (1 << 20) + 1, 5, 40000]
    off, n = ragged_offsets(rng, lens, 1 << 21)
    bits = typed_input(rng, n, t)
    with sorter(g, t, n) as s:
        for descending in (False, True):
            run_framed(s, bits, off, t, descending, 1 << 21)


@pytest.mark.parametrize("t", ["bf16", "u32", "i64"])
def test_in_place(g, t):
    rng = np.random.default_rng(13)
    max_len = 3 * T + 5
    off, n = ragged_offsets(rng, long_mix(t)[:-2] + list(rng.integers(0, 3000, 30)), max_len)
    bits = typed_input(rng, n, t)
    for rank_mode in (0, 1):
        with sorter(g, t, n, rank_mode) as s:
            run_framed(s, bits, off, t, True, max_len, inplace=True)
            run_framed(s, bits, off, t, False, max_len, inplace=True, indices=False)


# ---- 2. the short path and the test hook: the same output as sort_segments ----------------------------------------------------
@pytest.mark.parametrize("t", ["f16", "i32", "f64"])
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_debug_long_rows_equals_sort_segments(g, rank_mode, t):
    """with the hook every segment of 2 .. C keys takes the long path: a tile of counts (1 KiB) for every two keys at worst,
    so the handle is large for n"""
    rng = np.random.default_rng(17 + rank_mode)
    L = np.concatenate([edge_lengths(t), rng.integers(0, 300, 60)])
    off = offsets_of(L[rng.permutation(L.size)], start=3)
    n = int(off[-1]) + 4
    bits = typed_input(rng, n, t)
    with sorter(g, t, 1 << 27, rank_mode) as s:
        for descending in (False, True):
            want = run_framed(s, bits, off, t, descending, cap(t), entry="osb200_sort_segments")
            s.set_option("debug_long_rows", 1)
            got = run_framed(s, bits, off, t, descending, cap(t), plan=executed(bits, t))
            s.set_option("debug_long_rows", 0)
            same(got[0], want[0], "keys vs sort_segments")
            same(got[1], want[1], "indices vs sort_segments")


@pytest.mark.parametrize("t", ["bf16", "u32", "u64"])
def test_short_bound_is_sort_segments_on_any_handle(g, t):
    """max_segment_len <= C needs no workspace: a (4, 0) handle of max_n = num_segments runs 64-bit keys with indices"""
    rng = np.random.default_rng(19)
    L = shuffled_edges(rng, t)
    off = offsets_of(L)
    n = int(off[-1])
    bits = typed_input(rng, n, t)
    with g.OneSweepSorter(off.size, 4, 0) as s:
        for max_len in (cap(t), 300):
            want = run_framed(s, bits, off, t, True, max_len, entry="osb200_sort_segments")
            got = run_framed(s, bits, off, t, True, max_len)
            same(got[0], want[0], "keys")
            same(got[1], want[1], "indices")


# ---- 3. equal lengths: the same output as sort_long_rows ----------------------------------------------------------------------
@pytest.mark.parametrize("t", ["u16", "f32", "i64"])
def test_equal_lengths_match_sort_long_rows(g, t):
    rng = np.random.default_rng(23)
    for L, rows in ((cap(t) + 1, 5), (32000, 7), (151936, 3)):
        bits = typed_input(rng, rows * L, t)
        x = dev(bits, t)
        off = torch.arange(rows + 1, dtype=torch.int64, device="cuda") * L
        with sorter(g, t, rows * L) as s:
            for descending in (False, True):
                rk, ri = s.sort_long_rows(x.view(rows, L), t, descending)
                sk, si = s.sort_long_segments(x, off, t, descending)
                same(host(sk, t), host(rk, t).reshape(-1), f"{L}: keys")
                same(si.cpu().numpy(), ri.cpu().numpy().reshape(-1), f"{L}: indices")


# ---- 4. the plan: skipped places, odd and even executed counts, float specials, borders inside tiles ---------------------------
@pytest.mark.parametrize("t", ["u16", "f32", "u64"])
def test_all_equal_keys_execute_no_place(g, t):
    """no place executes: the copy home writes the keys and the positions 0 .. L - 1 inside the long segments only"""
    rng = np.random.default_rng(29)
    off, n = ragged_offsets(rng, [cap(t) + 1, 3 * T + 7, 40, 2, 500, T + 1], 4 * T)
    bits = np.full(n, random_bits(rng, 1, t)[0], dtype=TYPES[t][1])
    with sorter(g, t, n) as s:
        run_framed(s, bits, off, t, False, 4 * T, plan=0)
        run_framed(s, bits, off, t, True, 4 * T, indices=False, plan=0)
        run_framed(s, bits, off, t, False, 4 * T, inplace=True, plan=0)


@pytest.mark.parametrize("hi,places", [(1 << 8, 1), (1 << 16, 2), (1 << 20, 3)])
def test_int64_small_values(g, hi, places):
    rng = np.random.default_rng(31)
    off, n = ragged_offsets(rng, [20000, 3 * T + 1, 300, 17000, 5], 5 * T)
    bits = rng.integers(0, hi, n).astype(np.uint64)
    bits[0] = hi - 1  # every place below hi's top one differs
    with sorter(g, "i64", n) as s:
        for descending in (False, True):
            run_framed(s, bits, off, "i64", descending, 5 * T, plan=places)


@pytest.mark.parametrize("t", ["f16", "bf16", "f32", "f64"])
def test_float_specials(g, t):
    rng = np.random.default_rng(37)
    off, n = ragged_offsets(rng, [cap(t) + 1, 2 * T + 3, 100, 30000], 4 * T)
    sp = specials(t)
    bits = sp[rng.integers(0, sp.size, n)]
    with sorter(g, t, n) as s:
        for descending in (False, True):
            run_framed(s, bits, off, t, descending, 4 * T, plan=executed(bits, t))


@pytest.mark.parametrize("t", ["i16", "u32", "f64"])
def test_sorted_reversed_and_outlier_segments(g, t):
    """segments that start and end inside tiles: sorted, reversed, constant but for one outlier"""
    rng = np.random.default_rng(41)
    lens = [cap(t) + 1, 2 * T + 777, 3 * T - 5, 40001, 123]
    off, n = ragged_offsets(rng, lens, 4 * T + 100, start=4097)
    bits = typed_input(rng, n, t)
    for s_i in range(off.size - 1):
        lo, hi = int(off[s_i]), int(off[s_i + 1])
        if not (0 <= lo < hi <= n):
            continue
        seg = bits[lo:hi]
        kind = s_i % 3
        if kind == 0:
            bits[lo:hi] = seg[np.argsort(radix(seg, t), kind="stable")]
        elif kind == 1:
            bits[lo:hi] = seg[np.argsort(radix(seg, t), kind="stable")][::-1]
        else:
            bits[lo:hi] = seg[0]
            bits[lo + (hi - lo) // 2] = random_bits(rng, 1, t)[0]
    with sorter(g, t, n) as s:
        for descending in (False, True):
            run_framed(s, bits, off, t, descending, 4 * T + 100, plan=executed(bits, t))


@pytest.mark.parametrize("t,lengths", [("u16", list(range(1, 13)) + [cap("u16") + 3]), ("u32", [1, 2, 3, 5, cap("u32") + 3])])
def test_few_keys_at_misaligned_starts(g, t, lengths):
    """inputs that start off a 16-byte boundary, shorter than the keys before it: the plan's histogram must count exactly
    the n keys (a bound above C takes the long path's plan even with no long segment).  The row sort's long path under the
    test hook shares that plan."""
    from gpusorting_b200 import lib

    rng = np.random.default_rng(71)
    esz = width(t) // 8
    with sorter(g, t, 1 << 16) as s:
        for n in lengths:
            for k in range(16 // esz):
                bits = typed_input(rng, n, t)
                before, after = random_bits(rng, GUARD + k, t), random_bits(rng, GUARD, t)
                src = dev(np.concatenate([before, bits, after]), t)
                out = dev(np.full(n + 2 * GUARD + k, sentinel_bits(t), dtype=TYPES[t][1]), t)
                ix = torch.full((n + 2 * GUARD + k,), -1, dtype=torch.int32, device="cuda")
                at = GUARD + k
                off = offsets_of([n]) if n < 3 else offsets_of([1, n - 1])
                off_t = torch.from_numpy(off).cuda()
                for descending in (False, True):
                    st = call(s, src.data_ptr() + at * esz, out.data_ptr() + at * esz, ix.data_ptr() + at * 4, n, off_t,
                              off.size - 1, 1 << 20, t, descending)
                    assert st == OK, (n, k, st)
                    torch.cuda.synchronize()
                    want_k, want_i = oracle(bits, off, n, 1 << 20, t, descending, bits, np.zeros(n, dtype=np.uint32))
                    gk, gi = host(out, t), ix.cpu().numpy().view(np.uint32)
                    same(gk[at:at + n], want_k, f"{n} keys at +{k}: keys")
                    same(gi[at:at + n], want_i, f"{n} keys at +{k}: indices")
                    same(np.concatenate([gk[:at], gk[at + n:]]), np.full(at + GUARD, sentinel_bits(t), dtype=TYPES[t][1]),
                         f"{n} keys at +{k}: outside the keys")
                    assert (gi[:at] == 0xFFFFFFFF).all() and (gi[at + n:] == 0xFFFFFFFF).all(), f"{n} keys at +{k}: indices outside"
                    same(host(src, t)[at:at + n], bits, f"{n} keys at +{k}: input modified")
                    if n >= 2:  # one row of n keys on the long rows' path
                        s.set_option("debug_long_rows", 1)
                        st = lib.osb200_sort_long_rows(s._h, src.data_ptr() + at * esz, out.data_ptr() + at * esz,
                                                       ix.data_ptr() + at * 4, 1, n, esz, KEY_TYPE[t], 1 if descending else 0,
                                                       int(torch.cuda.current_stream().cuda_stream))
                        s.set_option("debug_long_rows", 0)
                        assert st == OK, (n, k, st)
                        torch.cuda.synchronize()
                        order = np.argsort(radix(bits, t, descending), kind="stable")
                        same(host(out, t)[at:at + n], bits[order], f"row of {n} at +{k}: keys")
                        same(ix.cpu().numpy().view(np.uint32)[at:at + n], order.astype(np.uint32), f"row of {n} at +{k}: indices")


# ---- 5. workspace: the worst case fits, one element less does not; argument errors -------------------------------------------
@pytest.mark.parametrize("t", ["bf16", "f32", "u64"])
def test_worst_case_workspace(g, t):
    """n == max_n in segments of C + 1 keys (the most tiles), then num_segments == max_n with mostly empty segments"""
    rng = np.random.default_rng(43)
    segs = 40
    n = segs * (cap(t) + 1)
    off = offsets_of([cap(t) + 1] * segs)
    bits = typed_input(rng, n, t)
    with sorter(g, t, n) as s:
        run_framed(s, bits, off, t, False, cap(t) + 1)
        # num_segments == max_n: empty segments, then three long ones
        many = np.zeros(n + 1, dtype=np.int64)
        many[-4:] = [n - 3 * (cap(t) + 1), n - 2 * (cap(t) + 1), n - (cap(t) + 1), n]
        run_framed(s, bits, many, t, True, cap(t) + 1)
    with sorter(g, t, n - 1) as s:
        x, y = dev(bits, t), dev(bits, t)
        off_t = torch.from_numpy(off).cuda()
        assert call(s, x.data_ptr(), y.data_ptr(), None, n, off_t, segs, cap(t) + 1, t, False) == SIZE


@pytest.mark.parametrize("t", ["bf16", "f32", "u64"])
def test_reductions_too_small_under_the_hook(g, t):
    """with the test hook a segment of two keys is long: the bound is a tile of counts per two keys, about 512 n bytes,
    which a handle of max_n = n cannot hold (OSB200_ERR_SIZE, nothing written), while the same call without the hook is
    sort_segments' launch on that handle"""
    rng = np.random.default_rng(73)
    n = 1 << 14
    off = offsets_of([n // 4] * 4)
    bits = typed_input(rng, n, t)
    with sorter(g, t, n) as s:
        s.set_option("debug_long_rows", 1)
        x = dev(bits, t)
        y = dev(np.full(n, sentinel_bits(t), dtype=TYPES[t][1]), t)
        off_t = torch.from_numpy(off).cuda()
        assert call(s, x.data_ptr(), y.data_ptr(), None, n, off_t, 4, n // 4, t, False) == SIZE
        torch.cuda.synchronize()
        same(host(y, t), np.full(n, sentinel_bits(t), dtype=TYPES[t][1]), "written after OSB200_ERR_SIZE")
        s.set_option("debug_long_rows", 0)
        run_framed(s, bits, off, t, False, n // 4)


def test_handle_shape_and_argument_errors(g):
    n, t = 3 * 20000, "f32"
    x = torch.zeros(2 * n + 16, dtype=torch.float64, device="cuda")
    y = torch.zeros(2 * n + 16, dtype=torch.float64, device="cuda")
    ix = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
    off = torch.zeros(n + 8, dtype=torch.int64, device="cuda")
    off[:4] = torch.tensor([0, 20000, 40000, n])
    p, q, r, o = x.data_ptr(), y.data_ptr(), ix.data_ptr(), off.data_ptr()

    def both(s, *args):
        a = g.lib.osb200_sort_segments(s._h if s else None, *args)
        b = g.lib.osb200_sort_long_segments(s._h if s else None, *args)
        return a, b

    with g.OneSweepSorter(n, 4, 0) as s:
        # the argument errors of sort_segments, in the same order, with a bound both calls take
        for args in ((None, q, r, n, o, 3, 64, 4, 2, 0, None), (p, None, r, n, o, 3, 64, 4, 2, 0, None),
                     (p, q, r, n, None, 3, 64, 4, 2, 0, None), (p + 2, q, r, n, o, 3, 64, 4, 2, 0, None),
                     (p, q + 1, r, n, o, 3, 64, 4, 2, 0, None), (p, q, r + 2, n, o, 3, 64, 4, 2, 0, None),
                     (p, q, r, n, o + 4, 3, 64, 4, 2, 0, None), (p, p + 4, r, n, o, 3, 64, 4, 2, 0, None),
                     (p, q, q, n, o, 3, 64, 4, 2, 0, None), (p, o, r, n, o, 3, 64, 4, 2, 0, None),
                     (p, q, r, n, o, 3, 64, 3, 2, 0, None), (p, q, r, n, o, 3, 64, 4, 5, 0, None),
                     (p, q, r, n, o, n + 1, 64, 4, 2, 0, None)):
            a, b = both(s, *args)
            assert a == b != OK, args
        assert both(None, p, q, r, n, o, 3, 64, 4, 2, 0, None) == (INVALID_ARG, INVALID_ARG)
        assert g.lib.osb200_sort_long_segments(s._h, p, q, None, n, o, 3, 0, 4, 2, 0, None) == OK  # no-op
        assert g.lib.osb200_sort_long_segments(s._h, p, q, None, n, o, 3, 20000, 4, 2, 0, None) == OK  # keys only, (4, 0)
        # indices on a handle without payloads; 8-byte keys on a 4-byte handle
        assert g.lib.osb200_sort_long_segments(s._h, p, q, r, n, o, 3, 20000, 4, 2, 0, None) == INVALID_ARG
        assert g.lib.osb200_sort_long_segments(s._h, p, q, None, n // 2, o, 1, 20000, 8, 5, 0, None) == INVALID_ARG
        assert g.lib.osb200_sort_long_segments(s._h, p, q, None, n + 1, o, 3, 20000, 4, 2, 0, None) == SIZE  # n > max_n
    with g.OneSweepSorter(2, 4, 4) as s:
        assert g.lib.osb200_sort_long_segments(s._h, p, q, r, n, o, 3, 20000, 4, 2, 0, None) == SIZE  # segments > max_n
    torch.cuda.synchronize()


# ---- 6. graphs, streams, a shared handle, the module function ----------------------------------------------------------------
def test_graph_capture_and_replay(g):
    """new keys and new offsets on every replay, the same max_segment_len"""
    rng = np.random.default_rng(47)
    t, n, segs, max_len = "f32", 300000, 12, 150000
    x = torch.zeros(n, dtype=torch.float32, device="cuda")
    off_t = torch.zeros(segs + 1, dtype=torch.int64, device="cuda")
    with sorter(g, t, n) as s:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            s.sort_long_segments(x, off_t, t, True, max_segment_len=max_len)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            v, i = s.sort_long_segments(x, off_t, t, True, max_segment_len=max_len)
        for replay in range(4):
            cuts = np.sort(rng.integers(0, n, segs - 1))
            off = np.concatenate([[0], cuts, [n]]).astype(np.int64)
            bits = typed_input(rng, n, t)
            if replay == 3:
                bits[:] = bits[0]
            x.copy_(dev(bits, t))
            off_t.copy_(torch.from_numpy(off))
            graph.replay()
            torch.cuda.synchronize()
            lo, hi = off[:-1], off[1:]
            ok = (lo <= hi) & (hi - lo <= max_len)
            want_k, want_i = oracle(bits, off, n, max_len, t, True, bits, np.zeros(n, dtype=np.uint32))
            mask = np.zeros(n, dtype=bool)
            for a, b in zip(lo[ok], hi[ok]):
                mask[a:b] = True
            same(host(v, t)[mask], want_k[mask], f"replay {replay}: keys")
            same(i.cpu().numpy().view(np.uint32)[mask], want_i[mask], f"replay {replay}: indices")
        del graph


def test_two_handles_on_two_streams(g):
    rng = np.random.default_rng(53)
    a, b = sorter(g, "u32", 1 << 20), sorter(g, "i64", 1 << 20)
    try:
        work = []
        for s, t in ((a, "u32"), (b, "i64")):
            off, n = ragged_offsets(rng, [50000, 20000, 300, 9000, 70000], 1 << 17)
            bits = typed_input(rng, n, t)
            work.append((s, t, bits, off, dev(bits, t), torch.from_numpy(off).cuda(), torch.cuda.Stream()))
        outs = []
        for s, t, bits, off, x, o, st in work:
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                outs.append(s.sort_long_segments(x, o, t, False, max_segment_len=1 << 17, stream=st))
        torch.cuda.synchronize()
        for (s, t, bits, off, x, o, st), (v, i) in zip(work, outs):
            n = bits.size
            wk, wi = oracle(bits, off, n, 1 << 17, t, False, host(v, t), i.cpu().numpy().view(np.uint32))
            same(host(v, t), wk, f"{t}: keys")
            same(i.cpu().numpy().view(np.uint32), wi, f"{t}: indices")
    finally:
        a.close()
        b.close()


def test_one_handle_shared_with_other_calls(g):
    """sort_long_segments alternating with the fused u32 sort, topk_segments and sort_segments on one (4, 4) handle: no
    call may read what another left in the reductions, the control block or the alternate buffers"""
    rng = np.random.default_rng(59)
    n = 1 << 21
    with g.OneSweepSorter(n, 4, 4) as s:
        for step in range(3):
            off, m = ragged_offsets(rng, [70000, 20001, 300, 16385, 2, 9000], 1 << 17)
            bits = typed_input(rng, m, "f32")
            run_framed(s, bits, off, "f32", step == 1, 1 << 17, plan=executed(bits, "f32"))
            u = rng.integers(0, 1 << 32, n, dtype=np.uint32)
            x = torch.from_numpy(u.view(np.int32).copy()).cuda()
            s.sort_keys(x)
            same(x.cpu().numpy().view(np.uint32), np.sort(u), f"step {step}: fused keys")
            lens = rng.integers(0, 3000, 200)
            so = offsets_of(lens)
            segs = typed_input(rng, int(so[-1]), "i32")
            xo = torch.from_numpy(so).cuda()
            topv, topi = s.topk_segments(dev(segs, "i32"), xo, 5, "i32", largest=True)
            v, i = s.sort_segments(dev(segs, "i32"), xo, "i32")
            wk, wi = oracle(segs, so, segs.size, 3000, "i32", False, segs, np.zeros(segs.size, dtype=np.uint32))
            same(host(v, "i32"), wk, f"step {step}: sort_segments keys")
            same(i.cpu().numpy().view(np.uint32), wi, f"step {step}: sort_segments indices")
            dk, di = oracle(segs, so, segs.size, 3000, "i32", True, segs, np.zeros(segs.size, dtype=np.uint32))
            tv, ti = host(topv, "i32"), topi.cpu().numpy().view(np.uint32)
            for j in range(0, 200, 7):
                m5 = min(5, int(lens[j]))
                same(tv[j, :m5], dk[so[j]:so[j] + m5], f"step {step}: top-k {j}")
                same(ti[j, :m5], di[so[j]:so[j] + m5], f"step {step}: top-k {j} indices")
            kb = typed_input(rng, 2 * 30000, "bf16")
            ob = offsets_of([30000, 30000])
            run_framed(s, kb, ob, "bf16", True, 30000, plan=executed(kb, "bf16"))


def test_module_function_grows_its_sorter(g):
    rng = np.random.default_rng(61)
    for n, t in ((200000, "f32"), (900000, "f32"), (300000, "i64"), (1 << 20, "bf16")):
        lens = [n // 2, n // 4, n - n // 2 - n // 4]
        off = offsets_of(lens)
        bits = typed_input(rng, n, t)
        v, i = g.sort_long_segments(dev(bits, t), torch.from_numpy(off).cuda(), descending=True)
        wk, wi = oracle(bits, off, n, n, t, True, bits, np.zeros(n, dtype=np.uint32))
        same(host(v, t), wk, f"{n} {t}: keys")
        same(i.cpu().numpy().view(np.uint32), wi, f"{n} {t}: indices")
        only = g.sort_long_segments(dev(bits, t), torch.from_numpy(off).cuda(), return_indices=False, max_segment_len=n)
        wk, _ = oracle(bits, off, n, n, t, False, bits, np.zeros(n, dtype=np.uint32))
        same(host(only, t), wk, f"{n} {t}: keys only")
    short = offsets_of([100, 3000, 7])
    bits = typed_input(rng, 3107, "u16")
    v, i = g.sort_long_segments(dev(bits, "u16"), torch.from_numpy(short).cuda())
    wk, wi = oracle(bits, short, 3107, 3107, "u16", False, bits, np.zeros(3107, dtype=np.uint32))
    same(host(v, "u16"), wk, "short: keys")
    same(i.cpu().numpy().view(np.uint32), wi, "short: indices")


# ---- 7. past 2^32 ----------------------------------------------------------------------------------------------------------------
def require(gib):
    free = torch.cuda.mem_get_info()[0]
    if free < gib * (1 << 30):
        pytest.skip(f"needs {gib} GiB of free device memory, {free / (1 << 30):.1f} GiB free")


def test_long_segment_past_2pow32_u16(g):
    """one long uint16 segment from 2^32 - 2^19 + 5 to 2^32 + 2^19 + 5, after a segment longer than max_segment_len (not
    written), sorted in place keys only: positions past 2^32 wrap in uint32 (about 36 GiB with the sorter)"""
    require(40)
    n = (1 << 32) + (1 << 20)
    lo, hi = (1 << 32) - (1 << 19) + 5, (1 << 32) + (1 << 19) + 5
    gen = torch.Generator(device="cuda").manual_seed(67)
    x = torch.randint(-(1 << 15), 1 << 15, (n,), generator=gen, device="cuda", dtype=torch.int16).view(torch.uint16)
    keep = x[lo - 4096:hi + 4096].clone()
    off = torch.tensor([0, lo, hi], dtype=torch.int64, device="cuda")
    with g.OneSweepSorter(n, 4, 0) as s:
        s.sort_long_segments(x, off, "u16", return_indices=False, inplace=True, max_segment_len=hi - lo)
        torch.cuda.synchronize()
        assert s.info("last_executed_passes") == 2
    got = x[lo - 4096:hi + 4096]
    assert torch.equal(got[:4096], keep[:4096]), "the skipped segment was written"
    assert torch.equal(got[-4096:], keep[-4096:]), "keys after the segment were written"
    want = torch.sort(keep[4096:-4096].view(torch.int16).int() & 0xFFFF, stable=True).values
    assert torch.equal(got[4096:-4096].view(torch.int16).int() & 0xFFFF, want)
