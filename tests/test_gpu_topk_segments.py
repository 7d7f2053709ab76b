"""osb200_topk_segments, OneSweepSorter.topk_segments and gpusorting_b200.topk_segments: the k smallest or largest keys of every
ragged segment given by offsets and their int32 positions, as rows of a [num_segments, k] output padded past each segment's
length.

The oracle is a vectorised numpy one: a stable lexsort of (radix image, segment id), cut to m = min(length, k) per segment and
padded with the key of the all-ones radix image and index -1 (tests/test_gpu_topk.py's radix helpers).  sorted=True must equal
it bit for bit; sorted=False must hold the same (key, position) pairs in columns 0 .. m-1 and exactly the padding after them.
The tests whose names contain "past_2pow" need up to about 40 GiB and skip, saying so, when less is free.  -m gpu"""
import numpy as np
import pytest
import torch

from tests.test_gpu_large_n import release, require
from tests.test_gpu_topk import (GUARD, KEY_TYPE, TYPES, cap, dev, from_radix, host, radix, random_bits, same, typed_input,
                                 width)
from tests.topk_plan import candidates_row

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
PAD_IDX = 0xFFFFFFFF


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def pad_key(t, largest):
    """the bit pattern whose radix image in the selection order is all ones"""
    c = TYPES[t][1]
    return from_radix(np.array([0 if largest else np.iinfo(c).max], dtype=c), t)[0]


def oracle(bits, off, k, t, largest):
    """(keys [S, k], uint32 indices [S, k]) of the segments [off[s], off[s+1]) of bits"""
    n, S = bits.size, off.size - 1
    lo, hi = off[:-1].astype(np.int64), off[1:].astype(np.int64)
    valid = (lo <= hi) & (hi <= n) & (hi - lo < (1 << 32))
    L = np.where(valid, hi - lo, 0)
    keys = np.full((S, k), pad_key(t, largest), dtype=TYPES[t][1])
    idx = np.full((S, k), PAD_IDX, dtype=np.uint32)
    total = int(L.sum())
    if total == 0 or k == 0:
        return keys, idx
    seg = np.repeat(np.arange(S), L)
    start = np.cumsum(L) - L
    pos = np.arange(total) - start[seg]
    gidx = lo[seg] + pos
    order = np.lexsort((radix(bits[gidx], t, largest), seg))
    rank = np.arange(total) - start[seg[order]]
    keep = rank < k
    o = order[keep]
    keys[seg[o], rank[keep]] = bits[gidx[o]]
    idx[seg[o], rank[keep]] = pos[o]
    return keys, idx


def check(s, x_bits, off, k, t, largest, what, x=None, offs=None):
    """topk_segments sorted and unsorted against the oracle"""
    x = dev(x_bits, t) if x is None else x
    offs = torch.from_numpy(off.astype(np.int64)).cuda() if offs is None else offs
    wk, wi = oracle(x_bits, off, k, t, largest)
    vals, idx = s.topk_segments(x, offs, k, t, largest, True)
    S = off.size - 1
    assert vals.shape == idx.shape == (S, k) and vals.dtype == x.dtype and idx.dtype == torch.int32
    same(host(vals, t).reshape(S, k), wk, f"{what}, k={k}, largest={largest}: keys")
    same(idx.cpu().numpy().view(np.uint32), wi, f"{what}, k={k}, largest={largest}: indices")
    uv, ui = s.topk_segments(x, offs, k, t, largest, False)
    uk, ui = host(uv, t).reshape(S, k), ui.cpu().numpy().view(np.uint32)
    # padding exactly in columns m .. k-1; the pairs of columns 0 .. m-1 sorted by position equal the oracle's
    same(ui == PAD_IDX, wi == PAD_IDX, f"{what}, k={k}: unsorted padding columns")
    by = np.argsort(ui.astype(np.int64), axis=-1, kind="stable")
    same(np.take_along_axis(ui, by, axis=-1), np.sort(wi.astype(np.int64), axis=-1).astype(np.uint32), f"{what}: unsorted positions")
    wby = np.argsort(wi.astype(np.int64), axis=-1, kind="stable")
    same(np.take_along_axis(uk, by, axis=-1), np.take_along_axis(wk, wby, axis=-1), f"{what}: unsorted keys")
    return vals, idx


def rank_mode_sorter(g, rank_mode, max_n=1 << 16):
    """a sorter whose workspace holds max_n segments' class lists, in the given rank mode"""
    s = g.OneSweepSorter(max_n, 4, 4)
    if rank_mode == 0 and not s.info("atomic_order_ok"):
        s.close()
        pytest.skip("the atomic rank mode failed its self-test on this device")
    s.set_option("rank_mode", rank_mode)
    return s


def edge_lengths(t):
    c = cap(t)
    return [0, 1, 2, 31, 32, 33, 255, 256, 257, 2048, 2049, c - 1, c, c + 1, 50_000, 128_256]


def edge_ks(t):
    return sorted({1, 2, 50, 256, 257, cap(t)})


# ---- 1. every dtype, both directions, both rank modes, the length edges and every k ------------------------------------------
@pytest.mark.parametrize("largest", [False, True])
@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_types_lengths_and_k(g, rank_mode, t, largest):
    rng = np.random.default_rng(list(TYPES).index(t) * 4 + largest * 2 + rank_mode)
    lens = edge_lengths(t)
    lens = lens + list(rng.permutation(lens)) + [1, 0, 0, 7]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    bits = typed_input(rng, int(off[-1]), t)
    x, offs = dev(bits, t), torch.from_numpy(off).cuda()
    with rank_mode_sorter(g, rank_mode) as s:
        for k in edge_ks(t) + [33, 2049]:
            if k <= cap(t):
                check(s, bits, off, k, t, largest, "edge lengths", x, offs)


@pytest.mark.parametrize("t", ["bf16", "f32", "i64"])
def test_k_against_length_on_both_paths(g, t):
    """k < L, k = L and k > L on the warp path (L <= 256) and on the select path"""
    rng = np.random.default_rng(5)
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        for L in (3, 100, 256, 300, 5000):
            for k in (L - 1, L, L + 1, min(cap(t), 4 * L)):
                off = np.arange(0, 9 * L + 1, L, dtype=np.int64)
                bits = typed_input(rng, 9 * L, t)
                check(s, bits, off, k, t, True, f"9 segments of {L}")


# ---- 2. ragged mixes, offsets with gaps, invalid segments ---------------------------------------------------------------------
def ragged(rng, kind, n_target):
    if kind == "uniform 1-8":
        return rng.integers(1, 9, n_target // 4)
    if kind == "uniform 1-64":
        return rng.integers(1, 65, n_target // 32)
    if kind == "uniform 257-4096":
        return rng.integers(257, 4097, max(1, n_target // 2000))
    if kind == "log-uniform 1-2^17":
        return np.exp(rng.uniform(0, np.log(1 << 17), max(1, n_target // 8000))).astype(np.int64)
    # runs of empty segments between short and long ones
    lens = rng.integers(0, 400, n_target // 200)
    lens[rng.random(lens.size) < 0.5] = 0
    return lens


@pytest.mark.parametrize("kind", ["uniform 1-8", "uniform 1-64", "uniform 257-4096", "log-uniform 1-2^17", "empty runs"])
@pytest.mark.parametrize("t", ["bf16", "f32", "u64"])
def test_ragged_mixes(g, t, kind):
    rng = np.random.default_rng(7)
    lens = ragged(rng, kind, 1 << 20)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    bits = typed_input(rng, int(off[-1]), t)
    with g.OneSweepSorter(1 << 20, 4, 4) as s:
        for k in (1, 8, 100, 1000):
            check(s, bits, off, k, t, True, kind)
        check(s, bits, off, 50, t, False, kind)


@pytest.mark.parametrize("t", ["i16", "f32", "f64"])
def test_gaps_start_and_invalid_segments(g, t):
    """offsets that start after 0 and leave gaps (expressed as overlapping and skipping segments), decreasing offsets and
    segments past n: the invalid ones are all padding, and positions outside every segment are never read into a result"""
    rng = np.random.default_rng(9)
    n = 200_000
    bits = typed_input(rng, n, t)
    off = np.array([17, 40, 40, 300, 250, 5000, 5001, 30_000, 29_000, 150_000, n - 3, n, n + 5, n + 1, 7, 7], dtype=np.int64)
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        for k in (1, 5, 300, 4000):
            for largest in (False, True):
                check(s, bits, off, k, t, largest, "gaps and invalid segments")


# ---- 3. ties at the boundary and keys that tie with the padding ---------------------------------------------------------------
@pytest.mark.parametrize("t", ["u16", "i32", "f32", "bf16", "u64", "f64"])
def test_ties_and_all_ones_keys(g, t):
    rng = np.random.default_rng(13)
    c = TYPES[t][1]
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        for L in (40, 256, 3000, 20_000):
            S = 7
            for largest in (False, True):
                pad = pad_key(t, largest)
                segs = {
                    "all equal": np.repeat(random_bits(rng, S, t), L),
                    "few distinct": random_bits(rng, 3, t)[rng.integers(0, 3, S * L)],
                    "keys that tie with the padding": np.where(rng.random(S * L) < 0.3, pad, random_bits(rng, S * L, t)).astype(c),
                }
                # a top bucket of exactly k keys
                k = min(50, L)
                top = c(width(t) - 8)
                r = radix(random_bits(rng, S * L, t), t, largest) & ~(c(0xFF) << top)
                r = r | (c(0x10) << top)
                hot = (np.arange(S)[:, None] * L + np.argsort(rng.random((S, L)), axis=-1)[:, :k]).reshape(-1)
                r[hot] &= ~(c(0xFF) << top)  # the first bucket in the selection order holds exactly k keys
                segs["bucket of exactly k"] = from_radix(~r if largest else r, t)
                off = np.arange(0, S * L + 1, L, dtype=np.int64)
                for name, bits in segs.items():
                    for kk in (1, k, L, L + 3):
                        if kk <= cap(t):
                            check(s, bits.astype(c), off, kk, t, largest, f"{name}, segments of {L}")


# ---- 4. agreement with topk_rows, sort_segments, the block path and the capacity hook ------------------------------------------
@pytest.mark.parametrize("t", ["f16", "u32", "f32", "i64"])
def test_equal_lengths_match_topk_rows_and_sort_segments(g, t):
    rng = np.random.default_rng(17)
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        for rows, L in ((300, 64), (50, 256), (20, 3000), (4, 20_000)):
            bits = typed_input(rng, rows * L, t)
            x = dev(bits, t)
            offs = torch.arange(0, rows * L + 1, L, dtype=torch.int64, device="cuda")
            for k in sorted({1, 8, min(L, 300), min(L, cap(t))}):
                for largest in (False, True):
                    # (unsorted, a select-path row of exactly k keys is written in one pass here, in D + 1 by topk_rows)
                    for srt in (True, False) if k < L or L <= 256 else (True,):
                        sv, si = s.topk_segments(x, offs, k, t, largest, srt)
                        rv, ri = s.topk_rows(x.view(rows, L), k, t, largest, srt)
                        same(host(sv, t), host(rv, t), f"{rows}x{L} k={k} sorted={srt}: keys against topk_rows")
                        same(si.cpu().numpy(), ri.cpu().numpy(), f"{rows}x{L} k={k} sorted={srt}: indices against topk_rows")
                    if L <= cap(t):
                        sv, si = s.topk_segments(x, offs, k, t, largest, True)
                        qv, qi = s.sort_segments(x, offs, t, largest)
                        same(host(sv, t), host(qv, t).reshape(rows, L)[:, :k], f"{rows}x{L} k={k}: keys against sort_segments")
                        same(si.cpu().numpy(), qi.cpu().numpy().reshape(rows, L)[:, :k], f"{rows}x{L}: indices against sort_segments")


@pytest.mark.parametrize("t", ["bf16", "i32", "u64", "f64"])
def test_warp_path_equals_block_path(g, t):
    rng = np.random.default_rng(19)
    lens = rng.integers(0, 257, 3000)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    bits = typed_input(rng, int(off[-1]), t)
    x, offs = dev(bits, t), torch.from_numpy(off).cuda()
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        for k in (1, 2, 50, 256, 300):
            for largest in (False, True):
                got = []
                for block in (0, 1):
                    s.set_option("debug_rows_block", block)
                    got.append(s.topk_segments(x, offs, k, t, largest, True))
                s.set_option("debug_rows_block", 0)
                same(host(got[0][0], t), host(got[1][0], t), f"k={k}: keys")
                same(got[0][1].cpu().numpy(), got[1][1].cpu().numpy(), f"k={k}: indices")
        s.set_option("debug_rows_block", 1)
        check(s, bits, off, 50, t, True, "block path", x, offs)
        s.set_option("debug_rows_block", 0)


@pytest.mark.parametrize("bits_", [32, 64])
def test_capacity_hook_at_c_and_c_plus_1_candidates(g, bits_):
    t = "u32" if bits_ == 32 else "u64"
    rng = np.random.default_rng(23 + bits_)
    C = 300
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        s.set_option("debug_topk_capacity", C)
        for level in (1, 2):
            for cand in (C, C + 1):
                for k in (1, 50, 256):
                    rows = [candidates_row(rng, int(L), k, cand, level, bits_) for L in (3000, 2000, 4000, 3000)]
                    lens = [r.size for r in rows]
                    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
                    check(s, np.concatenate(rows), off, k, t, False, f"{cand} candidates after level {level}")
        s.set_option("debug_topk_capacity", 0)


# ---- 5. sentinels around the outputs, n = 0, no-ops ------------------------------------------------------------------------------
@pytest.mark.parametrize("t", ["bf16", "i32", "f64"])
def test_odd_offsets_and_sentinels(g, t):
    rng = np.random.default_rng(29)
    lib = g.lib
    kt, kb = KEY_TYPE[t], width(t) // 8
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        for lens, k in (([3, 0, 40, 300], 7), ([5000, 1, 256, 0, 257], 300), ([20, 20_000], 2)):
            off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
            n, S = int(off[-1]), len(lens)
            m = S * k
            bits = typed_input(rng, n, t)
            for srt in (1, 0):
                kin = dev(np.concatenate([random_bits(rng, 1, t), bits, random_bits(rng, 2, t)]), t)
                out_bits = random_bits(rng, m + 2 * GUARD + 3, t)
                out = dev(out_bits, t)
                idx = torch.full((m + 2 * GUARD + 5,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
                offs = torch.from_numpy(off).cuda()
                o_in, o_out, o_idx = 1, GUARD + 3, GUARD + 5
                st = lib.osb200_topk_segments(s._h, kin.data_ptr() + o_in * kb, out.data_ptr() + o_out * kb, idx.data_ptr() + o_idx * 4,
                                              n, offs.data_ptr(), S, k, kb, kt, 1, srt, None)
                assert st == OK
                torch.cuda.synchronize()
                got, gi = host(out, t), idx.cpu().numpy().view(np.uint32)
                wk, wi = oracle(bits, off, k, t, True)
                gk, gx = got[o_out:o_out + m].reshape(S, k), gi[o_idx:o_idx + m].reshape(S, k)
                if srt:
                    same(gk, wk, "keys")
                    same(gx, wi, "indices")
                else:
                    same(np.sort(gx.astype(np.int64), axis=-1), np.sort(wi.astype(np.int64), axis=-1), "unsorted indices")
                same(np.concatenate([got[:o_out], got[o_out + m:]]), np.concatenate([out_bits[:o_out], out_bits[o_out + m:]]),
                     "sentinels around the keys")
                assert (gi[:o_idx] == 0x5A5A5A5A).all() and (gi[o_idx + m:] == 0x5A5A5A5A).all(), "sentinels around the indices"


def test_n_zero_pads_and_no_ops_leave_outputs(g):
    lib = g.lib
    with g.OneSweepSorter(1 << 10, 4, 4) as s:
        for t in TYPES:
            kt, kb = KEY_TYPE[t], width(t) // 8
            offs = torch.zeros(6, dtype=torch.int64, device="cuda")
            offs[3] = 4  # [0, 4) passes n = 0: invalid
            for largest in (0, 1):
                for k in (1, 300, cap(t)):
                    out = torch.zeros(5 * k * kb, dtype=torch.uint8, device="cuda")
                    idx = torch.zeros(5 * k, dtype=torch.int32, device="cuda")
                    assert lib.osb200_topk_segments(s._h, None, out.data_ptr(), idx.data_ptr(), 0, offs.data_ptr(), 5, k, kb, kt,
                                                    largest, 1, None) == OK
                    torch.cuda.synchronize()
                    assert (idx == -1).all()
                    keys = out.cpu().numpy().view(TYPES[t][1])
                    assert (keys == pad_key(t, largest)).all(), (t, largest, k)
            # k == 0 and num_segments == 0 touch nothing
            sent = torch.full((64,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
            sk = torch.full((64,), 0x3C, dtype=torch.int64, device="cuda")
            x = torch.ones(100, dtype=torch.int64, device="cuda")
            offs = torch.tensor([0, 50, 100], dtype=torch.int64, device="cuda")
            assert lib.osb200_topk_segments(s._h, x.data_ptr(), sk.data_ptr(), sent.data_ptr(), 100, offs.data_ptr(), 2, 0, kb, kt, 1, 1,
                                            None) == OK
            assert lib.osb200_topk_segments(s._h, x.data_ptr(), sk.data_ptr(), sent.data_ptr(), 100, offs.data_ptr(), 0, 8, kb, kt, 1, 1,
                                            None) == OK
            torch.cuda.synchronize()
            assert (sent == 0x5A5A5A5A).all() and (sk == 0x3C).all()


# ---- 6. argument errors ------------------------------------------------------------------------------------------------------------
def test_argument_errors(g):
    lib = g.lib
    a = torch.zeros(1 << 16, dtype=torch.int64, device="cuda")
    b = torch.zeros(1 << 16, dtype=torch.int64, device="cuda")
    c = torch.zeros(1 << 16, dtype=torch.int32, device="cuda")
    o = torch.tensor([0, 100, 4000, 4096], dtype=torch.int64, device="cuda")
    pa, pb, pc, po = a.data_ptr(), b.data_ptr(), c.data_ptr(), o.data_ptr()

    with g.OneSweepSorter(8, 4, 0) as small, g.OneSweepSorter(1 << 10, 4, 4) as s:
        def call(h=s._h, i=pa, out=pb, x=pc, n=4096, off=po, segs=3, k=64, kb=4, kt=2, largest=1, srt=1):
            return lib.osb200_topk_segments(h, i, out, x, n, off, segs, k, kb, kt, largest, srt, None)

        assert call() == OK
        assert call(h=small._h) == OK
        assert call(kb=8, kt=5, k=8192) == OK
        assert call(kb=2, kt=3, srt=0) == OK
        assert call(h=None) == INVALID_ARG
        assert call(i=None) == INVALID_ARG
        assert call(i=None, n=0) == OK
        assert call(out=None) == INVALID_ARG
        assert call(x=None) == INVALID_ARG
        assert call(off=None) == INVALID_ARG
        for kb, kt in ((4, 3), (4, 6), (8, 2), (2, 4), (2, -1), (3, 0), (16, 0), (0, 0)):
            assert call(kb=kb, kt=kt) == INVALID_ARG, (kb, kt)
        assert call(i=pa + 2) == INVALID_ARG
        assert call(out=pb + 4, kb=8, kt=3) == INVALID_ARG
        assert call(x=pc + 2) == INVALID_ARG
        assert call(off=po + 4) == INVALID_ARG
        assert call(i=pa + 2, out=pb + 6, x=pc + 4, kb=2, kt=0) == OK
        assert call(n=1 << 62) == INVALID_ARG
        assert call(segs=1 << 62, k=1) == INVALID_ARG
        assert call(segs=(1 << 58), k=64) == INVALID_ARG  # num_segments * k * 8 overflows
        # overlaps: input, offsets and both outputs
        assert call(out=pa) == INVALID_ARG
        assert call(out=pa + 4096 * 4 - 4) == INVALID_ARG
        assert call(out=pa + 4096 * 4) == OK
        assert call(x=pb + 3 * 64 * 4 - 4) == INVALID_ARG
        assert call(x=pb + 3 * 64 * 4) == OK
        assert call(off=pa + 8) == INVALID_ARG
        assert call(off=pb + 8) == INVALID_ARG
        assert call(off=pc + 8) == INVALID_ARG
        # k and num_segments
        assert call(k=16384) == OK
        assert call(k=16385) == SIZE
        assert call(k=16384, kb=2, kt=0) == OK
        assert call(k=16385, kb=2, kt=0) == SIZE
        assert call(k=8193, kb=8, kt=3) == SIZE
        assert call(k=5000) == OK  # larger than every segment
        assert call(h=small._h, segs=9, off=pa, i=pb, out=pc + 1024, x=pc + 40000, k=1) == SIZE  # more segments than max_n
        assert call(segs=0, i=None, out=None, x=None, off=None) == OK
        assert call(k=0, i=None, out=None, x=None, off=None) == OK
        torch.cuda.synchronize()


def test_python_errors_module_level_and_side_stream(g):
    x = torch.randn(10_000, device="cuda")
    offs = torch.tensor([0, 10, 5000, 10_000], dtype=torch.int64, device="cuda")
    with pytest.raises(TypeError):
        g.topk_segments(torch.zeros(8, dtype=torch.int8, device="cuda"), offs, 2)
    with pytest.raises(TypeError):
        g.topk_segments(torch.zeros(8), offs.cpu(), 2)
    with pytest.raises(TypeError):
        g.topk_segments(x.view(100, 100), offs, 2)
    with pytest.raises(TypeError):
        g.topk_segments(x, offs.int(), 2)
    with pytest.raises(TypeError):
        g.topk_segments(x, offs.cpu(), 2)
    with pytest.raises(ValueError):
        g.topk_segments(x, offs, -1)
    with pytest.raises(g.OneSweepError):
        g.topk_segments(x, offs, 16385)
    for t, (dt, _, _, _) in TYPES.items():
        rng = np.random.default_rng(3)
        bits = typed_input(rng, 10_000, t)
        vals, idx = g.topk_segments(dev(bits, t), offs, 20, largest=False)
        wk, wi = oracle(bits, offs.cpu().numpy(), 20, t, False)
        same(host(vals, t).reshape(3, 20), wk, f"{t} module level")
        same(idx.cpu().numpy().view(np.uint32), wi, f"{t} module level indices")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        vals, idx = g.topk_segments(x, offs, 8, stream=side)
    side.synchronize()
    assert torch.equal(vals[1], torch.topk(x[10:5000], 8).values)
    with g.OneSweepSorter(2, 4, 4) as s:
        with pytest.raises(ValueError):
            s.topk_segments(x, offs, -3, "f32")


def test_graph_capture_and_replay(g):
    rng = np.random.default_rng(31)
    lens = rng.integers(0, 3000, 400)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = int(off[-1])
    with g.OneSweepSorter(1 << 12, 4, 4) as s:
        x = torch.zeros(n, dtype=torch.float32, device="cuda")
        offs = torch.from_numpy(off).cuda()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for k in (8, 500):
                s.topk_segments(x, offs, k, "f32", True, True)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = [s.topk_segments(x, offs, k, "f32", True, True) for k in (8, 500)]
        for replay in range(3):
            bits = typed_input(rng, n, "f32")
            x.copy_(dev(bits, "f32"))
            graph.replay()
            torch.cuda.synchronize()
            for k, (v, i) in zip((8, 500), outs):
                wk, wi = oracle(bits, off, k, "f32", True)
                same(host(v, "f32").reshape(-1, k), wk, f"replay {replay} k={k}: keys")
                same(i.cpu().numpy().view(np.uint32), wi, f"replay {replay} k={k}: indices")
        del graph


def test_dense_composite_on_2pow26_keys(g):
    """float32 randn * 3 in log-uniform segments: values equal the dense torch composite's (pad with -inf, topk, mask)"""
    rng = np.random.default_rng(37)
    lens = np.exp(rng.uniform(0, np.log(1 << 17), 3000)).astype(np.int64)
    lens = lens[np.cumsum(lens) <= 1 << 26]
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).cuda()
    n, S = int(off[-1]), lens.size
    x = torch.randn(n, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda") * 3
    k = 50
    vals, idx = g.topk_segments(x, off, k)
    L = torch.from_numpy(lens).cuda()
    maxlen = int(L.max())
    dense = torch.full((S, maxlen), float("-inf"), device="cuda")
    seg = torch.repeat_interleave(torch.arange(S, device="cuda"), L)
    pos = torch.arange(n, device="cuda") - off[:-1][seg]
    dense[seg, pos] = x
    ref = torch.topk(dense, min(k, maxlen), dim=-1).values
    m = torch.clamp(L, max=k)
    mask = torch.arange(k, device="cuda")[None, :] < m[:, None]
    assert torch.equal(vals[mask], ref[:, :k][mask])
    assert (idx[~mask] == -1).all()
    assert torch.isnan(vals[~mask]).all()
    gi = idx.long()
    assert torch.equal(x[(off[:-1, None] + gi)[mask]], vals[mask])


# ---- 7. past 2^31 and 2^32 --------------------------------------------------------------------------------------------------------
def test_u16_segments_past_2pow32(g):
    """uint16 keys, n just past 2^32: warp-class and block-class segments straddle 2^31 and 2^32 (two sets of offsets over the
    same keys).  Background keys are below 1000; each segment holds 20 planted maxima 60000 + j at known positions, and its
    first 200 other keys tie at 5000, so the boundary of k = 64 falls among equal keys"""
    n = (1 << 32) + 30_100
    b31, b32 = 1 << 31, 1 << 32
    sets = {
        "block segments straddle": [b31 - 5000, b31 + 5000, b31 + 5100, b32 - 20_000, b32 + 10_000, b32 + 10_100, n],
        "warp segments straddle": [b31 - 100, b31 + 100, b32 - 100, b32 + 100, n],
    }
    require(g, "u16 segments past 2^32", 1 << 10, 4, 0, 2 * n + (1 << 20), 0)
    x = torch.empty(n, dtype=torch.int16, device="cuda")
    k = 64
    try:
        for name, ends in sets.items():
            x.random_(0, 1000)
            rng = np.random.default_rng(len(ends))
            bounds = [0] + ends
            want = {}
            for s_ in range(len(ends)):
                lo, hi = bounds[s_], bounds[s_ + 1]
                L = hi - lo
                p = np.unique(rng.integers(0, L, 40))[:20]
                tie = np.setdiff1d(np.arange(min(L, 200)), p)
                x[lo + torch.from_numpy(tie).cuda()] = 5000
                x[lo + torch.from_numpy(p).cuda()] = torch.arange(60000 - 65536, 60000 - 65536 + p.size, dtype=torch.int16,
                                                                  device="cuda")
                want[s_] = (np.concatenate([60000 + np.arange(p.size)[::-1], np.full(tie.size, 5000)])[:k],
                            np.concatenate([p[::-1], tie])[:k])
            off = torch.tensor(bounds, dtype=torch.int64, device="cuda")
            with g.OneSweepSorter(1 << 10, 4, 0) as s:
                for srt in (True, False):
                    vals, idx = s.topk_segments(x.view(torch.uint16), off, k, "u16", True, srt)
                    torch.cuda.synchronize()
                    v = vals.view(torch.int16).cpu().numpy().view(np.uint16).astype(np.int64)
                    i = idx.cpu().numpy().view(np.uint32).astype(np.int64)
                    for s_, (wv, wi) in want.items():
                        gv, gi = v[s_], i[s_]
                        if not srt:
                            o = np.lexsort((gi, -gv))
                            gv, gi = gv[o], gi[o]
                        same(gv, wv, f"{name}: segment {s_} values, sorted={srt}")
                        same(gi, wi, f"{name}: segment {s_} positions, sorted={srt}")
                    del vals, idx
    finally:
        del x
        release()


def test_u16_segment_of_2pow32_minus_1_and_2pow32_keys_past_2pow32(g):
    """a segment of 2^32 - 1 keys is valid, its planted maxima sit past 2^31 and at 2^32 - 2; one of 2^32 keys is all padding"""
    L = (1 << 32) - 1
    n = 1 << 32
    require(g, "u16 segment of 2^32 - 1 keys", 4, 4, 0, 2 * n + (1 << 20), 0)
    x = torch.zeros(n, dtype=torch.int16, device="cuda")
    try:
        x[(1 << 31) + 5] = 900
        x[(1 << 31) + 6] = 900
        x[L - 1] = 1000
        x[L] = 2000  # not in the first segment
        off = torch.tensor([0, L, 0, n], dtype=torch.int64, device="cuda")  # [0, 2^32 - 1), [2^32 - 1, 0): invalid, [0, 2^32)
        with g.OneSweepSorter(4, 4, 0) as s:
            vals, idx = s.topk_segments(x.view(torch.uint16), off, 4, "u16", True, True)
            torch.cuda.synchronize()
            v, i = vals.view(torch.int16).cpu().numpy().view(np.uint16), idx.cpu().numpy().view(np.uint32)
        same(v[0], np.array([1000, 900, 900, 0], dtype=np.uint16), "values of the 2^32 - 1 segment")
        same(i[0], np.array([L - 1, (1 << 31) + 5, (1 << 31) + 6, 0], dtype=np.uint32), "positions of the 2^32 - 1 segment")
        same(i[1:], np.full((3 - 1, 4), PAD_IDX, dtype=np.uint32), "the invalid and the 2^32-key segment are padding")
        same(v[1:], np.zeros((2, 4), dtype=np.uint16), "padding keys of largest u16")
    finally:
        del x
        release()


def test_f32_outputs_past_2pow31(g):
    """about 2^18 block-class segments at k = 8,192: outputs of more than 2^31 elements, mostly padding"""
    S, k, L = (1 << 18) + 5, 8192, 300
    n = S * L
    require(g, "f32 outputs past 2^31", S, 4, 0, 4 * n + 8 * S * k + (1 << 20), 0)
    assert S * k > 1 << 31
    x = torch.rand(n, device="cuda")
    try:
        top = torch.arange(S, device="cuda") * L + (torch.arange(S, device="cuda") * 7) % L
        x[top] = 2.0
        off = torch.arange(0, n + 1, L, dtype=torch.int64, device="cuda")
        with g.OneSweepSorter(S, 4, 0) as s:
            for srt in (True, False):
                vals, idx = s.topk_segments(x, off, k, "f32", True, srt)
                torch.cuda.synchronize()
                assert (idx[:, L:] == -1).all() and torch.isnan(vals[:, L:]).all()
                if srt:
                    assert (vals[:, 0] == 2.0).all() and torch.equal(idx[:, 0].long(), top - off[:-1])
                    assert (vals[:, 1:L] < 1.0).all() and (vals[:, 1:L - 1] >= vals[:, 2:L]).all()
                else:
                    assert torch.equal(torch.sort(idx[:, :L].long(), dim=1).values,
                                       torch.arange(L, device="cuda").expand(S, L))
                for r in (S - 1, S // 2):
                    seg = x[r * L:(r + 1) * L]
                    want = torch.sort(seg, descending=True, stable=True).values
                    got = torch.sort(vals[r, :L], descending=True).values
                    assert torch.equal(got, want)
                del vals, idx
    finally:
        del x
        release()


def test_segment_ids_past_2pow31(g):
    """2^31 + 4,099 segments whose non-empty ones have ids past 2^31, uint16 keys and k = 1"""
    S = (1 << 31) + 4099
    require(g, f"{S} segments", S, 4, 0, 8 * (S + 1) + 6 * S + (1 << 20), 0)
    rng = np.random.default_rng(41)
    lens = rng.integers(1, 600, 3000)
    n = int(lens.sum())
    first = S - lens.size
    off = torch.zeros(S + 1, dtype=torch.int64, device="cuda")
    try:
        off[first + 1:] = torch.from_numpy(np.cumsum(lens)).cuda()
        bits = random_bits(rng, n, "u16")
        x = dev(bits, "u16")
        with g.OneSweepSorter(S, 4, 0) as s:
            vals, idx = s.topk_segments(x, off, 1, "u16", True, True)
            torch.cuda.synchronize()
        assert (idx[:first] == -1).all() and (vals[:first].view(torch.int16) == 0).all()
        tail_off = np.concatenate([[0], np.cumsum(lens)])
        wk, wi = oracle(bits, tail_off, 1, "u16", True)
        same(host(vals[first:], "u16"), wk.reshape(-1), "keys of the segments past 2^31")
        same(idx[first:].cpu().numpy().view(np.uint32).reshape(-1), wi.reshape(-1), "indices of the segments past 2^31")
    finally:
        del off
        release()
