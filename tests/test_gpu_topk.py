"""osb200_topk_rows, OneSweepSorter.topk_rows and gpusorting_b200.topk: the k smallest or largest keys of every row and their
int32 positions, for 16-, 32- and 64-bit keys and rows of any length.

The oracle is numpy's stable argsort of each row's radix image (unsigned keys as they are, signed keys with the sign bit
flipped, floats in the total order of their bits; largest is the complement, so ties keep their input order), cut to k.
sorted=True must equal it bit for bit, keys and indices, and equal sort_rows(x, descending=largest) cut to k wherever the
row sort takes the row; sorted=False must hold the same (key, position) pairs.  Row lengths sit on both sides of the warp
path's limit (256), the block geometries and the shared-memory capacity C (16,384 keys, 8,192 for 64-bit keys), and go far
beyond it.  The "debug_topk_capacity" hook lowers C so that short rows take the passes that read global memory, with inputs
built by tests/topk_plan.py to hold exactly C and C + 1 candidates after the first and the second level.
The test whose name contains "past_2pow" needs about 9 GB: -k "not past_2pow" leaves it out of a quick run.  -m gpu"""
import numpy as np
import pytest
import torch

from tests.topk_plan import candidates_row, plan

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
# name -> (torch dtype, numpy container, signed view for the transfer, kind)
TYPES = {
    "u16": (torch.uint16, np.uint16, np.int16, "u"), "i16": (torch.int16, np.uint16, np.int16, "i"),
    "f16": (torch.float16, np.uint16, np.int16, "f"), "bf16": (torch.bfloat16, np.uint16, np.int16, "f"),
    "u32": (torch.uint32, np.uint32, np.int32, "u"), "i32": (torch.int32, np.uint32, np.int32, "i"),
    "f32": (torch.float32, np.uint32, np.int32, "f"),
    "u64": (torch.uint64, np.uint64, np.int64, "u"), "i64": (torch.int64, np.uint64, np.int64, "i"),
    "f64": (torch.float64, np.uint64, np.int64, "f"),
}
KEY_TYPE = {"u16": 0, "i16": 1, "f16": 2, "bf16": 3, "u32": 0, "i32": 1, "f32": 2, "u64": 3, "i64": 4, "f64": 5}
GUARD = 37


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def width(t):
    return np.dtype(TYPES[t][1]).itemsize * 8


def cap(t):
    return 8192 if width(t) == 64 else 16384


def lengths(t):
    c = cap(t)
    return [1, 2, 31, 32, 33, 255, 256, 257, 2048, 2049, c - 1, c, c + 1, 50_000, 128_256, (1 << 20) + 3]


def ks(t, row_len):
    return sorted({k for k in (1, 2, 50, 256, 257, row_len, cap(t)) if k <= row_len and k <= cap(t)})


def radix(bits, t, largest=False):
    """unsigned key whose ascending order is the requested order of the values with bit patterns `bits`"""
    u = bits.astype(TYPES[t][1])
    w = width(t)
    sign = u.dtype.type(1 << (w - 1))
    if TYPES[t][3] == "i":
        u = u ^ sign
    elif TYPES[t][3] == "f":
        u = np.where(u >> u.dtype.type(w - 1) == 1, ~u, u | sign).astype(u.dtype)
    return ~u if largest else u


def from_radix(r, t):
    """the bit patterns whose ascending radix image is r"""
    c = TYPES[t][1]
    r = r.astype(c)
    if TYPES[t][3] == "i":
        return r ^ c(1 << (width(t) - 1))
    if TYPES[t][3] == "f":
        return np.where(r >> c(width(t) - 1) == 1, r ^ c(1 << (width(t) - 1)), ~r).astype(c)
    return r


def random_bits(rng, n, t):
    c = TYPES[t][1]
    return rng.integers(0, np.iinfo(c).max, n, dtype=c, endpoint=True)


def dev(bits, t):
    return torch.from_numpy(bits.view(TYPES[t][2]).copy()).cuda().view(TYPES[t][0])


def host(x, t):
    return x.contiguous().view(TYPES[t][0]).view(getattr(torch, np.dtype(TYPES[t][2]).name)).cpu().numpy().view(TYPES[t][1])


def order_of(bits2d, t, largest):
    return np.argsort(radix(bits2d, t, largest), axis=-1, kind="stable")


def same(got, want, what):
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    assert got.size == want.size, f"{what}: {got.size} elements, want {want.size}"
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} of {want.size} elements differ, the first at {bad[0] if bad.size else -1}"


def check(s, x, bits2d, t, largest, k, what, order=None, row_sort=True):
    """topk_rows sorted and unsorted against the oracle (the stable order `order`, computed here if not given), and against
    sort_rows cut to k where the row fits it"""
    if order is None:
        order = order_of(bits2d, t, largest)
    want_i = order[:, :k]
    want_k = np.take_along_axis(bits2d, want_i, axis=-1)
    vals, idx = s.topk_rows(x, k, t, largest, True)
    assert vals.shape == idx.shape == (bits2d.shape[0], k) and vals.dtype == x.dtype and idx.dtype == torch.int32
    gi = idx.cpu().numpy().view(np.uint32).astype(np.int64)
    same(host(vals, t), want_k, f"{what}, k={k}: keys")
    same(gi, want_i, f"{what}, k={k}: indices")
    if row_sort and bits2d.shape[1] <= cap(t):
        rk, ri = s.sort_rows(x, t, largest)
        same(host(vals, t), host(rk[:, :k], t), f"{what}, k={k}: keys against sort_rows")
        same(gi, ri[:, :k].cpu().numpy().view(np.uint32), f"{what}, k={k}: indices against sort_rows")
    uv, ui = s.topk_rows(x, k, t, largest, False)
    ui = ui.cpu().numpy().view(np.uint32).astype(np.int64)
    by_pos = np.argsort(ui, axis=-1)
    same(np.take_along_axis(ui, by_pos, axis=-1), np.sort(want_i, axis=-1), f"{what}, k={k}: unsorted positions")
    same(np.take_along_axis(host(uv, t).reshape(ui.shape), by_pos, axis=-1),
         np.take_along_axis(bits2d, np.sort(want_i, axis=-1), axis=-1), f"{what}, k={k}: unsorted keys")


def rank_mode_sorter(g, rank_mode):
    s = g.OneSweepSorter(1, 4, 4)
    if rank_mode == 0 and not s.info("atomic_order_ok"):
        s.close()
        pytest.skip("the atomic rank mode failed its self-test on this device")
    s.set_option("rank_mode", rank_mode)
    return s


def typed_input(rng, n, t):
    """half drawn from 16 values (ties at the boundary), half uniform"""
    bits = random_bits(rng, n, t)
    pool = random_bits(rng, 16, t)
    tied = rng.random(n) < 0.5
    bits[tied] = pool[rng.integers(0, pool.size, int(tied.sum()))]
    return bits


# ---- 1. every dtype, both directions, both rank modes, every row length and k ---------------------------------------------
@pytest.mark.parametrize("largest", [False, True])
@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_types_lengths_and_k(g, rank_mode, t, largest):
    rng = np.random.default_rng(list(TYPES).index(t) * 4 + largest * 2 + rank_mode)
    with rank_mode_sorter(g, rank_mode) as s:
        for row_len in lengths(t):
            rows = max(1, min(37, 2_500_000 // row_len))
            bits = typed_input(rng, rows * row_len, t).reshape(rows, row_len)
            x = dev(bits, t)
            order = order_of(bits, t, largest)
            for k in ks(t, row_len):
                check(s, x, bits, t, largest, k, f"{rows} rows of {row_len}", order)


@pytest.mark.parametrize("t", ["bf16", "f32", "u64"])
def test_row_counts(g, t):
    """one row, and far more rows than resident warps or CTAs (every CTA's grid-stride loop wraps many times)"""
    rng = np.random.default_rng(11)
    with g.OneSweepSorter(1, 4, 4) as s:
        for rows, row_len, k in ((1, 40, 8), (1, 5000, 50), (200_000, 64, 2), (20_001, 256, 8), (3001, 300, 64),
                                 (1000, 4096, 64), (300, 20000, 100)):
            bits = typed_input(rng, rows * row_len, t).reshape(rows, row_len)
            check(s, dev(bits, t), bits, t, True, k, f"{rows} rows of {row_len}")


# ---- 2. inputs that steer the radix select ----------------------------------------------------------------------------------
def structured_rows(rng, t, rows, row_len, k):
    """{name: bits} of the inputs that change the level plan"""
    c = TYPES[t][1]
    out = {}
    if t in ("f32", "bf16"):
        logits = (torch.from_numpy(rng.standard_normal((rows, row_len)).astype(np.float32)) * 3).to(TYPES[t][0])
        out["randn*3 logits"] = host(logits, t).reshape(rows, row_len)
    out["uniform"] = random_bits(rng, rows * row_len, t).reshape(rows, row_len)
    out["all equal"] = np.repeat(random_bits(rng, rows, t)[:, None], row_len, axis=1)
    out["few distinct"] = random_bits(rng, 3, t)[rng.integers(0, 3, (rows, row_len))]
    srt = np.sort(radix(random_bits(rng, rows * row_len, t).reshape(rows, row_len), t), axis=-1)
    out["sorted"] = from_radix(srt, t)
    out["reversed"] = from_radix(srt[:, ::-1], t)
    # k equal maxima at the end of the row, the rest strictly smaller
    r = radix(random_bits(rng, rows * row_len, t).reshape(rows, row_len), t) >> c(1)
    r[:, -k:] = c(np.iinfo(c).max)
    out["k maxima at the end"] = from_radix(r, t)
    # the top bucket holds exactly k keys: the select stops after one level
    top = c(width(t) - 8)
    r = radix(random_bits(rng, rows * row_len, t).reshape(rows, row_len), t) & ~(c(0xFF) << top)
    r |= c(0x10) << top
    hot = np.argsort(rng.random((rows, row_len)), axis=-1)[:, :k]
    np.put_along_axis(r, hot, np.take_along_axis(r, hot, axis=-1) | (c(0xF0) << top), axis=-1)
    out["bucket of exactly k"] = from_radix(r, t)
    if width(t) == 64:
        out["small values"] = rng.integers(0, 1000, (rows, row_len)).astype(c)
    return out


@pytest.mark.parametrize("t", ["bf16", "f32", "i16", "u32", "i64", "f64"])
def test_structured_inputs(g, t):
    rng = np.random.default_rng(13)
    with g.OneSweepSorter(1, 4, 4) as s:
        for rows, row_len, k in ((9, 200, 8), (9, 3000, 50), (5, 20000, 256), (3, 128_256, 1024)):
            for name, bits in structured_rows(rng, t, rows, row_len, k).items():
                x = dev(np.ascontiguousarray(bits), t)
                for largest in (True, False):
                    check(s, x, bits, t, largest, k, f"{name}, {rows} rows of {row_len}, largest={largest}")


@pytest.mark.parametrize("t", ["f16", "bf16", "f32", "i32", "i64", "f64"])
def test_values_match_torch_topk(g, t):
    """values agree with torch.topk on inputs without NaN and -0.0 (torch orders those differently)"""
    gen = torch.Generator(device="cuda").manual_seed(17)
    for rows, row_len, k in ((4096, 64, 8), (64, 4096, 64), (8, 151_936, 50), (2, 128_256, 1024)):
        if TYPES[t][3] == "i":
            x = torch.randint(-1000, 1000, (rows, row_len), generator=gen, device="cuda", dtype=TYPES[t][0])
        else:
            x = (torch.randn(rows, row_len, generator=gen, device="cuda") * 3).to(TYPES[t][0])
            x = torch.where(x == 0, torch.ones_like(x), x)
        for largest in (True, False):
            vals, idx = g.topk(x, k, largest)
            ref = torch.topk(x, k, dim=-1, largest=largest).values
            assert torch.equal(vals, ref), f"{rows}x{row_len}, k={k}, largest={largest}"
            assert torch.equal(torch.gather(x, -1, idx.long()), vals)


# ---- 3. the shared-memory capacity hook and the warp path against the block path -------------------------------------------
@pytest.mark.parametrize("bits", [32, 64])
def test_capacity_hook_at_n_and_n_plus_1_candidates(g, bits):
    t = "u32" if bits == 32 else "u64"
    rng = np.random.default_rng(19 + bits)
    n = 300
    with g.OneSweepSorter(1, 4, 4) as s:
        s.set_option("debug_topk_capacity", n)
        for level in (1, 2):
            for cand in (n, n + 1):
                for k in (1, 50, 256):
                    rows = np.stack([candidates_row(rng, 3000, k, cand, level, bits) for _ in range(7)])
                    for r in rows:
                        p = plan(r, k, bits, n)
                        assert p[level]["candidates"] == cand and p[level]["compact"] == (cand <= n)
                    check(s, dev(rows, t), rows, t, False, k, f"{cand} candidates after level {level}", row_sort=False)
        # random rows of a few thousand keys: the candidates reach the lowered capacity at various levels
        for row_len in (1000, 3000, 7000):
            r = typed_input(rng, 9 * row_len, t).reshape(9, row_len)
            for k in (1, 50, 257):
                check(s, dev(r, t), r, t, True, k, f"capacity {n}, rows of {row_len}")
        s.set_option("debug_topk_capacity", 0)


@pytest.mark.parametrize("t", list(TYPES))
def test_warp_path_equals_block_path(g, t):
    rng = np.random.default_rng(23)
    with g.OneSweepSorter(1, 4, 4) as s:
        for row_len in (2, 17, 32, 33, 64, 65, 128, 129, 200, 256):
            bits = typed_input(rng, 513 * row_len, t).reshape(513, row_len)
            x = dev(bits, t)
            for k in sorted({1, 2, min(50, row_len), row_len}):
                for largest in (False, True):
                    got = []
                    for block in (0, 1):
                        s.set_option("debug_rows_block", block)
                        got.append(s.topk_rows(x, k, t, largest, True))
                    s.set_option("debug_rows_block", 0)
                    same(host(got[0][0], t), host(got[1][0], t), f"{row_len}, k={k}: keys")
                    same(got[0][1].cpu().numpy(), got[1][1].cpu().numpy(), f"{row_len}, k={k}: indices")
            s.set_option("debug_rows_block", 1)
            check(s, x, bits, t, True, min(50, row_len), f"block path, rows of {row_len}")
            s.set_option("debug_rows_block", 0)


# ---- 4. buffers at odd element offsets, sentinels around the outputs --------------------------------------------------------
@pytest.mark.parametrize("t", ["bf16", "i32", "f64"])
def test_odd_offsets_and_sentinels(g, t):
    rng = np.random.default_rng(29)
    lib = g.lib
    kt = KEY_TYPE[t]
    kb = width(t) // 8
    with g.OneSweepSorter(1, 4, 4) as s:
        for rows, row_len, k in ((33, 31, 5), (17, 200, 200), (5, 3000, 300), (3, 20000, 64)):
            for sort in (1, 0):
                n, m = rows * row_len, rows * k
                bits = typed_input(rng, n, t).reshape(rows, row_len)
                want_i = order_of(bits, t, True)[:, :k]
                want_k = np.take_along_axis(bits, want_i, axis=-1)
                kin = dev(np.concatenate([random_bits(rng, 1, t), bits.reshape(-1), random_bits(rng, 2, t)]), t)
                out_bits = random_bits(rng, m + 2 * GUARD + 3, t)
                out = dev(out_bits, t)
                idx = torch.full((m + 2 * GUARD + 5,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
                o_in, o_out, o_idx = 1, GUARD + 3, GUARD + 5
                st = lib.osb200_topk_rows(s._h, kin.data_ptr() + o_in * kb, out.data_ptr() + o_out * kb,
                                          idx.data_ptr() + o_idx * 4, rows, row_len, k, kb, kt, 1, sort, None)
                assert st == OK
                torch.cuda.synchronize()
                got = host(out, t)
                gi = idx.cpu().numpy().view(np.uint32)
                what = f"{rows}x{row_len}, k={k}, sorted={sort}"
                gk, gx = got[o_out:o_out + m].reshape(rows, k), gi[o_idx:o_idx + m].reshape(rows, k).astype(np.int64)
                if not sort:
                    by_pos = np.argsort(gx, axis=-1)
                    gk, gx = np.take_along_axis(gk, by_pos, axis=-1), np.take_along_axis(gx, by_pos, axis=-1)
                    want_i = np.sort(want_i, axis=-1)
                    want_k = np.take_along_axis(bits, want_i, axis=-1)
                same(gk, want_k, f"{what}: keys")
                same(gx, want_i, f"{what}: indices")
                same(np.concatenate([got[:o_out], got[o_out + m:]]), np.concatenate([out_bits[:o_out], out_bits[o_out + m:]]),
                     f"{what}: sentinels around the keys")
                assert (gi[:o_idx] == 0x5A5A5A5A).all() and (gi[o_idx + m:] == 0x5A5A5A5A).all(), "sentinels around the indices"


# ---- 5. graph capture and a side stream --------------------------------------------------------------------------------------
def test_graph_capture_and_replay(g):
    rng = np.random.default_rng(31)
    shapes = {"f32": ((4001, 64), 8), "bf16": ((300, 5000), 50), "i64": ((20, 20000), 300)}
    with g.OneSweepSorter(1, 4, 4) as s:
        bufs = {t: torch.zeros(shape, dtype=TYPES[t][0], device="cuda") for t, (shape, _) in shapes.items()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside the capture
            for t, b in bufs.items():
                s.topk_rows(b, shapes[t][1], t, True, True)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        outs = {}
        with torch.cuda.graph(graph):
            for t, b in bufs.items():
                outs[t] = s.topk_rows(b, shapes[t][1], t, True, True)
        for replay in range(3):
            data = {t: typed_input(rng, shape[0] * shape[1], t).reshape(shape) for t, (shape, _) in shapes.items()}
            for t, b in bufs.items():
                b.copy_(dev(data[t], t))
            graph.replay()
            torch.cuda.synchronize()
            for t, (_, k) in shapes.items():
                want_i = order_of(data[t], t, True)[:, :k]
                same(host(outs[t][0], t), np.take_along_axis(data[t], want_i, axis=-1), f"replay {replay} {t}: keys")
                same(outs[t][1].cpu().numpy().view(np.uint32), want_i, f"replay {replay} {t}: indices")
        del graph


def test_module_level_topk_and_python_errors(g):
    rng = np.random.default_rng(37)
    for t, (dt, _, _, _) in TYPES.items():
        for shape, k in (((100,), 7), ((3, 5, 600), 20), ((2, 0, 7), 3), ((4, 300), 0)):
            n = int(np.prod(shape))
            bits = typed_input(rng, n, t) if n else np.zeros(0, dtype=TYPES[t][1])
            x = dev(bits, t).reshape(shape)
            for largest in (False, True):
                vals, idx = g.topk(x, k, largest)
                assert vals.shape == idx.shape == shape[:-1] + (k,) and vals.dtype == dt and idx.dtype == torch.int32
                if n and k:
                    b2 = bits.reshape(-1, shape[-1])
                    want_i = order_of(b2, t, largest)[:, :k]
                    same(host(vals, t), np.take_along_axis(b2, want_i, axis=-1), f"{t} {shape}")
                    same(idx.cpu().numpy().view(np.uint32), want_i, f"{t} {shape} indices")
    side = torch.cuda.Stream()
    x = torch.randn(64, 5000, device="cuda")
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        vals, idx = g.topk(x, 40, stream=side)
    side.synchronize()
    assert torch.equal(vals, torch.topk(x, 40, dim=-1).values)
    with pytest.raises(TypeError):
        g.topk(torch.zeros(4, 4, dtype=torch.int8, device="cuda"), 2)
    with pytest.raises(TypeError):
        g.topk(torch.zeros(4, 4, device="cuda").t(), 2)  # not contiguous
    with pytest.raises(TypeError):
        g.topk(torch.zeros(4, 4), 2)  # not on the GPU
    with g.OneSweepSorter(1, 4, 4) as s:
        with pytest.raises(TypeError):
            s.topk_rows(torch.zeros(4, 4, dtype=torch.int8, device="cuda"), 2, "u32")
        with pytest.raises(TypeError):
            s.topk_rows(torch.zeros(4, 4), 2, "f32")
    with pytest.raises(g.OneSweepError):
        g.topk(torch.zeros(2, 20000, device="cuda"), 16385)
    with pytest.raises(g.OneSweepError):
        g.topk(torch.zeros(2, 10000, dtype=torch.int64, device="cuda"), 8193)
    with pytest.raises(g.OneSweepError):
        g.topk(torch.zeros(2, 10, device="cuda"), 11)


# ---- 6. argument errors through ctypes ---------------------------------------------------------------------------------------
def test_argument_errors(g):
    lib = g.lib
    n = 4096
    a = torch.zeros(8 * n, dtype=torch.int64, device="cuda")
    b = torch.zeros(4 * n, dtype=torch.int64, device="cuda")
    c = torch.zeros(8 * n, dtype=torch.int32, device="cuda")
    pa, pb, pc = a.data_ptr(), b.data_ptr(), c.data_ptr()

    def call(h, i=pa, o=pb, x=pc, rows=16, row_len=1024, k=64, kb=4, kt=2, largest=1, srt=1):
        return lib.osb200_topk_rows(h, i, o, x, rows, row_len, k, kb, kt, largest, srt, None)

    with g.OneSweepSorter(1, 8, 0) as wide, g.OneSweepSorter(1, 4, 4) as s:
        for h in (wide._h, s._h):  # any handle will do
            assert call(h) == OK
            assert call(h, kb=8, kt=5) == OK
            assert call(h, kb=2, kt=3, srt=0) == OK
        h = s._h
        assert call(None) == INVALID_ARG
        assert call(h, i=None) == INVALID_ARG
        assert call(h, o=None) == INVALID_ARG
        assert call(h, x=None) == INVALID_ARG  # the indices are required
        for kb, kt in ((4, 3), (4, 6), (8, 2), (2, 4), (2, -1), (3, 0), (16, 0), (0, 0)):
            assert call(h, kb=kb, kt=kt) == INVALID_ARG, (kb, kt)
        assert call(h, i=pa + 2, kb=4, kt=2) == INVALID_ARG  # misaligned keys
        assert call(h, o=pb + 4, kb=8, kt=3) == INVALID_ARG
        assert call(h, x=pc + 2) == INVALID_ARG  # misaligned indices
        assert call(h, i=pa + 2, o=pb + 6, x=pc + 4, kb=2, kt=0) == OK  # natural alignment is enough
        assert call(h, rows=1 << 62, row_len=8, k=1) == INVALID_ARG  # num_rows * row_len overflows
        assert call(h, rows=(1 << 62) + 1, row_len=4, k=1) == INVALID_ARG
        # no overlap at all: the outputs have another shape than the input
        assert call(h, o=pa) == INVALID_ARG
        assert call(h, o=pa + 16 * 1024 * 4 - 4) == INVALID_ARG
        assert call(h, o=pa + 16 * 1024 * 4, x=pc) == OK  # behind the keys
        assert call(h, x=pa + 64) == INVALID_ARG
        assert call(h, x=pb + 16) == INVALID_ARG
        assert call(h, x=pb + 16 * 64 * 4) == OK  # behind the values
        # k
        assert call(h, row_len=100, k=101) == INVALID_ARG
        assert call(h, rows=1, row_len=20000, k=16384) == OK
        assert call(h, rows=1, row_len=20000, k=16385) == SIZE
        assert call(h, rows=1, row_len=20000, k=16384, kb=2, kt=0) == OK
        assert call(h, rows=1, row_len=20000, k=16385, kb=2, kt=0) == SIZE
        assert call(h, rows=1, row_len=10000, k=8192, kb=8, kt=3) == OK
        assert call(h, rows=1, row_len=10000, k=8193, kb=8, kt=3) == SIZE
        # no-ops, whatever the pointers
        for kw in ({"rows": 0}, {"row_len": 0}, {"k": 0}):
            assert call(h, i=None, o=None, x=None, **kw) == OK, kw
        torch.cuda.synchronize()


# ---- 7. one row past 2^31 keys -----------------------------------------------------------------------------------------------
def test_bf16_row_past_2pow31(g):
    """one bfloat16 row of 2^31 + 4,099 keys whose k largest lie past position 2^31 (they read as negative int32 positions)
    and every other key is strictly smaller: the answer is known without a sort"""
    n, k = (1 << 31) + 4099, 64
    x = torch.rand(n, dtype=torch.bfloat16, device="cuda")  # [0, 1)
    planted = 2.0 + torch.arange(k, device="cuda", dtype=torch.float32) / 64  # distinct bfloat16 values in [2, 3)
    pos = (1 << 31) + 17 + torch.randperm(4000, device="cuda")[:k].sort().values
    x[pos] = planted.to(torch.bfloat16)[torch.randperm(k, device="cuda")]
    vals, idx = g.topk(x.view(1, n), k)
    want_v, order = torch.sort(x[pos].float(), descending=True, stable=True)
    assert torch.equal(vals[0].float(), want_v)
    assert torch.equal(idx[0].long() & 0xFFFFFFFF, pos[order])
    assert (idx[0] < 0).all()
    del x
    torch.cuda.empty_cache()
