"""osb200_sort_rows, OneSweepSorter.sort_rows and gpusorting_b200.sort_rows: every row of a batch sorted stable along its
last dimension, for 16-, 32- and 64-bit keys, with int32 indices within the row.

Every case compares element by element with numpy's stable argsort of each row's radix image (radix below: unsigned keys as
they are, signed keys with the sign bit flipped, floats in the total order of their bits; descending is the complement, so
ties keep their input order in both directions).  Keys and indices are compared bit for bit.  The row lengths sit on both
sides of every boundary: the warp path's buckets (32, 64, 128, 256 keys), the block path's two geometries (2,048 and 16,384
keys, 8,192 for 64-bit keys) and the size limit.  Rows of at most 256 keys are also compared with the block path through the
"debug_rows_block" hook.  -m gpu"""
import ctypes

import numpy as np
import pytest
import torch

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
LENS = [1, 2, 31, 32, 33, 64, 65, 128, 129, 255, 256, 257, 2048, 2049, 8192, 8193, 16384]
GUARD = 37


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def width(t):
    return np.dtype(TYPES[t][1]).itemsize * 8


def cap(t):
    return 8192 if width(t) == 64 else 16384


def radix(bits, t, descending=False):
    """unsigned key whose ascending order is the requested order of the values with bit patterns `bits`"""
    u = bits.astype(TYPES[t][1])
    w = width(t)
    sign = u.dtype.type(1 << (w - 1))
    if TYPES[t][3] == "i":
        u = u ^ sign
    elif TYPES[t][3] == "f":
        u = np.where(u >> u.dtype.type(w - 1) == 1, ~u, u | sign).astype(u.dtype)
    return ~u if descending else u


def specials(t):
    """+-0, subnormals, +-max, +-inf and NaNs of both signs with different payloads"""
    pos = {
        "f16": [0, 1, 0x03FF, 0x0400, 0x7BFF, 0x7C00, 0x7C01, 0x7E00, 0x7FFF],
        "bf16": [0, 1, 0x007F, 0x0080, 0x7F7F, 0x7F80, 0x7F81, 0x7FC0, 0x7FFF],
        "f32": [0, 1, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0x7F800000, 0x7F800001, 0x7FC00000, 0x7FFFFFFF],
        "f64": [0, 1, 0x000FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF, 0x7FF0000000000000, 0x7FF0000000000001,
                0x7FF8000000000000, 0x7FFFFFFFFFFFFFFF],
    }[t]
    sign = 1 << (width(t) - 1)
    return np.array(pos + [sign | p for p in pos], dtype=TYPES[t][1])


def random_bits(rng, n, t):
    c = TYPES[t][1]
    return rng.integers(0, np.iinfo(c).max, n, dtype=c, endpoint=True)


def typed_input(rng, n, t):
    """half drawn from 16 values (ties, so stability shows in the indices), half uniform; floats contain the specials"""
    bits = random_bits(rng, n, t)
    pool = random_bits(rng, 16, t)
    if TYPES[t][3] == "f":
        sp = specials(t)
        bits[rng.integers(0, n, min(n, sp.size))] = sp[: min(n, sp.size)]
        pool = np.concatenate([pool, sp])
    tied = rng.random(n) < 0.5
    bits[tied] = pool[rng.integers(0, pool.size, int(tied.sum()))]
    return bits


def dev(bits, t):
    return torch.from_numpy(bits.view(TYPES[t][2]).copy()).cuda().view(TYPES[t][0])


def host(x, t):
    return x.view(TYPES[t][0]).view(getattr(torch, np.dtype(TYPES[t][2]).name)).cpu().numpy().view(TYPES[t][1])


def oracle(bits2d, t, descending):
    order = np.argsort(radix(bits2d, t, descending), axis=-1, kind="stable")
    return np.take_along_axis(bits2d, order, axis=-1), order.astype(np.uint32)


def same(got, want, what):
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    assert got.size == want.size, f"{what}: {got.size} elements, want {want.size}"
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} of {want.size} elements differ, the first at {bad[0] if bad.size else -1}"


def check(s, bits2d, t, descending, what):
    """sort_rows with and without indices, out of place (input untouched) and in place, against the oracle"""
    want_k, want_i = oracle(bits2d, t, descending)
    x = dev(bits2d, t)
    vals, idx = s.sort_rows(x, t, descending)
    assert vals.shape == x.shape == idx.shape and vals.dtype == x.dtype and idx.dtype == torch.int32
    same(host(x, t), bits2d, f"{what}: input modified")
    same(host(vals, t), want_k, f"{what}: keys")
    same(idx.cpu().numpy().view(np.uint32), want_i, f"{what}: indices")
    only = s.sort_rows(x, t, descending, return_indices=False)
    same(host(only, t), want_k, f"{what}: keys only")
    y = x.clone()
    out, idx2 = s.sort_rows(y, t, descending, inplace=True)
    assert out.data_ptr() == y.data_ptr()
    same(host(y, t), want_k, f"{what}: in place")
    same(idx2.cpu().numpy().view(np.uint32), want_i, f"{what}: in place indices")
    y = x.clone()
    s.sort_rows(y, t, descending, return_indices=False, inplace=True)
    same(host(y, t), want_k, f"{what}: in place keys only")


def rank_mode_sorter(g, rank_mode):
    s = g.OneSweepSorter(1, 4, 4)
    if rank_mode == 0 and not s.info("atomic_order_ok"):
        s.close()
        pytest.skip("the atomic rank mode failed its self-test on this device")
    s.set_option("rank_mode", rank_mode)
    return s


# ---- 1. every dtype, both orders, both rank modes, row lengths around every boundary --------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_types_orders_and_lengths(g, rank_mode, t, descending):
    rng = np.random.default_rng(list(TYPES).index(t) * 4 + descending * 2 + rank_mode)
    with rank_mode_sorter(g, rank_mode) as s:
        for row_len in [L for L in LENS if L <= cap(t)]:
            rows = 3 if row_len >= 2048 else 37
            check(s, typed_input(rng, rows * row_len, t).reshape(rows, row_len), t, descending, f"{rows} rows of {row_len}")


@pytest.mark.parametrize("t", ["bf16", "f32", "u64"])
def test_row_counts(g, t):
    """one row, an odd count, and far more rows than there are resident warps (each warp sorts many rows)"""
    rng = np.random.default_rng(11)
    with g.OneSweepSorter(1, 4, 4) as s:
        for rows, row_len in ((1, 32), (1, 200), (1, 4000), (1001, 96), (200_000, 32), (20_001, 255), (3001, 300)):
            check(s, typed_input(rng, rows * row_len, t).reshape(rows, row_len), t, True, f"{rows} rows of {row_len}")


# ---- 2. stability, float specials, per-row pass skipping ------------------------------------------------------------------
@pytest.mark.parametrize("t", ["i16", "f32", "i64"])
def test_duplicate_heavy_rows(g, t):
    rng = np.random.default_rng(13)
    with g.OneSweepSorter(1, 4, 4) as s:
        for row_len in (32, 100, 256, 1000, 4096):
            rows = 65
            bits = random_bits(rng, 3, t)[rng.integers(0, 3, rows * row_len)].reshape(rows, row_len)
            for descending in (False, True):
                check(s, bits, t, descending, f"3 distinct values, rows of {row_len}, descending={descending}")


@pytest.mark.parametrize("t", ["f16", "bf16", "f32", "f64"])
def test_float_specials(g, t):
    rng = np.random.default_rng(17)
    sp = specials(t)
    with g.OneSweepSorter(1, 4, 4) as s:
        for row_len in (sp.size, 64, 300, 5000):
            rows = 9
            bits = sp[rng.integers(0, sp.size, rows * row_len)].reshape(rows, row_len)
            for descending in (False, True):
                check(s, bits, t, descending, f"specials, rows of {row_len}, descending={descending}")


@pytest.mark.parametrize("t", ["u64", "i64", "f64", "u32", "u16"])
def test_constant_high_digits(g, t):
    """rows whose radix images differ only in their low byte (the warp path skips every other pass), rows whose keys are all
    equal (every pass skipped) and rows mixing both; both paths"""
    rng = np.random.default_rng(19)
    c = TYPES[t][1]
    with g.OneSweepSorter(1, 4, 4) as s:
        for block in (0, 1):
            s.set_option("debug_rows_block", block)
            for row_len in (32, 77, 256):
                rows = 501
                base = random_bits(rng, rows, t)[:, None] & ~c(0xFF)
                low = rng.integers(0, 256, (rows, row_len)).astype(c)
                low[::3] = low[::3, :1]  # every third row: all keys equal
                r = base | low
                # the bit patterns whose ascending radix image is r (the descending image ~r has constant high bytes too)
                bits = r
                if TYPES[t][3] == "i":
                    bits = r ^ c(1 << (width(t) - 1))
                elif TYPES[t][3] == "f":
                    bits = np.where(r >> c(width(t) - 1) == 1, r ^ c(1 << (width(t) - 1)), ~r).astype(c)
                for descending in (False, True):
                    check(s, bits, t, descending, f"low byte only, rows of {row_len}, block={block}, descending={descending}")


# ---- 3. the warp path against the block path ------------------------------------------------------------------------------
@pytest.mark.parametrize("t", list(TYPES))
def test_warp_path_equals_block_path(g, t):
    rng = np.random.default_rng(23)
    with g.OneSweepSorter(1, 4, 4) as s:
        for row_len in (2, 17, 32, 33, 64, 65, 128, 129, 200, 256):
            x = dev(typed_input(rng, 513 * row_len, t).reshape(513, row_len), t)
            for descending in (False, True):
                s.set_option("debug_rows_block", 0)
                wk, wi = s.sort_rows(x, t, descending)
                s.set_option("debug_rows_block", 1)
                bk, bi = s.sort_rows(x, t, descending)
                what = f"rows of {row_len}, descending={descending}"
                same(host(wk, t), host(bk, t), f"{what}: keys")
                assert torch.equal(wi, bi), f"{what}: indices"


# ---- 4. buffers at odd element offsets, sentinels around the outputs ------------------------------------------------------
@pytest.mark.parametrize("t", ["bf16", "i32", "f64"])
def test_odd_offsets_and_sentinels(g, t):
    rng = np.random.default_rng(29)
    lib = g.lib
    kt = KEY_TYPE[t]
    kb = width(t) // 8
    with g.OneSweepSorter(1, 4, 4) as s:
        for rows, row_len in ((33, 31), (17, 200), (5, 3000)):
            n = rows * row_len
            bits = typed_input(rng, n, t).reshape(rows, row_len)
            want_k, want_i = oracle(bits, t, False)
            kin = dev(np.concatenate([random_bits(rng, 1, t), bits.reshape(-1), random_bits(rng, 2, t)]), t)
            out_bits = random_bits(rng, n + 2 * GUARD + 3, t)
            out = dev(out_bits, t)
            idx = torch.full((n + 2 * GUARD + 5,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
            o_in, o_out, o_idx = 1, GUARD + 3, GUARD + 5
            st = lib.osb200_sort_rows(s._h, kin.data_ptr() + o_in * kb, out.data_ptr() + o_out * kb,
                                      idx.data_ptr() + o_idx * 4, rows, row_len, kb, kt, 0, None)
            assert st == OK
            torch.cuda.synchronize()
            got = host(out, t)
            same(got[o_out:o_out + n], want_k, f"{rows}x{row_len}: keys")
            same(np.concatenate([got[:o_out], got[o_out + n:]]), np.concatenate([out_bits[:o_out], out_bits[o_out + n:]]),
                 f"{rows}x{row_len}: sentinels around the keys")
            gi = idx.cpu().numpy().view(np.uint32)
            same(gi[o_idx:o_idx + n], want_i, f"{rows}x{row_len}: indices")
            assert (gi[:o_idx] == 0x5A5A5A5A).all() and (gi[o_idx + n:] == 0x5A5A5A5A).all(), "sentinels around the indices"


# ---- 5. graph capture ----------------------------------------------------------------------------------------------------
def test_graph_capture_and_replay(g):
    rng = np.random.default_rng(31)
    shapes = {"f32": (4001, 64), "bf16": (300, 1000), "i64": (700, 129)}
    with g.OneSweepSorter(1, 4, 4) as s:
        bufs = {t: torch.zeros(shape, dtype=TYPES[t][0], device="cuda") for t, shape in shapes.items()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside the capture
            for t, b in bufs.items():
                s.sort_rows(b, t, True)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        outs = {}
        with torch.cuda.graph(graph):
            for t, b in bufs.items():
                outs[t] = s.sort_rows(b, t, True)
        for replay in range(3):
            data = {t: typed_input(rng, shape[0] * shape[1], t).reshape(shape) for t, shape in shapes.items()}
            for t, b in bufs.items():
                b.copy_(dev(data[t], t))
            graph.replay()
            torch.cuda.synchronize()
            for t in shapes:
                want_k, want_i = oracle(data[t], t, True)
                same(host(outs[t][0], t), want_k, f"replay {replay} {t}: keys")
                same(outs[t][1].cpu().numpy().view(np.uint32), want_i, f"replay {replay} {t}: indices")
        del graph


# ---- 6. the Python layer -------------------------------------------------------------------------------------------------
def test_module_level_sort_rows(g):
    rng = np.random.default_rng(37)
    for t, (dt, _, _, _) in TYPES.items():
        for shape in ((100,), (3, 5, 60), (2, 0, 7), (4, 0)):
            n = int(np.prod(shape))
            bits = typed_input(rng, n, t) if n else np.zeros(0, dtype=TYPES[t][1])
            x = dev(bits, t).reshape(shape)
            for descending in (False, True):
                vals, idx = g.sort_rows(x, descending)
                assert vals.shape == idx.shape == x.shape and vals.dtype == dt and idx.dtype == torch.int32
                if n:
                    want_k, want_i = oracle(bits.reshape(shape), t, descending)
                    same(host(vals, t), want_k, f"{t} {shape}")
                    same(idx.cpu().numpy().view(np.uint32), want_i, f"{t} {shape} indices")
                only = g.sort_rows(x, descending, return_indices=False)
                assert isinstance(only, torch.Tensor) and only.shape == x.shape
    side = torch.cuda.Stream()
    x = torch.randn(64, 256, device="cuda")
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        vals, idx = g.sort_rows(x, stream=side)
    side.synchronize()
    assert torch.equal(vals, torch.sort(x, dim=-1, stable=True).values)
    with pytest.raises(TypeError):
        g.sort_rows(torch.zeros(4, 4, dtype=torch.int8, device="cuda"))
    with pytest.raises(TypeError):
        g.sort_rows(torch.zeros(4, 4, device="cuda").t())  # not contiguous
    with pytest.raises(TypeError):
        g.sort_rows(torch.zeros(4, 4))  # not on the GPU
    with pytest.raises(g.OneSweepError):
        g.sort_rows(torch.zeros(2, 16385, device="cuda"))
    with pytest.raises(g.OneSweepError):
        g.sort_rows(torch.zeros(2, 8193, dtype=torch.int64, device="cuda"))


# ---- 7. argument errors through ctypes -----------------------------------------------------------------------------------
def test_argument_errors(g):
    lib = g.lib
    n = 4096
    a = torch.zeros(4 * n, dtype=torch.int64, device="cuda")
    b = torch.zeros(4 * n, dtype=torch.int64, device="cuda")
    c = torch.zeros(8 * n, dtype=torch.int32, device="cuda")  # 16,384 indices and more
    pa, pb, pc = a.data_ptr(), b.data_ptr(), c.data_ptr()

    def call(h, i=pa, o=pb, x=pc, rows=16, row_len=256, kb=4, kt=2, desc=0):
        return lib.osb200_sort_rows(h, i, o, x, rows, row_len, kb, kt, desc, None)

    with g.OneSweepSorter(1, 8, 0) as wide, g.OneSweepSorter(1, 4, 4) as s:
        for h in (wide._h, s._h):  # any handle will do
            assert call(h) == OK
            assert call(h, kb=8, kt=5) == OK
            assert call(h, kb=2, kt=3) == OK
        h = s._h
        assert call(None) == INVALID_ARG
        assert call(h, i=None) == INVALID_ARG
        assert call(h, o=None) == INVALID_ARG
        assert call(h, x=None) == OK  # keys only
        for kb, kt in ((4, 3), (4, 6), (8, 2), (2, 4), (2, -1), (3, 0), (16, 0), (0, 0)):
            assert call(h, kb=kb, kt=kt) == INVALID_ARG, (kb, kt)
        assert call(h, i=pa + 2, kb=4, kt=2) == INVALID_ARG  # misaligned keys
        assert call(h, o=pb + 4, kb=8, kt=3) == INVALID_ARG
        assert call(h, x=pc + 2) == INVALID_ARG  # misaligned indices
        assert call(h, i=pa + 2, o=pb + 6, x=pc + 4, kb=2, kt=0) == OK  # natural alignment is enough
        assert call(h, rows=1 << 62, row_len=8) == INVALID_ARG  # num_rows * row_len overflows
        assert call(h, rows=(1 << 62) + 1, row_len=4) == INVALID_ARG
        # overlaps: in == out is in place; any other overlap is refused
        assert call(h, o=pa) == OK
        assert call(h, o=pa + 4) == INVALID_ARG
        assert call(h, x=pa + 64) == INVALID_ARG
        assert call(h, x=pb + 16) == INVALID_ARG
        assert call(h, o=pa, x=pa + 16 * 256 * 4) == OK  # behind the keys
        # sizes
        assert call(h, rows=1, row_len=16384) == OK
        assert call(h, rows=1, row_len=16385) == SIZE
        assert call(h, rows=1, row_len=16384, kb=2, kt=0) == OK
        assert call(h, rows=1, row_len=16385, kb=2, kt=0) == SIZE
        assert call(h, rows=1, row_len=8192, kb=8, kt=3) == OK
        assert call(h, rows=1, row_len=8193, kb=8, kt=3) == SIZE
        # no-ops, whatever the pointers
        assert call(h, i=None, o=None, x=None, rows=0) == OK
        assert call(h, i=None, o=None, x=None, row_len=0) == OK
        torch.cuda.synchronize()
        # row_len == 1: the keys are copied and the indices are zero
        x = torch.arange(100, dtype=torch.float32, device="cuda").neg()
        out = torch.full((100,), 7.0, device="cuda")
        idx = torch.full((100,), 9, dtype=torch.int32, device="cuda")
        assert lib.osb200_sort_rows(h, x.data_ptr(), out.data_ptr(), idx.data_ptr(), 100, 1, 4, 2, 1, None) == OK
        torch.cuda.synchronize()
        assert torch.equal(out, x) and not idx.any()


# ---- 8. cross-check against torch.sort at 2^26 keys -----------------------------------------------------------------------
def no_nan_no_signed_zero(t, n, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if t == "i64":
        return torch.randint(-(1 << 62), 1 << 62, (n,), generator=gen, device="cuda", dtype=torch.int64)
    x = torch.randn(n, generator=gen, device="cuda").to(TYPES[t][0])
    return torch.where(x == 0, torch.ones_like(x), x)  # torch orders -0.0 == +0.0, the bit order does not


@pytest.mark.parametrize("row_len", [64, 4096])
@pytest.mark.parametrize("t", ["f32", "bf16", "i64"])
def test_against_torch_sort(g, t, row_len):
    n = 1 << 26
    x = no_nan_no_signed_zero(t, n, 41).view(-1, row_len)
    for descending in (False, True):
        ref, order = torch.sort(x, dim=-1, descending=descending, stable=True)
        vals, idx = g.sort_rows(x, descending)
        assert torch.equal(vals, ref), f"keys, descending={descending}"
        assert torch.equal(idx.long(), order), f"indices, descending={descending}"
        del ref, order, vals, idx
