"""osb200_sort_long_rows, OneSweepSorter.sort_long_rows and gpusorting_b200.sort_long_rows: every row of a batch sorted stable
along its last dimension for rows of any length, 16-, 32- and 64-bit keys, with int32 indices within the row.

Rows above the row sort's limit (C = 16,384 keys, 8,192 for 64-bit keys) take the long path: an LSD radix sort per row over
tiles of T = 8,192 keys that never straddle rows.  Every case compares element by element, keys and indices bit for bit,
with numpy's stable argsort of each row's radix image (the oracle of tests/test_gpu_rows.py).  The lengths sit around C and
around multiples of T; the inputs hold ties, float specials, constant digit places, sorted and reversed rows, outliers and
rows structured by T.  The "debug_long_rows" hook sends short rows down the long path, which must then equal
osb200_sort_rows bit for bit.  -m gpu; the past_2pow tests need up to about 34 GiB of free device memory."""
import gc

import numpy as np
import pytest
import torch

from tests import bigcheck, structured
from tests.test_gpu_rows import KEY_TYPE, LENS, TYPES, dev, host, oracle, radix, random_bits, same, specials, typed_input, width

pytestmark = pytest.mark.gpu

OK, INVALID_ARG, SIZE = 0, -1, -2
T = 8192  # the long path's tile
GUARD = 41


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
    """a sorter whose workspace takes rows of t: (4, 4) for 16- and 32-bit keys, (8, 4) for 64-bit keys"""
    s = g.OneSweepSorter(max_n, 8 if width(t) == 64 else 4, 4 if indices else 0)
    if rank_mode is not None:
        if rank_mode == 0 and not s.info("atomic_order_ok"):
            s.close()
            pytest.skip("the atomic rank mode failed its self-test on this device")
        s.set_option("rank_mode", rank_mode)
    return s


def executed(bits, t):
    """the passes the plan runs: the digit places on which the keys of the call are not all equal"""
    img = radix(bits.reshape(-1), t)
    return sum(int(np.unique((img >> img.dtype.type(8 * p)) & img.dtype.type(255)).size > 1) for p in range(width(t) // 8))


def check(s, bits2d, t, descending, what, plan=True):
    """sort_long_rows with and without indices, out of place (input untouched) and in place, against the oracle; plan: the
    executed pass count of the handle's last plan"""
    want_k, want_i = oracle(bits2d, t, descending)
    x = dev(bits2d, t)
    vals, idx = s.sort_long_rows(x, t, descending)
    assert vals.shape == x.shape == idx.shape and vals.dtype == x.dtype and idx.dtype == torch.int32
    same(host(x, t), bits2d, f"{what}: input modified")
    same(host(vals, t), want_k, f"{what}: keys")
    same(idx.cpu().numpy().view(np.uint32), want_i, f"{what}: indices")
    if plan:
        assert s.info("last_executed_passes") == executed(bits2d, t), f"{what}: executed passes"
    only = s.sort_long_rows(x, t, descending, return_indices=False)
    same(host(only, t), want_k, f"{what}: keys only")
    y = x.clone()
    out, idx2 = s.sort_long_rows(y, t, descending, inplace=True)
    assert out.data_ptr() == y.data_ptr()
    same(host(y, t), want_k, f"{what}: in place")
    same(idx2.cpu().numpy().view(np.uint32), want_i, f"{what}: in place indices")
    y = x.clone()
    s.sort_long_rows(y, t, descending, return_indices=False, inplace=True)
    same(host(y, t), want_k, f"{what}: in place keys only")


def long_lens(t):
    c = cap(t)
    return [c + 1, 2 * c, 3 * T - 1, 3 * T, 3 * T + 1, 5 * T - 1, 5 * T + 1]


# ---- 1. every dtype, both orders, both rank modes, lengths around C and multiples of T, 1, 2 and 7 rows ---------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_types_orders_and_lengths(g, rank_mode, t, descending):
    rng = np.random.default_rng(list(TYPES).index(t) * 4 + descending * 2 + rank_mode)
    lens = long_lens(t)
    with sorter(g, t, 7 * max(lens), rank_mode) as s:
        for i, row_len in enumerate(lens):
            rows = (1, 2, 7)[i % 3]
            check(s, typed_input(rng, rows * row_len, t).reshape(rows, row_len), t, descending, f"{rows} rows of {row_len}")


# ---- 2. the vocabularies of the README's workloads, a prime near 10^5, 2^20 + 3, more rows than resident CTAs -------------
@pytest.mark.parametrize("t", ["f32", "bf16", "i64", "u16"])
def test_vocabulary_lengths(g, t):
    rng = np.random.default_rng(5 + list(TYPES).index(t))
    with sorter(g, t, 300 * 32000) as s:
        for rows, row_len in ((3, 32000), (2, 128256), (2, 151936), (3, 99991), (1, (1 << 20) + 3), (300, 32000)):
            bits = typed_input(rng, rows * row_len, t).reshape(rows, row_len)
            for descending in (False, True):
                check(s, bits, t, descending, f"{rows} rows of {row_len}")


# ---- 3. float specials, all-equal rows, small int64 values, sorted / reversed / one-outlier rows -------------------------
@pytest.mark.parametrize("t", ["f16", "bf16", "f32", "f64"])
def test_float_specials(g, t):
    rng = np.random.default_rng(11)
    row_len = cap(t) + 5
    sp = specials(t)
    bits = sp[rng.integers(0, sp.size, 3 * row_len)].reshape(3, row_len)
    with sorter(g, t, bits.size) as s:
        for descending in (False, True):
            check(s, bits, t, descending, "specials")


@pytest.mark.parametrize("t", list(TYPES))
def test_all_equal_rows_skip_every_place(g, t):
    rng = np.random.default_rng(13)
    row_len = 2 * T + 3
    bits = np.full((4, row_len), random_bits(rng, 1, t)[0], dtype=TYPES[t][1])
    with sorter(g, t, bits.size) as s:
        check(s, bits, t, False, "all equal")
        assert s.info("last_executed_passes") == 0


@pytest.mark.parametrize("hi", [1 << 8, 1 << 16, 1 << 20, 1 << 24])
def test_int64_small_values(g, hi):
    """values below 2^8 .. 2^24: the upper places are skipped, leaving 1, 2, 3 or 4 executed passes (odd ones copy home)"""
    rng = np.random.default_rng(17)
    bits = rng.integers(0, hi, (3, 3 * T + 11)).astype(np.uint64)
    bits[0, 0] = 0
    bits[0, 1] = hi - 1
    with sorter(g, "i64", bits.size) as s:
        for descending in (False, True):
            check(s, bits, "i64", descending, f"below {hi}")


@pytest.mark.parametrize("t", ["u32", "f32", "bf16", "i64"])
def test_sorted_reversed_and_outlier_rows(g, t):
    rng = np.random.default_rng(19)
    row_len = 4 * T + 100
    base = np.sort(typed_input(rng, 3 * row_len, t).reshape(3, row_len), axis=-1)
    order = np.argsort(radix(base, t), axis=-1, kind="stable")
    srt = np.take_along_axis(base, order, axis=-1)
    out = np.full((3, row_len), srt[0, 0], dtype=srt.dtype)
    out[:, row_len // 3] = srt[0, -1]
    with sorter(g, t, 3 * row_len) as s:
        for bits, what in ((srt, "sorted"), (srt[:, ::-1].copy(), "reversed"), (out, "one outlier")):
            for descending in (False, True):
                check(s, bits, t, descending, what)


# ---- 4. rows structured by the long path's tile size ----------------------------------------------------------------------
STRUCTURED = [
    ("runs", lambda n, lay, p, seed: structured.runs(n, T, lay, p, seed, T // 2 + 3, "random")),
    ("runs_asc", lambda n, lay, p, seed: structured.runs(n, T, lay, p, seed, 33, "asc")),
    ("tile_blocks", lambda n, lay, p, seed: structured.tile_blocks(n, T, lay, p, seed)),
    ("outlier_above", lambda n, lay, p, seed: structured.outlier(n, T, lay, p, seed, n // 2 + 7, True)),
    ("outlier_below", lambda n, lay, p, seed: structured.outlier(n, T, lay, p, seed, n - 1, False)),
    ("tile_tie", lambda n, lay, p, seed: structured.tile_tie(n, T, lay, p, seed)),
]


@pytest.mark.parametrize("name,gen", STRUCTURED, ids=[s[0] for s in STRUCTURED])
@pytest.mark.parametrize("key", ["u32", "f32", "i64"])
def test_structured_by_tile(g, key, name, gen):
    """rows of 4 T keys (whole tiles), so every generator's tiles are the long path's: digit runs, single-digit tiles, lone
    outliers and tied digits inside a row and across its tile borders.  The structure is in one place p, the only one the
    plan executes."""
    w = width(key)
    lay = structured.layout(w)
    rows, row_len = 3, 4 * T
    with sorter(g, key, rows * row_len) as s:
        for p in (0, w // 8 - 1):
            image, plan = gen(rows * row_len, lay, p, 100 + p)
            bits = structured.to_bits(image, w, TYPES[key][3]).numpy().view(TYPES[key][1]).reshape(rows, row_len)
            check(s, bits, key, False, f"{name} in place {p}", plan=False)
            x = dev(bits, key)
            s.sort_long_rows(x, key)
            assert s.info("last_executed_passes") == plan.executed == 1
            assert s.info("last_skip_mask") == plan.skip


# ---- 5. the test hook: short rows on the long path equal the row sort ------------------------------------------------------
@pytest.mark.parametrize("t", ["u16", "bf16", "i32", "f32", "u64", "f64"])
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_debug_long_rows_equals_sort_rows(g, rank_mode, t):
    rng = np.random.default_rng(23 + rank_mode)
    with sorter(g, t, 1 << 20, rank_mode) as s:
        for row_len in [L for L in LENS if 2 <= L <= cap(t)]:
            rows = 3 if row_len >= 2048 else 37
            bits = typed_input(rng, rows * row_len, t).reshape(rows, row_len)
            for descending in (False, True):
                x = dev(bits, t)
                s.set_option("debug_long_rows", 0)
                k0, i0 = s.sort_rows(x, t, descending)
                s.set_option("debug_long_rows", 1)
                k1, i1 = s.sort_long_rows(x, t, descending)
                assert s.info("last_executed_passes") == executed(bits, t)
                same(host(k1, t), host(k0, t), f"{rows}x{row_len}: keys")
                same(i1.cpu().numpy(), i0.cpu().numpy(), f"{rows}x{row_len}: indices")


# ---- 6. buffers at element offsets inside guarded allocations ---------------------------------------------------------------
@pytest.mark.parametrize("t", ["u16", "f32", "f64"])
def test_odd_offsets_and_sentinels(g, t):
    rng = np.random.default_rng(29)
    kt, kb = KEY_TYPE[t], width(t) // 8
    with sorter(g, t, 1 << 18) as s:
        for rows, row_len in ((1, cap(t) + 1), (3, 3 * T + 5), (2, 5 * T - 1)):
            n = rows * row_len
            bits = typed_input(rng, n, t).reshape(rows, row_len)
            want_k, want_i = oracle(bits, t, False)
            for o_in in (1, 3):
                kin = dev(np.concatenate([random_bits(rng, o_in, t), bits.reshape(-1), random_bits(rng, 2, t)]), t)
                out_bits = random_bits(rng, n + 2 * GUARD + 3, t)
                out = dev(out_bits, t)
                idx = torch.full((n + 2 * GUARD + 5,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
                o_out, o_idx = GUARD + o_in, GUARD + 5
                st = g.lib.osb200_sort_long_rows(s._h, kin.data_ptr() + o_in * kb, out.data_ptr() + o_out * kb,
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


# ---- 7. against torch.sort on the workload shapes ----------------------------------------------------------------------------
@pytest.mark.parametrize("shape,dtype", [((1024, 128256), torch.float32), ((256, 151936), torch.bfloat16),
                                         ((16, 1 << 20), torch.int64)], ids=["f32", "bf16", "i64"])
def test_against_torch_sort(g, shape, dtype):
    """on a sorter of its own, closed at the end: the workload shapes would otherwise stay allocated in the module calls'
    cached sorters for the rest of the session, memory that later tests of 2^30 keys need"""
    key = {torch.float32: "f32", torch.bfloat16: "bf16", torch.int64: "i64"}[dtype]
    gen = torch.Generator(device="cuda").manual_seed(37)
    if dtype.is_floating_point:
        x = (torch.randn(shape, generator=gen, device="cuda") * 3).to(dtype)
        x[x == 0] = 1  # no -0.0 (torch orders it equal to +0.0)
    else:
        x = torch.randint(-(1 << 40), 1 << 40, shape, generator=gen, device="cuda", dtype=dtype)
    with sorter(g, key, x.numel()) as s:
        for descending in (False, True):
            v, i = s.sort_long_rows(x, key, descending)
            wv, wi = torch.sort(x, dim=-1, descending=descending, stable=True)
            assert torch.equal(v.view(torch.int16 if dtype == torch.bfloat16 else v.dtype),
                               wv.view(torch.int16 if dtype == torch.bfloat16 else wv.dtype)), f"values, descending={descending}"
            assert torch.equal(i.long(), wi), f"indices, descending={descending}"
            del v, i, wv, wi


# ---- 8. argument errors through ctypes ---------------------------------------------------------------------------------------
def test_argument_errors(g):
    lib = g.lib
    rows, row_len = 4, 20000
    n = rows * row_len
    a = torch.zeros(n + 64, dtype=torch.float32, device="cuda")
    b = torch.zeros(n + 64, dtype=torch.float32, device="cuda")
    c = torch.zeros(n + 64, dtype=torch.int32, device="cuda")
    w = torch.zeros(n + 64, dtype=torch.float64, device="cuda")
    w2 = torch.zeros(n + 64, dtype=torch.float64, device="cuda")
    pa, pb, pc, pw = a.data_ptr(), b.data_ptr(), c.data_ptr(), w.data_ptr()

    def call(h, i=pa, o=pb, x=pc, rows=rows, row_len=row_len, kb=4, kt=2, desc=0):
        return lib.osb200_sort_long_rows(h, i, o, x, rows, row_len, kb, kt, desc, None)

    h44, h40, h84, h80 = (g.OneSweepSorter(n, 4, 4), g.OneSweepSorter(n, 4, 0), g.OneSweepSorter(n, 8, 4),
                          g.OneSweepSorter(n, 8, 0))
    small = g.OneSweepSorter(n - 1, 4, 4)
    try:
        assert call(None) == INVALID_ARG
        assert call(h44._h, i=None) == INVALID_ARG and call(h44._h, o=None) == INVALID_ARG
        assert call(h44._h, i=pa + 2) == INVALID_ARG and call(h44._h, o=pb + 1) == INVALID_ARG
        assert call(h44._h, x=pc + 2) == INVALID_ARG
        assert call(h44._h, kt=5) == INVALID_ARG and call(h44._h, kb=3) == INVALID_ARG
        assert call(h44._h, o=pa + 4) == INVALID_ARG, "out overlapping in (not equal)"
        assert call(h44._h, x=pa + 4 * 100) == INVALID_ARG, "indices overlapping the keys"
        assert call(h44._h, o=pa) == OK, "in place"
        assert call(h44._h, x=None) == OK
        assert call(small._h) == SIZE, "n > max_n"
        assert call(h44._h, i=pw, o=w2.data_ptr(), rows=rows // 2, kb=8, kt=5) == INVALID_ARG, "a 4-byte handle, 8-byte keys"
        assert call(h84._h, i=pw, o=pw + 8 * 8, rows=1, row_len=8193, kb=8, kt=5, x=None) == INVALID_ARG, "overlap"
        assert call(h40._h) == INVALID_ARG, "indices on a handle without payloads"
        assert call(h40._h, x=None) == OK and call(h80._h, x=None) == OK and call(h84._h) == OK
        # rows of at most C keys take osb200_sort_rows' launch on any handle
        tiny = g.OneSweepSorter(1, 4, 0)
        try:
            assert call(tiny._h, rows=3, row_len=16384) == OK
            assert call(tiny._h, rows=3, row_len=16385) == INVALID_ARG
            assert call(tiny._h, rows=3, row_len=16385, x=None) == SIZE
        finally:
            tiny.close()
        assert call(h44._h, rows=0) == OK and call(h44._h, row_len=0) == OK
        assert call(h84._h, i=pw, o=w2.data_ptr(), rows=rows // 2, kb=8, kt=5) == OK
        torch.cuda.synchronize()
    finally:
        for s in (h44, h40, h84, h80, small):
            s.close()


def test_module_function_grows_its_sorter(g):
    from gpusorting_b200 import onesweep

    rng = np.random.default_rng(41)
    for t, shape in (("f32", (2, 20000)), ("f32", (5, 40000)), ("i64", (3, 9000)), ("bf16", (4, 3000))):
        bits = typed_input(rng, shape[0] * shape[1], t).reshape(shape)
        x = dev(bits, t)
        v, i = g.sort_long_rows(x)
        want_k, want_i = oracle(bits, t, False)
        same(host(v, t), want_k, f"{t} {shape}: keys")
        same(i.cpu().numpy().view(np.uint32), want_i, f"{t} {shape}: indices")
        only = g.sort_long_rows(x, descending=True, return_indices=False)
        same(host(only, t), oracle(bits, t, True)[0], f"{t} {shape}: descending keys")
        if shape[1] > cap(t):
            kb = 8 if width(t) == 64 else 4
            key = (x.device.index, kb, 4, int(torch.cuda.current_stream().cuda_stream))
            assert onesweep._CACHE[key].max_n >= x.numel()


# ---- 9. graphs and sharing ------------------------------------------------------------------------------------------------------
def test_graph_capture_and_replay(g):
    rng = np.random.default_rng(43)
    shapes = {"f32": (3, 40000), "bf16": (2, 70001), "i64": (5, 9000)}
    sorters = {t: sorter(g, t, shape[0] * shape[1]) for t, shape in shapes.items()}
    try:
        bufs = {t: torch.zeros(shape, dtype=TYPES[t][0], device="cuda") for t, shape in shapes.items()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for t, b in bufs.items():
                sorters[t].sort_long_rows(b, t, True)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = {t: sorters[t].sort_long_rows(b, t, True) for t, b in bufs.items()}
        for replay in range(3):
            want = {}
            for t, shape in shapes.items():
                bits = typed_input(rng, shape[0] * shape[1], t).reshape(shape)
                if replay == 2:
                    bits[:] = bits[0, 0]  # every place skipped: the copy home with positions
                bufs[t].copy_(dev(bits, t))
                want[t] = oracle(bits, t, True)
            graph.replay()
            torch.cuda.synchronize()
            for t, (v, i) in outs.items():
                same(host(v, t), want[t][0], f"replay {replay} {t}: keys")
                same(i.cpu().numpy().view(np.uint32), want[t][1], f"replay {replay} {t}: indices")
        del graph
    finally:
        for s in sorters.values():
            s.close()


def test_two_handles_on_two_streams(g):
    rng = np.random.default_rng(47)
    shape = (6, 50000)
    a, b = sorter(g, "f32", shape[0] * shape[1]), sorter(g, "f32", shape[0] * shape[1])
    try:
        bits = [typed_input(rng, shape[0] * shape[1], "f32").reshape(shape) for _ in range(2)]
        xs = [dev(v, "f32") for v in bits]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        for st in streams:
            st.wait_stream(torch.cuda.current_stream())
        res = []
        for s, x, st in zip((a, b), xs, streams):
            res.append(s.sort_long_rows(x, "f32", False, stream=st))
        torch.cuda.synchronize()
        for (v, i), bt in zip(res, bits):
            wk, wi = oracle(bt, "f32", False)
            same(host(v, "f32"), wk, "keys")
            same(i.cpu().numpy().view(np.uint32), wi, "indices")
    finally:
        a.close()
        b.close()


def test_one_handle_shared_with_other_calls(g):
    """sort_long_rows alternating with the fused u32 sort, argsort, sort_segments and topk_segments on one (4, 4) handle:
    the tile counts in the reductions and the plan must not leak into the other calls, nor theirs into it"""
    rng = np.random.default_rng(53)
    n = 1 << 21
    with g.OneSweepSorter(n, 4, 4) as s:
        for step in range(3):
            rows = typed_input(rng, 3 * 70000, "f32").reshape(3, 70000)
            check(s, rows, "f32", step == 1, f"step {step}: long rows")
            u = rng.integers(0, 1 << 32, n, dtype=np.uint32)
            x = torch.from_numpy(u.view(np.int32).copy()).cuda()
            s.sort_keys(x)
            same(x.cpu().numpy().view(np.uint32), np.sort(u), f"step {step}: fused keys")
            assert s.info("last_fused_kept") == 1
            check(s, typed_input(rng, 2 * 20000, "bf16").reshape(2, 20000), "bf16", True, f"step {step}: bf16 long rows")
            f = typed_input(rng, n, "f32")
            v, i = s.argsort(dev(f, "f32"), "f32")
            wk, wi = oracle(f.reshape(1, -1), "f32", False)
            same(host(v, "f32"), wk, f"step {step}: argsort keys")
            same(i.cpu().numpy().view(np.uint32), wi, f"step {step}: argsort indices")
            lens = rng.integers(0, 3000, 200)
            off = np.concatenate([[0], np.cumsum(lens)])
            segs = typed_input(rng, int(off[-1]), "i32")
            xo = torch.from_numpy(off.astype(np.int64)).cuda()
            v, i = s.sort_segments(dev(segs, "i32"), xo, "i32")
            topv, topi = s.topk_segments(dev(segs, "i32"), xo, 5, "i32", largest=True)
            gv, gi, tv, ti = host(v, "i32"), i.cpu().numpy().view(np.uint32), host(topv, "i32"), topi.cpu().numpy()
            for j in range(200):
                lo, hi = off[j], off[j + 1]
                if hi - lo == 0:
                    continue
                wk, wi = oracle(segs[lo:hi].reshape(1, -1), "i32", False)
                same(gv[lo:hi], wk, f"step {step}: segment {j}")
                same(gi[lo:hi], wi, f"step {step}: segment {j} indices")
                dk, di = oracle(segs[lo:hi].reshape(1, -1), "i32", True)
                m = min(5, hi - lo)
                same(tv[j, :m], dk.reshape(-1)[:m], f"step {step}: top-k {j}")
                same(ti[j, :m].view(np.uint32), di.reshape(-1)[:m], f"step {step}: top-k {j} indices")


# ---- 10. past 2^31 and 2^32 ------------------------------------------------------------------------------------------------------
def require(gib):
    free = torch.cuda.mem_get_info()[0]
    if free < gib * (1 << 30):
        pytest.skip(f"needs {gib} GiB of free device memory, {free / (1 << 30):.1f} GiB free")


def test_one_row_past_2pow31_u16(g):
    """one row of 2^31 + 2^20 + 3 uint16 keys (about 34 GiB with the sorter): positions past 2^31 read negative in int32"""
    require(34)
    row_len = (1 << 31) + (1 << 20) + 3
    gen = torch.Generator(device="cuda").manual_seed(59)
    x = torch.randint(-(1 << 15), 1 << 15, (1, row_len), generator=gen, device="cuda", dtype=torch.int16).view(torch.uint16)
    with g.OneSweepSorter(row_len, 4, 4) as s:
        v, i = s.sort_long_rows(x, "u16")
        torch.cuda.synchronize()
        assert s.info("last_executed_passes") == 2
        bigcheck.check_sorted_by_position(v.reshape(-1), i.reshape(-1), x.reshape(-1), bigcheck.key_radix("u16"), 1 << 28)


def test_batch_past_2pow32_u16(g):
    """4,097 rows of 2^20 + 7 uint16 keys, more than 2^32 in all, sorted in place keys only (about 27 GiB with the sorter)"""
    require(27)
    rows, row_len = 4097, (1 << 20) + 7
    gen = torch.Generator(device="cuda").manual_seed(61)
    x = torch.randint(-(1 << 15), 1 << 15, (rows, row_len), generator=gen, device="cuda", dtype=torch.int16).view(torch.uint16)
    keep = x[-3:].clone(), x[:2].clone()
    with g.OneSweepSorter(rows * row_len, 4, 0) as s:
        s.sort_long_rows(x, "u16", descending=True, return_indices=False, inplace=True)
        torch.cuda.synchronize()
    for src, out in ((keep[0], x[-3:]), (keep[1], x[:2])):
        want = torch.sort(src.view(torch.int16).int() & 0xFFFF, dim=-1, descending=True, stable=True).values
        assert torch.equal(out.view(torch.int16).int() & 0xFFFF, want)
    for lo in range(0, rows, 256):
        blk = x[lo:lo + 256].view(torch.int16).int() & 0xFFFF
        assert bool((blk[:, 1:] <= blk[:, :-1]).all()), f"rows {lo}.. not descending"
