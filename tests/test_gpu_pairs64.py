"""64-bit keys with uint32 payloads: osb200_create_pairs64, osb200_sort_pairs_typed and osb200_argsort on a (8, 4) handle, and
the Python calls on top of them (OneSweepSorter(max_n, 8, 4), the module-level argsort and Sort).

Every case compares element by element with numpy's stable argsort of tests.oraclelib.to_radix of the uint64 bits; the
payloads of sort_pairs_typed are random 32-bit words, the argsort's indices ARE the stable order, and the argsort's input
must be bit-identical afterwards.  The cases reach every place where the 64-bit pairs differ from the other pairs passes:
the single-block path (n <= 8,192) and the multi-kernel path on both sides of its tile, the padding of the ragged last
tile (all ones, which keys whose radix image is all ones tie with), 0 to 8 executed passes, HOT passes, stalled tiles
(the argsort's first pass re-reduces from the caller's input), graph replays whose plans differ from the capture's, payload
views at 4-byte offsets, both rank modes, and a cross-check against torch.sort up to 2^30 keys.  -m gpu"""
import ctypes
import gc

import numpy as np
import pytest
import torch

from tests.oraclelib import from_radix, to_radix

pytestmark = pytest.mark.gpu

GiB = 1 << 30
OK, INVALID_ARG, SIZE, UNSUPPORTED = 0, -1, -2, -3
TYPES = ["u64", "i64", "f64"]
KIND = {"u64": "u", "i64": "i", "f64": "f"}
KEY_TYPE = {"u32": 0, "i32": 1, "f32": 2, "u64": 3, "i64": 4, "f64": 5}
DTYPE = {"u64": torch.uint64, "i64": torch.int64, "f64": torch.float64}
SMALL = 8192  # the single-block path of 64-bit keys
GUARD = 64


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


@pytest.fixture(scope="module")
def tile(g):
    with g.OneSweepSorter(16, 8, 4) as s:
        return s.info("tile_keys")


def sizes(t):
    return sorted({0, 1, 2, 1000, SMALL - 1, SMALL, SMALL + 1, t - 1, t, t + 1, 3 * t + 5, (1 << 22) + 4099})


def specials():
    """+-0, subnormals, +-max, +-inf and NaNs of both signs with different payloads (float64 bit patterns)"""
    pos = [0, 1, 0x000FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF, 0x7FF0000000000000, 0x7FF0000000000001,
           0x7FF8000000000000, 0x7FFFFFFFFFFFFFFF, 0x7FF4A5A5A5A5A5A5, 0x3FF0000000000000]
    return np.array(pos + [(1 << 63) | p for p in pos], dtype=np.uint64)


def typed_input(rng, n, key_type):
    """64-bit patterns: half drawn from 64 values (ties, so stability is observable), half uniform; floats contain every
    special value"""
    bits = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    pool = rng.integers(0, 1 << 64, 64, dtype=np.uint64)
    if key_type == "f64":
        sp = specials()
        pool[:sp.size] = sp
        if n >= 4 * sp.size:
            bits[rng.choice(n, sp.size, replace=False)] = sp
    tied = rng.random(n) < 0.5
    bits[tied] = pool[rng.integers(0, pool.size, int(tied.sum()))]
    return bits


def dev(bits, key_type, extra=0, rng=None):
    """bits (uint64) on the device as a tensor of the key type's dtype; `extra` random guard elements after them"""
    a = bits if not extra else np.concatenate([bits, rng.integers(0, 1 << 64, extra, dtype=np.uint64)])
    return torch.from_numpy(a.view(np.int64).copy()).cuda().view(DTYPE[key_type])


def host(t):
    return t.view(torch.int64).cpu().numpy().view(np.uint64)


def host32(t):
    return t.cpu().numpy().view(np.uint32)


def rank_modes(s):
    return [0, 1] if s.info("atomic_order_ok") else [1]


def same(got, want, what):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} of {want.size} elements differ, the first at {bad[0] if bad.size else -1}"


def check_all(s, bits, key_type, descending, what, rng, entry=("pairs", "argsort")):
    """runs sort_pairs_typed and argsort on `bits` and compares each with the stable order of the radix key"""
    n = bits.size
    order = np.argsort(to_radix(bits, KIND[key_type], descending), kind="stable").astype(np.uint32)
    want = bits[order]
    if "pairs" in entry:
        k = dev(bits, key_type, GUARD, rng)
        vals = rng.integers(0, 1 << 32, n + GUARD, dtype=np.uint64).astype(np.uint32)
        v = torch.from_numpy(vals.view(np.int32).copy()).cuda()
        guard = host(k[n:])
        s.sort_pairs_typed(k, v, key_type, descending, n=n)
        got = host(k)
        same(got[:n], want, f"sort_pairs_typed keys, {what}")
        same(got[n:], guard, f"sort_pairs_typed key guard after n, {what}")
        gv = host32(v)
        same(gv[:n], vals[:n][order], f"sort_pairs_typed payloads, {what}")
        same(gv[n:], vals[n:], f"sort_pairs_typed payload guard after n, {what}")
    if "argsort" in entry:
        kin = dev(bits, key_type)
        out, idx = s.argsort(kin, key_type, descending)
        assert out.dtype == kin.dtype and idx.dtype == torch.int32 and out.numel() == n == idx.numel()
        same(host(kin), bits, f"argsort input modified, {what}")
        same(host(out), want, f"argsort keys, {what}")
        same(host32(idx), order, f"argsort indices, {what}")


def radix_input(rng, n, varying_bytes, fill=0x5AA5C33C0FF01EE1):
    """radix images whose bytes outside `varying_bytes` are those of `fill`: exactly len(varying_bytes) passes execute"""
    mask = np.uint64(sum(0xFF << (8 * b) for b in varying_bytes))
    r = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    r[rng.random(n) < 0.3] = r[0]  # ties
    return (r & mask) | (np.uint64(fill) & ~mask)


# ---- 1. types, orders, sizes, rank modes ---------------------------------------------------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("key_type", TYPES)
def test_types_orders_and_sizes(g, tile, key_type, descending):
    rng = np.random.default_rng(TYPES.index(key_type) * 2 + descending)
    with g.OneSweepSorter(max(sizes(tile)), 8, 4) as s:
        assert s.info("tile_keys") == tile >= 4096
        for rank_mode in rank_modes(s):
            s.set_option("rank_mode", rank_mode)
            for n in sizes(tile):
                check_all(s, typed_input(rng, n, key_type), key_type, descending, f"n={n} rank_mode={rank_mode}", rng)
        s.set_option("small_path", 0)  # the multi-kernel path at the single-block path's sizes
        for n in (2, 1000, SMALL):
            check_all(s, typed_input(rng, n, key_type), key_type, descending, f"n={n} small_path=0", rng)


def test_one_key_writes_both_outputs(g):
    with g.OneSweepSorter(16, 8, 4) as s:
        kin = torch.tensor([-(1 << 40) - 7], dtype=torch.int64, device="cuda")
        out, idx = s.argsort(kin, "i64")
        assert out.tolist() == [-(1 << 40) - 7] and idx.tolist() == [0]


def test_keys_only_calls_on_the_pairs_handle(g, tile):
    rng = np.random.default_rng(2)
    n = 3 * tile + 5
    bits = typed_input(rng, n, "i64")
    with g.OneSweepSorter(n, 8, 4) as s:
        k = dev(bits, "u64")
        s.sort_keys(k)
        same(host(k), np.sort(bits), "sort_keys (osb200_sort_keys_u64)")
        k = dev(bits, "i64")
        s.sort_keys_typed(k, "i64", descending=True)
        same(host(k), bits[np.argsort(to_radix(bits, "i", True), kind="stable")], "sort_keys_typed")
        h = bits.copy()
        s.sort_host(h)
        same(h, np.sort(bits), "sort_host (osb200_sort_host_keys_u64)")


# ---- 2. float special values ---------------------------------------------------------------------------------------------
def test_float_specials(g, tile):
    rng = np.random.default_rng(5)
    sp = specials()
    with g.OneSweepSorter(1 << 20, 8, 4) as s:
        for n in (sp.size, 5000, 3 * tile + 5, (1 << 20) - 3):  # the single-block and the multi-kernel path
            bits = sp[rng.integers(0, sp.size, n)]
            for descending in (False, True):
                check_all(s, bits, "f64", descending, f"specials n={n} descending={descending}", rng)


# ---- 3. 0 to 8 executed passes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key_type,descending", [("u64", False), ("f64", True), ("i64", False)])
def test_executed_passes(g, tile, key_type, descending):
    n = 5 * tile + 77
    rng = np.random.default_rng(7)
    places = [0, 7, 3, 5, 1, 6, 2, 4]
    with g.OneSweepSorter(n, 8, 4) as s:
        for short_circuit in (1, 0):
            s.set_option("short_circuit", short_circuit)
            for executed in range(9):
                bits = from_radix(radix_input(rng, n, places[:executed]), KIND[key_type], descending)
                what = f"{executed} varying bytes short_circuit={short_circuit}"
                for entry in ("pairs", "argsort"):
                    check_all(s, bits, key_type, descending, what, rng, entry=(entry,))
                    assert s.info("last_executed_passes") == (executed if short_circuit else 8), f"{entry} {what}"


# ---- 4. hot passes -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_hot_passes(g, rank_mode):
    n = (1 << 22) + 999
    rng = np.random.default_rng(9)
    bits = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    bits[rng.random(n) < 0.3] = np.uint64(0x3FF0000000000000)  # 1.0: every digit place has a bin with >= n/8 keys
    with g.OneSweepSorter(n, 8, 4) as s:
        if rank_mode not in rank_modes(s):
            pytest.skip("the atomic rank mode failed its self-test on this device")
        s.set_option("rank_mode", rank_mode)
        for hot in (1, 0):
            s.set_option("hot_passes", hot)
            for entry in ("pairs", "argsort"):
                check_all(s, bits, "f64", False, f"hot_passes={hot}", rng, entry=(entry,))
                assert s.info("last_hot_mask") == (0xFF if hot else 0), f"{entry} hot={hot}"


# ---- 5. stalled tiles ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stall_every", [2, 3, 7])
def test_stalled_tiles(g, stall_every):
    """every stall_every-th tile withholds its reduction: its successors re-reduce it (the argsort's first pass: from the
    caller's untouched input); the low-entropy input runs its passes in the persistent HOT instantiation"""
    n = (1 << 21) + 4099
    rng = np.random.default_rng(11 + stall_every)
    with g.OneSweepSorter(1 << 22, 8, 4) as s:
        s.set_option("spin_cap", 16)
        s.set_option("debug_stall_every", stall_every)
        check_all(s, typed_input(rng, n, "i64"), "i64", stall_every == 3, f"stall_every={stall_every}", rng)
        bits = rng.integers(0, 1 << 64, 1 << 22, dtype=np.uint64)
        bits[rng.random(bits.size) < 0.4] = bits[0]
        for max_ctas in (3, 0):
            s.set_option("debug_max_ctas", max_ctas)
            check_all(s, bits, "u64", False, f"hot stall_every={stall_every} max_ctas={max_ctas}", rng)
            assert s.info("last_hot_mask") == 0xFF


# ---- 6. keys whose radix image is all ones (the padding of the ragged last tile and of the small path) -------------------
@pytest.mark.parametrize("key_type,descending", [("u64", False), ("i64", True), ("f64", False), ("f64", True)])
def test_all_ones_radix_keys(g, tile, key_type, descending):
    rng = np.random.default_rng(13)
    ones = np.uint64(0xFFFFFFFFFFFFFFFF)
    with g.OneSweepSorter(1 << 18, 8, 4) as s:
        for small in (1, 0):
            s.set_option("small_path", small)
            for n in (1000, SMALL, 3 * tile + 5, 5 * tile + 3):
                r = rng.integers(0, 1 << 64, n, dtype=np.uint64)
                r[rng.random(n) < 0.5] = ones
                r[-7:] = ones  # the last tile ends in them
                r[rng.random(n) < 0.1] = np.uint64(0xFFFFFFFFFFFFFF00) | (r[0] & np.uint64(0xFF))  # ties in the high digits
                bits = from_radix(r, KIND[key_type], descending)
                check_all(s, bits, key_type, descending, f"n={n} small_path={small}", rng)


# ---- 7. graph capture ----------------------------------------------------------------------------------------------------
def test_graph_replays_with_changing_plans(g, tile):
    """both entry points captured once and replayed with inputs whose plans execute 8, 3, 0 and 8 passes"""
    n = 9 * tile + 1001
    rng = np.random.default_rng(17)
    plans = [(list(range(8)), 8), ([0, 2, 5], 3), ([], 0), (list(range(8)), 8)]
    kt, desc = "f64", True
    with g.OneSweepSorter(n, 8, 4) as s:
        kbuf = torch.zeros(n, dtype=torch.float64, device="cuda")
        vbuf = torch.zeros(n, dtype=torch.int32, device="cuda")
        kin = torch.zeros(n, dtype=torch.float64, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside the capture
            s.sort_pairs_typed(kbuf, vbuf, kt, desc)
            s.argsort(kin, kt, desc)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graphs = {}
        for entry in ("pairs", "argsort"):
            graphs[entry] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[entry]):
                if entry == "pairs":
                    s.sort_pairs_typed(kbuf, vbuf, kt, desc)
                else:
                    out, idx = s.argsort(kin, kt, desc)
        for i, (varying, executed) in enumerate(plans):
            bits = from_radix(radix_input(rng, n, varying), "f", desc)
            order = np.argsort(to_radix(bits, "f", desc), kind="stable").astype(np.uint32)
            t = torch.from_numpy(bits.view(np.int64).copy()).cuda().view(torch.float64)
            for entry in ("pairs", "argsort"):
                what = f"replay {i} ({executed} passes) of {entry}"
                kbuf.copy_(t)
                kin.copy_(t)
                vbuf.copy_(torch.arange(n, dtype=torch.int32, device="cuda"))
                graphs[entry].replay()
                torch.cuda.synchronize()
                if entry == "argsort":
                    same(host(kin), bits, f"{what}: input modified")
                    same(host(out), bits[order], what)
                    same(host32(idx), order, what)
                else:
                    same(host(kbuf), bits[order], what)
                    same(host32(vbuf), order, what)
                assert s.info("last_executed_passes") == executed, what
        del graphs


# ---- 8. payloads at 4-byte offsets ---------------------------------------------------------------------------------------
def test_payload_views_at_4_byte_offsets(g, tile):
    rng = np.random.default_rng(19)
    with g.OneSweepSorter(1 << 16, 8, 4) as s:
        for n in (5000, 3 * tile + 5):
            bits = typed_input(rng, n, "i64")
            order = np.argsort(to_radix(bits, "i"), kind="stable")
            for off in (1, 2, 3):  # +4, +8, +12 bytes
                vals = rng.integers(0, 1 << 32, n + 4, dtype=np.uint64).astype(np.uint32)
                vbuf = torch.from_numpy(vals.view(np.int32).copy()).cuda()
                k = dev(bits, "i64")
                s.sort_pairs_typed(k, vbuf[off:off + n], "i64")
                got = host32(vbuf)
                same(host(k), bits[order], f"keys n={n} offset={4 * off}")
                same(got[off:off + n], vals[off:off + n][order], f"payloads n={n} offset={4 * off}")
                same(got[:off], vals[:off], f"before the view n={n} offset={4 * off}")
                same(got[off + n:], vals[off + n:], f"after the view n={n} offset={4 * off}")


# ---- 9. cross-check against torch.sort -----------------------------------------------------------------------------------
def torch_keys(n, dtype, seed):
    """uniform int64 or normal float64 values without NaN and without -0.0 (torch orders -0.0 == +0.0, the bit order does not)"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if dtype == torch.int64:
        return torch.randint(-(1 << 62), 1 << 62, (n,), dtype=torch.int64, device="cuda", generator=gen)
    x = torch.randn(n, dtype=torch.float64, device="cuda", generator=gen)
    return torch.where(x == 0, torch.zeros_like(x), x)


CHUNK = 1 << 27


def against_torch(g, n, dtype, key_type, seed, descending):
    gc.collect()
    torch.cuda.empty_cache()
    # handle + input, output keys, indices + torch.sort's values, int64 indices and its scratch
    need = g.lib.osb200_workspace_bytes(n, 8, 4) + 20 * n + 40 * n
    free, _ = torch.cuda.mem_get_info()
    if free < need + 4 * GiB:
        pytest.skip(f"needs {need / GiB:.1f} GiB (+4 GiB headroom), {free / GiB:.1f} GiB free")
    x = torch_keys(n, dtype, seed)
    s = g.OneSweepSorter(n, 8, 4)
    try:
        out, idx = s.argsort(x, key_type, descending)
    finally:
        torch.cuda.synchronize()
        s.close()
    del s
    gc.collect()
    torch.cuda.empty_cache()
    ref, order = torch.sort(x, descending=descending, stable=True)
    for a in range(0, n, CHUNK):
        b = min(a + CHUNK, n)
        assert torch.equal(out[a:b], ref[a:b]), f"keys [{a}, {b})"
        assert torch.equal(idx[a:b].long() & 0xFFFFFFFF, order[a:b]), f"indices [{a}, {b})"
    del x, out, idx, ref, order
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("key_type,descending", [("i64", False), ("f64", True)])
def test_against_torch_sort_2pow28(g, key_type, descending):
    against_torch(g, 1 << 28, DTYPE[key_type], key_type, 23, descending)


def test_f64_argsort_2pow30_against_torch_sort(g):
    against_torch(g, 1 << 30, torch.float64, "f64", 29, False)


# ---- 10. argument errors -------------------------------------------------------------------------------------------------
def test_argument_errors(g):
    n = 4096
    lib = g.lib
    a = torch.zeros(2 * n, dtype=torch.int64, device="cuda")  # room for n keys and, behind them, n indices
    b = torch.zeros(n + 8, dtype=torch.int64, device="cuda")
    c = torch.zeros(n + 16, dtype=torch.int32, device="cuda")
    pa, pb, pc = a.data_ptr(), b.data_ptr(), c.data_ptr()

    def pairs(s, k=pa, v=pc, m=n, key_type=KEY_TYPE["i64"], desc=0):
        return lib.osb200_sort_pairs_typed(s._h, k, v, m, key_type, desc, None)

    def argsort(s, i=pa, o=pb, x=pc, m=n, key_type=KEY_TYPE["i64"], desc=0):
        return lib.osb200_argsort(s._h, i, o, x, m, key_type, desc, None)

    with g.OneSweepSorter(n, 8, 0) as keys_only, g.OneSweepSorter(n, 4, 4) as narrow:
        assert pairs(keys_only) == INVALID_ARG      # value_bytes 0
        assert argsort(keys_only) == INVALID_ARG
        for kt in ("u64", "i64", "f64"):            # 64-bit key types on a 4-byte handle
            assert pairs(narrow, key_type=KEY_TYPE[kt]) == INVALID_ARG, kt
            assert argsort(narrow, key_type=KEY_TYPE[kt]) == INVALID_ARG, kt
    with g.OneSweepSorter(n, 8, 4) as s:
        assert s.key_bytes == 8 and s.value_bytes == 4
        for kt in (0, 1, 2, -1, 6, 100):             # 32-bit key types and unknown ones
            assert pairs(s, key_type=kt) == INVALID_ARG, kt
            assert argsort(s, key_type=kt) == INVALID_ARG, kt
        for off in (4, 8, 12):                       # keys at +4 .. +12 B
            assert pairs(s, k=pa + off) == INVALID_ARG, off
            assert argsort(s, i=pa + off) == INVALID_ARG, off
            assert argsort(s, o=pb + off) == INVALID_ARG, off
            assert argsort(s, x=pc + off) == INVALID_ARG, off
            assert pairs(s, v=pc + off) == OK, off   # values at 4-byte offsets are fine
        assert pairs(s, k=None) == INVALID_ARG
        assert pairs(s, v=None) == INVALID_ARG
        assert argsort(s, i=None) == INVALID_ARG
        assert argsort(s, o=None) == INVALID_ARG
        assert argsort(s, x=None) == INVALID_ARG
        assert argsort(s, o=pa) == INVALID_ARG                        # in == out
        assert argsort(s, o=pa + 8 * n - 16) == INVALID_ARG           # the output's head overlaps the input's tail
        assert argsort(s, i=pb, o=pa, x=pa + 8 * n) == OK             # indices right behind the output keys (8n bytes)
        assert argsort(s, i=pb, o=pa, x=pa + 8 * n - 16) == INVALID_ARG  # indices overlap the output keys
        assert argsort(s, x=pa + 8 * n - 16) == INVALID_ARG           # indices overlap the input's tail
        assert pairs(s, m=n + 1) == SIZE
        assert argsort(s, m=n + 1) == SIZE
        assert pairs(s, m=0, k=None, v=None) == OK
        assert argsort(s, m=0, i=None, o=None, x=None) == OK
        for kt in ("u64", "i64", "f64"):
            assert pairs(s, key_type=KEY_TYPE[kt], desc=1) == OK
            assert argsort(s, key_type=KEY_TYPE[kt]) == OK
        # what does not take 64-bit keys with payloads stays as it is on this handle
        assert lib.osb200_sort_pairs_u32(s._h, pa, pc, n, None) == INVALID_ARG
        assert lib.osb200_sort_bits(s._h, pa, pc, n, 0, 64, None) == INVALID_ARG
        assert lib.osb200_segmented_sort_u32(s._h, pa, pc, pb, 1, 16, None) == INVALID_ARG
        hk, hv = np.zeros(16, np.uint64), np.zeros(16, np.uint32)
        assert lib.osb200_sort_host_pairs_u32(s._h, hk.ctypes.data, hv.ctypes.data, 16) == INVALID_ARG
        torch.cuda.synchronize()
        for v in (0, 1):
            s.set_option("variant", v)
            assert pairs(s) == UNSUPPORTED
            assert argsort(s) == UNSUPPORTED
        s.set_option("variant", 2)
        with pytest.raises(TypeError):
            s.argsort(torch.zeros(16, dtype=torch.int32, device="cuda"), "i32")
        with pytest.raises(TypeError):
            s.sort_pairs_typed(torch.zeros(16, dtype=torch.float32, device="cuda"),
                               torch.zeros(16, dtype=torch.int32, device="cuda"), "f32")
    h = ctypes.c_void_p()
    assert lib.osb200_create_pairs64(None, 1024) == INVALID_ARG
    assert lib.osb200_create_pairs64(ctypes.byref(h), 0) == INVALID_ARG
    assert lib.osb200_create_pairs64(ctypes.byref(h), (1 << 34) + 1) == INVALID_ARG
    assert h.value is None
    assert lib.osb200_create(ctypes.byref(h), 1024, 8, 4) == UNSUPPORTED


# ---- 11. module-level calls ----------------------------------------------------------------------------------------------
def test_module_level_argsort_on_a_side_stream(g):
    n = 3 * SMALL + 17
    rng = np.random.default_rng(29)
    bits = typed_input(rng, n, "i64")
    kin = dev(bits, "i64")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    out, idx = g.argsort(kin, "i64", descending=True, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    same(host(kin), bits, "input modified")
    order = np.argsort(to_radix(bits, "i", True), kind="stable").astype(np.uint32)
    same(host(out), bits[order], "keys")
    same(host32(idx), order, "indices")
    ref, ref_order = torch.sort(kin, descending=True, stable=True)
    assert torch.equal(out, ref) and torch.equal(idx.long(), ref_order)


def test_module_level_sort_of_int64_keys_with_int32_values(g, tile):
    rng = np.random.default_rng(31)
    for n in (5000, 3 * tile + 5):
        bits = typed_input(rng, n, "u64")
        vals = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
        k = dev(bits, "i64")
        v = torch.from_numpy(vals.view(np.int32).copy()).cuda()
        g.Sort(k, v)
        torch.cuda.synchronize()
        order = np.argsort(bits, kind="stable")  # unsigned bits, as sort_pairs orders every integer container
        same(host(k), bits[order], f"keys n={n}")
        same(host32(v), vals[order], f"values n={n}")
