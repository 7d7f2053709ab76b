"""osb200_argsort / OneSweepSorter.argsort / argsort: the stable sort of 32-bit keys and its permutation, input untouched.

The library makes the indices on the device: the histogram and the first EXECUTED digit pass read the caller's input, and
that pass writes every key's input position as its payload; the other passes are the pairs passes.  So the cases below
reach every place where "first executed pass" is decided differently: every number of executed passes (0 to 4, with and
without pass skipping), the HOT instantiation of the pass (low-entropy inputs, both rank modes), the forward-progress
fallback (which in the first pass must re-reduce the caller's input), graph replays whose plans differ from the capture's,
the single-block path for n <= 16,384, and n past 2^31.

Every case compares keys and indices element by element with numpy's stable argsort of the radix key (tests.oraclelib
.to_radix) or with torch.sort(stable=True) of the same key, and checks that the input is bit-identical to a copy taken
before the call.  -m gpu"""
import gc

import numpy as np
import pytest
import torch

from tests.oraclelib import from_radix, to_radix

pytestmark = pytest.mark.gpu

GiB = 1 << 30
KINDS = {"u32": "u", "i32": "i", "f32": "f"}
OK, INVALID_ARG, SIZE, UNSUPPORTED = 0, -1, -2, -3


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def dev(a):
    return torch.from_numpy(a.view(np.int32).copy()).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32)


def float_specials():
    """+-0, subnormals, +-max, +-inf and NaNs of both signs (bit patterns)"""
    pos = [0, 1, 0x007FFFFF, 0x7F7FFFFF, 0x7F800000, 0x7F800001, 0x7FC00000, 0x7FFFFFFF, 0x7FC005A5]
    return np.array(pos + [0x80000000 | p for p in pos], dtype=np.uint32)


def typed_input(rng, n, key_type):
    """uint32 bits of n keys: half drawn from 64 values (ties, so stability is observable), half uniform; floats contain
    every special value"""
    bits = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    pool = rng.integers(0, 1 << 32, 64, dtype=np.uint64).astype(np.uint32)
    if key_type == "f32":
        sp = float_specials()
        pool[:sp.size] = sp
        if n >= 4 * sp.size:
            bits[rng.choice(n, sp.size, replace=False)] = sp
    tied = rng.random(n) < 0.5
    bits[tied] = pool[rng.integers(0, pool.size, int(tied.sum()))]
    return bits


def numpy_check(bits, key_type, descending, out, idx, what):
    order = np.argsort(to_radix(bits, KINDS[key_type], descending), kind="stable").astype(np.uint32)
    assert np.array_equal(host(idx), order), f"indices: {what}"
    assert np.array_equal(host(out), bits[order]), f"keys: {what}"


def radix64(t, key_type, descending):
    """int64 tensor whose ascending order is the requested order of the 32-bit keys in t (torch mirror of to_radix)"""
    u = t.view(torch.int32).long() & 0xFFFFFFFF
    if key_type == "i32":
        u = u ^ 0x80000000
    elif key_type == "f32":
        u = torch.where((u >> 31) == 1, u ^ 0xFFFFFFFF, u | 0x80000000)
    return 0xFFFFFFFF - u if descending else u


def torch_check(kin, key_type, descending, out, idx, what):
    _, order = torch.sort(radix64(kin, key_type, descending), stable=True)
    assert torch.equal(idx.long(), order), f"indices: {what}"
    assert torch.equal(out.view(torch.int32), kin.view(torch.int32)[order]), f"keys: {what}"


def run(s, kin, key_type, descending, **kw):
    """argsort on s, asserting that the input is left bit-identical"""
    before = kin.clone()
    out, idx = s.argsort(kin, key_type, descending, **kw)
    torch.cuda.synchronize()
    assert torch.equal(kin.view(torch.int32), before.view(torch.int32)), "the input was modified"
    assert out.dtype == kin.dtype and idx.dtype == torch.int32 and out.numel() == idx.numel()
    return out, idx


def tile_keys(g):
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        return s.info("tile_keys")


def sizes(g):
    t = tile_keys(g)
    return [0, 1, 2, 1000, 16384, 16385, 3 * t + 5, (1 << 22) + 4099]


# ---- 1. types, orders, sizes --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("key_type", ["u32", "i32", "f32"])
def test_types_orders_and_sizes(g, key_type, descending):
    rng = np.random.default_rng(["u32", "i32", "f32"].index(key_type) * 2 + descending)
    ns = sizes(g)
    with g.OneSweepSorter(max(ns), 4, 4) as s:
        for n in ns:
            bits = typed_input(rng, n, key_type)
            kin = dev(bits)
            if key_type == "f32":
                kin = kin.view(torch.float32)
            out, idx = run(s, kin, key_type, descending)
            numpy_check(bits, key_type, descending, out, idx, f"n={n}")
        for mode in rank_modes(s):  # the single-block path's instantiation of each rank mode
            s.set_option("rank_mode", mode)
            for n in [x for x in ns if x <= 16384]:
                bits = typed_input(rng, n, key_type)
                out, idx = run(s, dev(bits), key_type, descending)
                numpy_check(bits, key_type, descending, out, idx, f"n={n} rank_mode={mode}")
        s.set_option("small_path", 0)  # the multi-kernel path at the single-block path's sizes
        for n in [x for x in ns if x <= 16384]:
            bits = typed_input(rng, n, key_type)
            out, idx = run(s, dev(bits), key_type, descending)
            numpy_check(bits, key_type, descending, out, idx, f"n={n} small_path=0")


def test_one_key_writes_both_outputs(g):
    with g.OneSweepSorter(16, 4, 4) as s:
        kin = torch.tensor([-7], dtype=torch.int32, device="cuda")
        out, idx = s.argsort(kin, "i32")
        assert out.tolist() == [-7] and idx.tolist() == [0]


# ---- 2. every number of executed passes ---------------------------------------------------------------------------------
def constant_places_input(rng, n, varying):
    """radix keys in which only the byte places in `varying` differ between keys"""
    r = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    c = np.uint32(0x5AA53CC3)
    mask = np.uint32(sum(0xFF << (8 * p) for p in varying))
    return (r & mask) | (c & ~mask)


EXECUTED = [((), 0), ((3,), 1), ((0, 2), 2), ((0, 1, 3), 3), ((0, 1, 2, 3), 4)]


@pytest.mark.parametrize("key_type,descending", [("u32", False), ("f32", True)])
def test_every_number_of_executed_passes(g, key_type, descending):
    n = 5 * tile_keys(g) + 77
    rng = np.random.default_rng(5)
    with g.OneSweepSorter(n, 4, 4) as s:
        for short_circuit in (1, 0):
            s.set_option("short_circuit", short_circuit)
            for varying, executed in EXECUTED:
                bits = from_radix(constant_places_input(rng, n, varying), KINDS[key_type], descending)
                out, idx = run(s, dev(bits), key_type, descending)
                numpy_check(bits, key_type, descending, out, idx, f"varying places {varying} short_circuit={short_circuit}")
                assert s.info("last_executed_passes") == (executed if short_circuit else 4)


# ---- 3. low entropy: the HOT passes -------------------------------------------------------------------------------------
def rank_modes(s):
    return [0, 1] if s.info("atomic_order_ok") else [1]


@pytest.mark.parametrize("preset", [3, 4, 5])
def test_low_entropy_runs_hot_passes(g, preset):
    n = 1 << 24
    kin = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(kin, preset - 1, 60 + preset)  # entropy preset p ANDs p random words
    with g.OneSweepSorter(n, 4, 4) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for key_type, descending in (("u32", False), ("i32", True)):
                out, idx = run(s, kin, key_type, descending)
                torch_check(kin, key_type, descending, out, idx, f"preset {preset} rank_mode={mode} {key_type}")
                assert s.info("last_hot_mask") != 0


# ---- 4. forward-progress fallback ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["uniform", "hot"])
def test_stalled_tiles_re_reduce_the_input_in_the_first_pass(g, kind):
    """every third tile withholds its reduction, so its successors re-reduce it themselves; in the first executed pass of
    an argsort they must count the caller's input (the output buffers hold whatever was there before)"""
    n = (1 << 22) + 4099
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    if kind == "hot":
        bits[rng.random(n) < 0.8] = 0x3F8000A5
    with g.OneSweepSorter(n, 4, 4) as s:
        s.set_option("spin_cap", 16)
        s.set_option("debug_stall_every", 3)
        s.set_option("debug_max_ctas", 8)
        for key_type, descending in (("u32", False), ("f32", True)):
            kin = dev(bits)
            out, idx = run(s, kin, key_type, descending)
            torch_check(kin, key_type, descending, out, idx, f"{kind} {key_type}")
            assert (s.info("last_hot_mask") != 0) == (kind == "hot")


# ---- 5. graph capture ---------------------------------------------------------------------------------------------------
def test_graph_replays_with_changing_plans(g):
    """one captured argsort replayed with inputs whose plans execute 4, 1, 3 and 0 passes"""
    n = 9 * tile_keys(g) + 1001
    rng = np.random.default_rng(11)
    inputs = [(constant_places_input(rng, n, v), e) for v, e in
              [((0, 1, 2, 3), 4), ((3,), 1), ((0, 1, 3), 3), ((), 0), ((0, 1, 2, 3), 4)]]
    with g.OneSweepSorter(n, 4, 4) as s:
        kin = torch.zeros(n, dtype=torch.int32, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside the capture
            s.argsort(kin, "f32", True)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out, idx = s.argsort(kin, "f32", True)
        for i, (radix, executed) in enumerate(inputs):
            bits = from_radix(radix, "f", True)
            kin.copy_(torch.from_numpy(bits.view(np.int32)))
            before = kin.clone()
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(kin, before), f"replay {i}: the input was modified"
            numpy_check(bits, "f32", True, out, idx, f"replay {i} ({executed} passes)")
            assert s.info("last_executed_passes") == executed
        del graph


# ---- 6. argument errors -------------------------------------------------------------------------------------------------
def test_argument_errors(g):
    n = 4096
    lib = g.lib
    a = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
    b = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
    c = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
    pa, pb, pc = a.data_ptr(), b.data_ptr(), c.data_ptr()

    def call(s, i=pa, o=pb, x=pc, m=n, key_type=0, desc=0):
        return lib.osb200_argsort(s._h, i, o, x, m, key_type, desc, None)

    with g.OneSweepSorter(n, 4, 0) as keys_only, g.OneSweepSorter(n, 8, 0) as wide:
        assert call(keys_only) == INVALID_ARG
        assert call(wide, key_type=3) == INVALID_ARG
    with g.OneSweepSorter(n, 4, 4) as s:
        for kt in (3, 4, 5, 6, -1):
            assert call(s, key_type=kt) == INVALID_ARG, kt
        assert call(s, i=None) == INVALID_ARG
        assert call(s, o=None) == INVALID_ARG
        assert call(s, x=None) == INVALID_ARG
        assert call(s, i=pa + 4) == INVALID_ARG
        assert call(s, o=pb + 4) == INVALID_ARG
        assert call(s, x=pc + 8) == INVALID_ARG
        assert call(s, o=pa) == INVALID_ARG          # in == out
        assert call(s, x=pa + 16) == INVALID_ARG     # indices overlap the input
        assert call(s, i=pb + 16) == INVALID_ARG     # input overlaps the output
        assert call(s, m=n + 1) == SIZE
        assert call(s, m=0, i=None, o=None, x=None) == OK
        assert call(s) == OK
        torch.cuda.synchronize()
        s.set_option("variant", 0)
        assert call(s) == UNSUPPORTED
        with pytest.raises(g.OneSweepError):
            s.argsort(a, "u32")


# ---- 7. past 2^31 -------------------------------------------------------------------------------------------------------
CHUNK = 1 << 28


def test_argsort_u32_past_2pow31(g):
    n = (1 << 31) + 12345
    gc.collect()
    torch.cuda.empty_cache()
    # handle (alt keys + indices, descriptors) + input, output keys, indices + one chunk of int64 indices and gathered keys
    need = g.lib.osb200_workspace_bytes(n, 4, 4) + 12 * n + CHUNK * 24
    free, _ = torch.cuda.mem_get_info()
    if free < need + 4 * GiB:
        pytest.skip(f"needs {need / GiB:.1f} GiB (+4 GiB headroom), {free / GiB:.1f} GiB free")
    kin = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(kin, 0, 17)
    for a in range(0, n, CHUNK):
        kin[a:a + CHUNK].bitwise_and_(0xFFFFF)  # 20-bit keys: ~2048 copies of every value, stability is observable
    s = g.OneSweepSorter(n, 4, 4)
    try:
        out, idx = s.argsort(kin, "u32")
    finally:
        torch.cuda.synchronize()
        s.close()
    del s
    gc.collect()
    torch.cuda.empty_cache()
    for a in range(0, n, CHUNK):
        b = min(a + CHUNK, n)
        e = min(b + 1, n)  # one element of overlap: runs of equal keys cross chunk borders
        ks = out[a:e]
        assert bool((ks[1:] >= ks[:-1]).all()), f"sorted, output [{a}, {e})"
        ix = idx[a:e].long() & 0xFFFFFFFF
        assert torch.equal(kin[ix[:b - a]], out[a:b]), f"out[i] == in[idx[i]], output [{a}, {b})"
        assert bool(((ix[1:] > ix[:-1]) | (ks[1:] != ks[:-1])).all()), f"indices ascend inside runs, output [{a}, {e})"
        del ks, ix
    del out, idx
    gc.collect()
    torch.cuda.empty_cache()
    # the input left as it was: regenerate it chunk by chunk
    again = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(again, 0, 17)
    for a in range(0, n, CHUNK):
        ref = again[a:a + CHUNK].bitwise_and_(0xFFFFF)
        assert torch.equal(kin[a:a + CHUNK], ref), f"input modified in [{a}, {a + CHUNK})"
    del again, ref, kin
    gc.collect()
    torch.cuda.empty_cache()


# ---- 8. module-level call -----------------------------------------------------------------------------------------------
def test_module_level_argsort_on_a_side_stream(g):
    n = 3 * 16384 + 17
    rng = np.random.default_rng(23)
    bits = typed_input(rng, n, "i32")
    kin = dev(bits)
    before = kin.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    out, idx = g.argsort(kin, "i32", descending=True, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(kin, before)
    numpy_check(bits, "i32", True, out, idx, "module-level argsort on a side stream")
    ref, order = torch.sort(kin, descending=True, stable=True)
    assert torch.equal(out, ref) and torch.equal(idx.long(), order)
