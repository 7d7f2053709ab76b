"""osb200_sort_keys16 / osb200_sort_pairs16 / osb200_argsort16 and their Python methods: 16-bit keys (uint16, int16, float16,
bfloat16) sorted in two digit passes on a 4-byte sorter.

Every case compares element by element with numpy's stable argsort of the 16-bit radix key (radix16 below, which restates
tests.oraclelib.to_radix for 16-bit containers); payloads are the input index, so the payloads and indices ARE the stable
order.  The cases reach every place where the key width matters: the single-block path (n <= 16,384) and the multi-kernel
path on both sides of the tile sizes (12,288 keys, 8,192 pairs), the padding of the ragged last tile (0xFFFF, which keys
whose radix image is 0xFFFF tie with), 0/1/2 executed passes, the HOT passes, stalled tiles, graph replays whose plans
differ from the capture's, both rank modes, and n past 2^31.  In-place calls must leave a guard region after n untouched
and argsort16 its input bit-identical.  -m gpu"""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GiB = 1 << 30
OK, INVALID_ARG, SIZE, UNSUPPORTED = 0, -1, -2, -3
TYPES = ["u16", "i16", "f16", "bf16"]
DTYPE = {"u16": torch.uint16, "i16": torch.int16, "f16": torch.float16, "bf16": torch.bfloat16}
T_KEYS, T_PAIRS = 12288, 8192  # keys per tile of the 16-bit keys pass / pairs and argsort pass
# the single-block path ends at 16,384 keys; 3 * 16,384 + 5 and both sides of the 12,288-key tile as well
SIZES = [0, 1, 2, 1000, T_KEYS - 1, T_KEYS + 1, 16383, 16384, 16385, 3 * T_KEYS + 5, 3 * 16384 + 5, 5 * T_PAIRS + 3,
         (1 << 22) + 4099, (1 << 26) + 1]
GUARD = 64


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def radix16(bits: np.ndarray, key_type: str, descending: bool = False) -> np.ndarray:
    """uint16 key whose ascending order is the requested order of the 16-bit values `bits` (oraclelib.to_radix for 16-bit
    containers): unsigned as is, signed with the sign bit flipped, floats (f16, bf16) in the total order of their bits;
    descending complements the key, so a stable sort on it keeps equal keys in input order in both directions."""
    u = bits.astype(np.uint16)
    if key_type == "i16":
        u = u ^ np.uint16(0x8000)
    elif key_type in ("f16", "bf16"):
        u = np.where(u >> np.uint16(15) == 1, ~u, u | np.uint16(0x8000)).astype(np.uint16)
    return ~u if descending else u


def from_radix16(r: np.ndarray, key_type: str, descending: bool = False) -> np.ndarray:
    """inverse of radix16"""
    u = ~r if descending else r.copy()
    if key_type == "i16":
        u = u ^ np.uint16(0x8000)
    elif key_type in ("f16", "bf16"):
        u = np.where(u >> np.uint16(15) == 1, u ^ np.uint16(0x8000), ~u).astype(np.uint16)
    return u.astype(np.uint16)


def specials(key_type):
    """+-0, subnormals, +-max, +-inf and NaNs of both signs with different payloads (bit patterns)"""
    if key_type == "f16":
        pos = [0, 1, 0x03FF, 0x0400, 0x7BFF, 0x7C00, 0x7C01, 0x7E00, 0x7FFF, 0x7E5A]
    else:
        pos = [0, 1, 0x007F, 0x0080, 0x7F7F, 0x7F80, 0x7F81, 0x7FC0, 0x7FFF, 0x7FA5]
    return np.array(pos + [0x8000 | p for p in pos], dtype=np.uint16)


def typed_input(rng, n, key_type):
    """16-bit patterns: half drawn from 64 values (ties, so stability is observable), half uniform; floats contain every
    special value"""
    bits = rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16)
    pool = rng.integers(0, 1 << 16, 64, dtype=np.uint32).astype(np.uint16)
    if key_type in ("f16", "bf16"):
        sp = specials(key_type)
        pool[:sp.size] = sp
        if n >= 4 * sp.size:
            bits[rng.choice(n, sp.size, replace=False)] = sp
    tied = rng.random(n) < 0.5
    bits[tied] = pool[rng.integers(0, pool.size, int(tied.sum()))]
    return bits


def dev(bits, key_type, extra=0, rng=None):
    """bits (uint16) on the device as a tensor of the key type's dtype; `extra` random guard elements after them"""
    a = bits if not extra else np.concatenate([bits, rng.integers(0, 1 << 16, extra, dtype=np.uint32).astype(np.uint16)])
    return torch.from_numpy(a.view(np.int16).copy()).cuda().view(DTYPE[key_type])


def host(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def rank_modes(s):
    return [0, 1] if s.info("atomic_order_ok") else [1]


def same(got, want, what):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} of {want.size} elements differ, the first at {bad[0] if bad.size else -1}"


def check_all(s, bits, key_type, descending, what, rng, entry=("keys", "pairs", "argsort")):
    """runs the three entry points on `bits` and compares each with the stable order of the radix key"""
    n = bits.size
    order = np.argsort(radix16(bits, key_type, descending), kind="stable").astype(np.uint32)
    want = bits[order]
    if "keys" in entry:
        k = dev(bits, key_type, GUARD, rng)
        guard = host(k[n:])
        s.sort_keys16(k, key_type, descending, n=n)
        got = host(k)
        same(got[:n], want, f"sort_keys16 keys, {what}")
        same(got[n:], guard, f"sort_keys16 guard after n, {what}")
    if "pairs" in entry:
        k = dev(bits, key_type, GUARD, rng)
        v = torch.arange(n + GUARD, dtype=torch.int32, device="cuda")
        guard = host(k[n:])
        s.sort_pairs16(k, v, key_type, descending, n=n)
        got = host(k)
        same(got[:n], want, f"sort_pairs16 keys, {what}")
        same(got[n:], guard, f"sort_pairs16 key guard after n, {what}")
        gv = v.cpu().numpy().view(np.uint32)
        same(gv[:n], order, f"sort_pairs16 payloads, {what}")
        same(gv[n:], np.arange(n, n + GUARD, dtype=np.uint32), f"sort_pairs16 payload guard after n, {what}")
    if "argsort" in entry:
        kin = dev(bits, key_type)
        out, idx = s.argsort16(kin, key_type, descending)
        assert out.dtype == kin.dtype and idx.dtype == torch.int32 and out.numel() == n == idx.numel()
        same(host(kin), bits, f"argsort16 input modified, {what}")
        same(host(out), want, f"argsort16 keys, {what}")
        same(idx.cpu().numpy().view(np.uint32), order, f"argsort16 indices, {what}")


# ---- 1. types, orders, sizes, rank modes ---------------------------------------------------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("key_type", TYPES)
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_types_orders_and_sizes(g, rank_mode, key_type, descending):
    rng = np.random.default_rng(TYPES.index(key_type) * 4 + descending * 2 + rank_mode)
    with g.OneSweepSorter(max(SIZES), 4, 4) as s:
        if rank_mode not in rank_modes(s):
            pytest.skip("the atomic rank mode failed its self-test on this device")
        s.set_option("rank_mode", rank_mode)
        for n in SIZES:
            check_all(s, typed_input(rng, n, key_type), key_type, descending, f"n={n}", rng)
        s.set_option("small_path", 0)  # the multi-kernel path at the single-block path's sizes
        for n in [x for x in SIZES if 2 <= x <= 16384]:
            check_all(s, typed_input(rng, n, key_type), key_type, descending, f"n={n} small_path=0", rng)


def test_keys_only_sorter(g):
    """sort_keys16 on a (4, 0) sorter: its tiles are no smaller than that handle's descriptors assume"""
    rng = np.random.default_rng(3)
    n = 9 * T_KEYS + 11
    with g.OneSweepSorter(n, 4, 0) as s:
        for key_type in TYPES:
            check_all(s, typed_input(rng, n, key_type), key_type, False, f"(4, 0) sorter {key_type}", rng, entry=("keys",))


def test_one_key_writes_both_outputs(g):
    with g.OneSweepSorter(16, 4, 4) as s:
        kin = torch.tensor([-7], dtype=torch.int16, device="cuda")
        out, idx = s.argsort16(kin, "i16")
        assert out.tolist() == [-7] and idx.tolist() == [0]


# ---- 2. float special values ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key_type", ["f16", "bf16"])
def test_float_specials(g, key_type):
    rng = np.random.default_rng(5)
    sp = specials(key_type)
    with g.OneSweepSorter(1 << 20, 4, 4) as s:
        for n in (sp.size, 5000, 3 * T_KEYS + 5, (1 << 20) - 3):  # the single-block and the multi-kernel path
            bits = sp[rng.integers(0, sp.size, n)]
            for descending in (False, True):
                check_all(s, bits, key_type, descending, f"specials n={n} descending={descending}", rng)


# ---- 3. 0, 1 and 2 executed passes ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("key_type,descending", [("u16", False), ("bf16", True), ("i16", True)])
def test_executed_passes(g, key_type, descending):
    n = 5 * T_KEYS + 77
    rng = np.random.default_rng(7)
    with g.OneSweepSorter(n, 4, 4) as s:
        for short_circuit in (1, 0):
            s.set_option("short_circuit", short_circuit)
            for mask, executed in ((0x0000, 0), (0x00FF, 1), (0xFF00, 1), (0xFFFF, 2)):
                r = (rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16) & np.uint16(mask)) | np.uint16(0x5AA5 & ~mask)
                bits = from_radix16(r, key_type, descending)
                what = f"varying mask {mask:#06x} short_circuit={short_circuit}"
                for entry in ("keys", "pairs", "argsort"):
                    check_all(s, bits, key_type, descending, what, rng, entry=(entry,))
                    assert s.info("last_executed_passes") == (executed if short_circuit else 2), f"{entry} {what}"


# ---- 4. hot passes -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_hot_passes(g, rank_mode):
    n = (1 << 22) + 999
    rng = np.random.default_rng(9)
    bits = rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16)
    bits[rng.random(n) < 0.3] = 0x3F80  # bf16 1.0: both digit places have a bin with >= n/8 keys
    with g.OneSweepSorter(n, 4, 4) as s:
        if rank_mode not in rank_modes(s):
            pytest.skip("the atomic rank mode failed its self-test on this device")
        s.set_option("rank_mode", rank_mode)
        for hot in (1, 0):
            s.set_option("hot_passes", hot)
            for entry in ("keys", "pairs", "argsort"):
                check_all(s, bits, "bf16", False, f"hot_passes={hot}", rng, entry=(entry,))
                assert (s.info("last_hot_mask") == 0b11) if hot else (s.info("last_hot_mask") == 0), f"{entry} hot={hot}"


# ---- 5. stalled tiles ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stall_every", [2, 3, 7])
def test_stalled_tiles(g, stall_every):
    """every stall_every-th tile withholds its reduction: its successors re-reduce it (argsort16's first pass: the caller's
    input), on 1, 3 or all resident CTAs of the persistent keys pass"""
    n = (1 << 21) + 4099
    rng = np.random.default_rng(11 + stall_every)
    bits = typed_input(rng, n, "f16")
    with g.OneSweepSorter(n, 4, 4) as s:
        s.set_option("spin_cap", 16)
        s.set_option("debug_stall_every", stall_every)
        for max_ctas in (1, 3, 0):
            s.set_option("debug_max_ctas", max_ctas)
            check_all(s, bits, "f16", max_ctas == 3, f"stall_every={stall_every} max_ctas={max_ctas}", rng)


# ---- 6. keys whose radix image is 0xFFFF (the padding of the ragged last tile) --------------------------------------------
@pytest.mark.parametrize("key_type,descending", [("u16", False), ("i16", True), ("bf16", False), ("f16", True)])
def test_all_ones_radix_keys(g, key_type, descending):
    rng = np.random.default_rng(13)
    with g.OneSweepSorter(1 << 18, 4, 4) as s:
        for small in (1, 0):
            s.set_option("small_path", small)
            for n in (1000, 16384, 3 * T_KEYS + 5, 5 * T_PAIRS + 3):
                r = rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16)
                r[rng.random(n) < 0.5] = 0xFFFF
                r[-7:] = 0xFFFF  # the last tile ends in them
                r[rng.random(n) < 0.1] = 0xFF00 | (r[0] & 0xFF)  # and ties in the high digit 0xFF
                bits = from_radix16(r, key_type, descending)
                check_all(s, bits, key_type, descending, f"n={n} small_path={small}", rng)


# ---- 7. graph capture ----------------------------------------------------------------------------------------------------
def test_graph_replays_with_changing_plans(g):
    """each entry point captured once and replayed with inputs whose plans execute 2, 1, 0 and 2 passes"""
    n = 9 * T_KEYS + 1001
    rng = np.random.default_rng(17)
    masks = [(0xFFFF, 2), (0xFF00, 1), (0x0000, 0), (0xFFFF, 2)]
    kt, desc = "bf16", True
    with g.OneSweepSorter(n, 4, 4) as s:
        kbuf = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
        vbuf = torch.zeros(n, dtype=torch.int32, device="cuda")
        kin = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside the capture
            s.sort_keys16(kbuf, kt, desc)
            s.sort_pairs16(kbuf, vbuf, kt, desc)
            s.argsort16(kin, kt, desc)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graphs = {}
        for entry in ("keys", "pairs", "argsort"):
            graphs[entry] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[entry]):
                if entry == "keys":
                    s.sort_keys16(kbuf, kt, desc)
                elif entry == "pairs":
                    s.sort_pairs16(kbuf, vbuf, kt, desc)
                else:
                    out, idx = s.argsort16(kin, kt, desc)
        for i, (mask, executed) in enumerate(masks):
            r = (rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16) & np.uint16(mask)) | np.uint16(0xC33C & ~mask)
            r[rng.random(n) < 0.3] = r[0]  # ties
            bits = from_radix16(r, kt, desc)
            order = np.argsort(radix16(bits, kt, desc), kind="stable").astype(np.uint32)
            t = torch.from_numpy(bits.view(np.int16).copy()).cuda().view(torch.bfloat16)
            for entry in ("keys", "pairs", "argsort"):
                what = f"replay {i} ({executed} passes) of {entry}"
                kbuf.copy_(t)
                kin.copy_(t)
                vbuf.copy_(torch.arange(n, dtype=torch.int32, device="cuda"))
                graphs[entry].replay()
                torch.cuda.synchronize()
                if entry == "argsort":
                    same(host(kin), bits, f"{what}: input modified")
                    same(host(out), bits[order], what)
                    same(idx.cpu().numpy().view(np.uint32), order, what)
                else:
                    same(host(kbuf), bits[order], what)
                    if entry == "pairs":
                        same(vbuf.cpu().numpy().view(np.uint32), order, what)
                assert s.info("last_executed_passes") == executed, what
        del graphs


# ---- 8. cross-check against torch.sort -----------------------------------------------------------------------------------
def normal16(n, dtype, seed):
    """normal-distributed values without NaN and without -0.0 (torch orders -0.0 == +0.0, the bit order does not)"""
    x = torch.randn(n, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda").to(dtype)
    return torch.where(x == 0, torch.zeros_like(x), x)


@pytest.mark.parametrize("key_type", ["f16", "bf16"])
def test_against_torch_sort(g, key_type):
    n = 1 << 24
    x = normal16(n, DTYPE[key_type], 19)
    with g.OneSweepSorter(n, 4, 4) as s:
        for descending in (False, True):
            ref, order = torch.sort(x, descending=descending, stable=True)
            k = x.clone()
            s.sort_keys16(k, key_type, descending)
            assert torch.equal(k.view(torch.int16), ref.view(torch.int16)), f"sort_keys16 descending={descending}"
            out, idx = s.argsort16(x, key_type, descending)
            assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), f"argsort16 keys descending={descending}"
            assert torch.equal(idx.long(), order), f"argsort16 indices descending={descending}"


CHUNK = 1 << 27


def test_bf16_argsort_2pow30_against_torch_sort(g):
    n = 1 << 30
    gc.collect()
    torch.cuda.empty_cache()
    # handle + input, output keys, indices + torch.sort's values, int64 indices and its scratch
    need = g.lib.osb200_workspace_bytes(n, 4, 4) + 8 * n + 26 * n
    free, _ = torch.cuda.mem_get_info()
    if free < need + 4 * GiB:
        pytest.skip(f"needs {need / GiB:.1f} GiB (+4 GiB headroom), {free / GiB:.1f} GiB free")
    x = normal16(n, torch.bfloat16, 23)
    s = g.OneSweepSorter(n, 4, 4)
    try:
        out, idx = s.argsort16(x, "bf16")
    finally:
        torch.cuda.synchronize()
        s.close()
    del s
    gc.collect()
    torch.cuda.empty_cache()
    ref, order = torch.sort(x, stable=True)
    for a in range(0, n, CHUNK):
        b = min(a + CHUNK, n)
        assert torch.equal(out[a:b].view(torch.int16), ref[a:b].view(torch.int16)), f"keys [{a}, {b})"
        assert torch.equal(idx[a:b].long(), order[a:b]), f"indices [{a}, {b})"
    del x, out, idx, ref, order
    gc.collect()
    torch.cuda.empty_cache()


# ---- 9. argument errors --------------------------------------------------------------------------------------------------
def test_argument_errors(g):
    n = 4096
    lib = g.lib
    a = torch.zeros(8 * n, dtype=torch.int16, device="cuda")  # room for n keys and, behind them, n indices
    b = torch.zeros(2 * n + 64, dtype=torch.int16, device="cuda")
    c = torch.zeros(n + 16, dtype=torch.int32, device="cuda")
    pa, pb, pc = a.data_ptr(), b.data_ptr(), c.data_ptr()

    def keys(s, k=pa, m=n, key_type=0, desc=0):
        return lib.osb200_sort_keys16(s._h, k, m, key_type, desc, None)

    def pairs(s, k=pa, v=pc, m=n, key_type=0, desc=0):
        return lib.osb200_sort_pairs16(s._h, k, v, m, key_type, desc, None)

    def argsort(s, i=pa, o=pb, x=pc, m=n, key_type=0, desc=0):
        return lib.osb200_argsort16(s._h, i, o, x, m, key_type, desc, None)

    with g.OneSweepSorter(n, 8, 0) as wide, g.OneSweepSorter(n, 4, 0) as keys_only:
        assert keys(wide) == INVALID_ARG
        assert pairs(wide) == INVALID_ARG
        assert argsort(wide) == INVALID_ARG
        assert pairs(keys_only) == INVALID_ARG      # value_bytes 0
        assert argsort(keys_only) == INVALID_ARG
        assert keys(keys_only) == OK
    with g.OneSweepSorter(n, 4, 4) as s:
        for kt in (4, 5, -1, 100):
            assert keys(s, key_type=kt) == INVALID_ARG, kt
            assert pairs(s, key_type=kt) == INVALID_ARG, kt
            assert argsort(s, key_type=kt) == INVALID_ARG, kt
        for off in range(2, 16, 2):  # keys at +2 .. +14 B
            assert keys(s, k=pa + off) == INVALID_ARG, off
            assert pairs(s, k=pa + off) == INVALID_ARG, off
            assert argsort(s, i=pa + off) == INVALID_ARG, off
            assert argsort(s, o=pb + off) == INVALID_ARG, off
        assert argsort(s, x=pc + 4) == INVALID_ARG
        assert argsort(s, x=pc + 8) == INVALID_ARG
        for off in (4, 8, 12):  # values at 4-byte offsets are fine
            assert pairs(s, v=pc + off) == OK, off
        assert keys(s, k=None) == INVALID_ARG
        assert pairs(s, v=None) == INVALID_ARG
        assert argsort(s, i=None) == INVALID_ARG
        assert argsort(s, o=None) == INVALID_ARG
        assert argsort(s, x=None) == INVALID_ARG
        assert argsort(s, o=pa) == INVALID_ARG                       # in == out
        assert argsort(s, o=pa + 2 * n - 16) == INVALID_ARG          # the output's head overlaps the input's tail
        assert argsort(s, o=pa + 2 * n) == OK                        # adjacent: no overlap (2n bytes of keys)
        assert argsort(s, i=pb, o=pa, x=pa + 2 * n) == OK            # indices right behind the output keys
        assert argsort(s, i=pb, o=pa, x=pa + 2 * n - 16) == INVALID_ARG  # indices overlap the output keys
        assert keys(s, m=n + 1) == SIZE
        assert pairs(s, m=n + 1) == SIZE
        assert argsort(s, m=n + 1) == SIZE
        assert keys(s, m=0, k=None) == OK and keys(s, m=1, k=None) == OK
        assert pairs(s, m=0, k=None, v=None) == OK
        assert argsort(s, m=0, i=None, o=None, x=None) == OK
        for kt in range(4):
            assert keys(s, key_type=kt, desc=1) == OK
            assert pairs(s, key_type=kt) == OK
            assert argsort(s, key_type=kt) == OK
        torch.cuda.synchronize()
        for v in (0, 1):
            s.set_option("variant", v)
            assert keys(s) == UNSUPPORTED
            assert pairs(s) == UNSUPPORTED
            assert argsort(s) == UNSUPPORTED
        s.set_option("variant", 2)
        with pytest.raises(TypeError):
            s.sort_keys16(torch.zeros(16, dtype=torch.int32, device="cuda"), "i16")
        with pytest.raises(TypeError):
            s.sort_keys_typed(torch.zeros(16, dtype=torch.int16, device="cuda"), "i32")
    with pytest.raises(g.OneSweepError):
        with g.OneSweepSorter(n, 4, 0) as s:
            s.argsort16(a[:n], "i16")


# ---- 10. module-level call -----------------------------------------------------------------------------------------------
def test_module_level_argsort16_on_a_side_stream(g):
    n = 3 * 16384 + 17
    rng = np.random.default_rng(29)
    bits = typed_input(rng, n, "i16")
    kin = dev(bits, "i16")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    out, idx = g.argsort16(kin, "i16", descending=True, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    same(host(kin), bits, "input modified")
    order = np.argsort(radix16(bits, "i16", True), kind="stable").astype(np.uint32)
    same(host(out), bits[order], "keys")
    same(idx.cpu().numpy().view(np.uint32), order, "indices")
    ref, ref_order = torch.sort(kin, descending=True, stable=True)
    assert torch.equal(out, ref) and torch.equal(idx.long(), ref_order)


# ---- 11. past 2^31 -------------------------------------------------------------------------------------------------------
def test_argsort16_past_2pow31(g):
    n = (1 << 31) + 12345
    gc.collect()
    torch.cuda.empty_cache()
    # handle + input, output keys, indices + one chunk of int64 indices and gathered keys
    need = g.lib.osb200_workspace_bytes(n, 4, 4) + 8 * n + CHUNK * 24
    free, _ = torch.cuda.mem_get_info()
    if free < need + 4 * GiB:
        pytest.skip(f"needs {need / GiB:.1f} GiB (+4 GiB headroom), {free / GiB:.1f} GiB free")
    kin = torch.randint(-(1 << 15), 1 << 15, (n,), dtype=torch.int16, device="cuda")  # ~32K copies of every value
    before = kin.clone()
    s = g.OneSweepSorter(n, 4, 4)
    try:
        out, idx = s.argsort16(kin, "i16")
    finally:
        torch.cuda.synchronize()
        s.close()
    del s
    gc.collect()
    torch.cuda.empty_cache()
    assert torch.equal(kin, before), "the input was modified"
    del before
    for a in range(0, n, CHUNK):
        b = min(a + CHUNK, n)
        e = min(b + 1, n)  # one element of overlap: runs of equal keys cross chunk borders
        ks = out[a:e]
        assert bool((ks[1:] >= ks[:-1]).all()), f"sorted, output [{a}, {e})"
        ix = idx[a:e].long() & 0xFFFFFFFF
        assert torch.equal(kin[ix[:b - a]], out[a:b]), f"out[i] == in[idx[i]], output [{a}, {b})"
        assert bool(((ix[1:] > ix[:-1]) | (ks[1:] != ks[:-1])).all()), f"indices ascend inside runs, output [{a}, {e})"
        del ks, ix
    del out, idx, kin
    gc.collect()
    torch.cuda.empty_cache()
