"""Every path that ranks tiles, on inputs structured by position (tests/structured.py): sorted runs of chosen lengths,
tiles of a single digit, sorted / reversed / nearly sorted / run-concatenated / organ-pipe keys, one outlier key, hot
digits that differ from tile to tile, per-tile counts at the hot-digit threshold, ties, and global bins at the hot rule's
boundary.

Each arm (entry point and key type) sorts each input past 2^22 keys (the HOT kernel), at 3T + 5 keys (the plain kernel
only) and, for runs, whole keys and outliers, at sizes the single-block sort takes; every case runs with hot passes on
and off, in every rank mode the device allows, and on the u32 keys and argsort arms with 0, 1 and 3 persistent CTAs.
Keys, payloads and indices are compared element by element with the stable sort of the radix image (torch.sort on the
device from 2^20 keys, numpy's stable argsort below); argsorts must leave their input bit-identical; the plan the sort
reports (skip mask, hot mask, executed passes) must be expected_plan of the input, and the tile size the one the input
was built for.  Row sorts and segmented sorts get sorted, reversed, run and one-outlier rows and segments.  -m gpu"""
import zlib
from typing import Callable, NamedTuple, Optional

import numpy as np
import pytest
import torch

from tests import structured as st
from tests import test_gpu_rows as rows
from tests.test_gpu_segmented import seg_oracle

pytestmark = pytest.mark.gpu

T_KEYS16, T_PAIRS16 = 12288, 8192  # tiles of the 16-bit keys pass and of the 16-bit pairs / argsort pass
DTYPE = {(16, "i"): torch.int16, (16, "f"): torch.bfloat16, (32, "u"): torch.int32, (32, "i"): torch.int32,
         (32, "f"): torch.float32, (64, "u"): torch.int64, (64, "i"): torch.int64, (64, "f"): torch.float64}


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


class Arm(NamedTuple):
    name: str
    shape: tuple                 # (key_bytes, value_bytes) of the sorter
    T: int                       # tile of the pass the arm runs
    width: int
    kind: str                    # "u", "i" or "f"
    descending: bool
    run: Callable                # (sorter, typed input) -> (sorted keys, payloads / indices or None)
    argsort: bool = False
    ctas: bool = False           # also run with debug_max_ctas 1 and 3
    bits: Optional[tuple] = None  # sort_bits: (begin_bit, end_bit)
    tile_info: bool = True       # info("tile_keys") is this arm's tile (not for the 16-bit calls on a 4-byte sorter)


def _iota(x):
    return torch.arange(x.numel(), dtype=torch.int32, device=x.device)


def _keys(s, x):
    t = x.clone()
    return s.sort_keys(t), None


def _pairs(s, x):
    return s.sort_pairs(x.clone(), _iota(x))


def _pairs_typed(kt, desc):
    return lambda s, x: s.sort_pairs_typed(x.clone(), _iota(x), kt, desc)


def _argsort(kt, desc):
    return lambda s, x: s.argsort(x, kt, desc)


def _keys16(kt, desc):
    return lambda s, x: (s.sort_keys16(x.clone(), kt, desc), None)


def _pairs16(kt, desc):
    return lambda s, x: s.sort_pairs16(x.clone(), _iota(x), kt, desc)


def _argsort16(kt, desc):
    return lambda s, x: s.argsort16(x, kt, desc)


def _bits(b, e, pairs):
    if pairs:
        return lambda s, x: s.sort_bits(x.clone(), b, e, _iota(x))
    return lambda s, x: (s.sort_bits(x.clone(), b, e), None)


ARMS = [
    Arm("u32_keys", (4, 0), 16384, 32, "u", False, _keys, ctas=True),
    Arm("u32_pairs", (4, 4), 8192, 32, "u", False, _pairs),
    Arm("f32_pairs_desc", (4, 4), 8192, 32, "f", True, _pairs_typed("f32", True)),
    Arm("i32_argsort", (4, 4), 8192, 32, "i", False, _argsort("i32", False), argsort=True, ctas=True),
    Arm("f32_argsort_desc", (4, 4), 8192, 32, "f", True, _argsort("f32", True), argsort=True, ctas=True),
    Arm("u64_keys", (8, 0), 8192, 64, "u", False, _keys),
    Arm("i64_argsort", (8, 4), 8192, 64, "i", False, _argsort("i64", False), argsort=True),
    Arm("f64_argsort_desc", (8, 4), 8192, 64, "f", True, _argsort("f64", True), argsort=True),
    Arm("f64_pairs", (8, 4), 8192, 64, "f", False, _pairs_typed("f64", False)),
    Arm("bf16_keys_desc", (4, 4), T_KEYS16, 16, "f", True, _keys16("bf16", True), tile_info=False),
    Arm("i16_keys", (4, 4), T_KEYS16, 16, "i", False, _keys16("i16", False), tile_info=False),
    Arm("bf16_pairs", (4, 4), T_PAIRS16, 16, "f", False, _pairs16("bf16", False), tile_info=False),
    Arm("i16_pairs_desc", (4, 4), T_PAIRS16, 16, "i", True, _pairs16("i16", True), tile_info=False),
    Arm("bf16_argsort_desc", (4, 4), T_PAIRS16, 16, "f", True, _argsort16("bf16", True), argsort=True, tile_info=False),
    Arm("i16_argsort", (4, 4), T_PAIRS16, 16, "i", False, _argsort16("i16", False), argsort=True, tile_info=False),
] + [Arm(f"bits_{b}_{e}_{'pairs' if pairs else 'keys'}", (4, 4 if pairs else 0), 8192 if pairs else 16384, 32, "u",
         False, _bits(b, e, pairs), bits=(b, e))
     for b, e in ((0, 9), (5, 8), (2, 15)) for pairs in (False, True)]  # last digit: 1, 3 and 5 bits


def arm_layout(arm):
    return st.layout(arm.width, *arm.bits) if arm.bits else st.layout(arm.width)


def cases(arm, size, device="cuda"):
    """(label, n, thunk -> (image, plan)) of one arm at one size class; thunks build on the device"""
    T = arm.T
    lay = arm_layout(arm)
    top = len(lay.places) - 1
    few = lay.places[-1][1] < 8  # bit ranges: the structure goes into the narrow last digit
    out = []

    def add(label, n, fn, *args, p=None):
        q = top if few else (p if p is not None else len(out) % len(lay.places))
        seed = zlib.crc32(f"{arm.name} {label} {n}".encode())
        out.append((f"{label} n={n} place={q}", n, lambda: fn(n, T, lay, q, seed, *args, device=device)))

    def add_whole(n):
        if not few:
            for shape in st.WHOLE_SHAPES:
                seed = zlib.crc32(f"{arm.name} {shape} {n}".encode())
                out.append((f"whole {shape} n={n}", n, lambda shape=shape, seed=seed: st.whole_keys(n, T, lay, seed, shape, device)))

    def add_outliers(n):
        for pos in sorted({x for x in (0, T - 1, T, n - 1) if x < n}):
            for above in (False, True):
                add(f"outlier pos={pos} above={above}", n, st.outlier, pos, above)

    if size == "hot":
        n = st.hot_n(T)
        for j, R in enumerate(st.run_lengths(T)):
            add(f"runs R={R} {st.RUN_ORDERS[j % 3]}", n, st.runs, R, st.RUN_ORDERS[j % 3])
        add("tile_blocks", n, st.tile_blocks)
        add_whole(n)
        add_outliers(n)
        if not few:
            add("hot_block", n, st.hot_block, T // 3 + 7)
            add("tile_local_hot", n, st.tile_local_hot)
            nw = st.whole_tiles_n(T)
            for k in (T // 8, T // 8 - 1):
                for lead in (False, True):
                    add(f"tile_threshold k={k} lead={lead}", nw, st.tile_threshold, k, lead)
            add("tile_tie", nw, st.tile_tie)
            for n, c in (((1 << 22), 1 << 19), ((1 << 22), (1 << 19) - 1), ((1 << 22) - 1, 1 << 19)):
                add(f"global_boundary c={c}", n, st.global_boundary, c)
    elif size == "plain":
        n = 3 * T + 5
        for R in st.run_lengths(T):
            for order in st.RUN_ORDERS:
                add(f"runs R={R} {order}", n, st.runs, R, order)
        add("tile_blocks", n, st.tile_blocks)
        add_whole(n)
        add_outliers(n)
        if not few:
            add("hot_block", n, st.hot_block, T // 3 + 7)
            add("tile_local_hot", n, st.tile_local_hot)
    else:  # the single-block sort: every sort of at most small_path_max_n keys
        cap = 8192 if arm.width == 64 else 16384
        for n in (777, cap):
            for R in (1, 32, 33, 257):
                add(f"runs R={R} random", n, st.runs, R, "random")
            add_whole(n)
            add_outliers(n)
    return out


def same(got, want, what):
    if torch.equal(got, want):
        return
    bad = torch.nonzero(got != want).reshape(-1)
    raise AssertionError(f"{what}: {bad.numel()} of {want.numel()} differ, the first at {int(bad[0]) if bad.numel() else -1}")


def ref_order(key, width):
    """stable argsort of radix images: torch.sort on the device from 2^20 keys, numpy below"""
    if key.numel() >= 1 << 20:
        return torch.sort(st.ordered(key, width), stable=True).indices
    a = key.cpu().numpy()
    a = a.view(np.uint64) if width == 64 else a
    return torch.from_numpy(np.argsort(a, kind="stable")).to(key.device)


def rank_modes(s):
    return [0, 1] if s.info("atomic_order_ok") else [1]


@pytest.mark.parametrize("size", ["hot", "plain", "single"])
@pytest.mark.parametrize("arm", ARMS, ids=[a.name for a in ARMS])
def test_structured(g, arm, size):
    lay = arm_layout(arm)
    todo = cases(arm, size)
    max_n = max(n for _, n, _ in todo)
    with g.OneSweepSorter(max_n, *arm.shape) as s:
        if arm.tile_info:
            assert s.info("tile_keys") == arm.T
        small = s.info("small_path_max_n")  # (16-bit keys on a 4-byte sorter: 16,384, as for 32-bit keys)
        assert (max_n <= small) == (size == "single")
        for label, n, make in todo:
            image, promised = make()
            plan = st.expected_plan(image, lay.places)
            assert plan == promised, f"{label}: the input's plan is {plan}, its generator promised {promised}"
            bits = st.to_bits(image, arm.width, arm.kind, arm.descending)
            x = bits.view(DTYPE[(arm.width, arm.kind)])
            key = image if arm.bits is None else (image >> arm.bits[0]) & ((1 << (arm.bits[1] - arm.bits[0])) - 1)
            order = ref_order(key, arm.width)
            want = bits[order]
            del image, key
            for mode in rank_modes(s):
                s.set_option("rank_mode", mode)
                for hot in (1, 0):
                    s.set_option("hot_passes", hot)
                    for ctas in ((0, 1, 3) if arm.ctas and size != "single" else (0,)):
                        s.set_option("debug_max_ctas", ctas)
                        what = f"{arm.name} {label} rank_mode={mode} hot_passes={hot} debug_max_ctas={ctas}"
                        keys, pay = arm.run(s, x)
                        same(keys.view(bits.dtype), want, f"{what}: keys")
                        if pay is not None:
                            same(pay.long() & 0xFFFFFFFF, order, f"{what}: payloads")
                        if arm.argsort:
                            same(x.view(bits.dtype), bits, f"{what}: input modified")
                        if n > small:
                            assert s.info("last_skip_mask") == plan.skip, what
                            assert s.info("last_hot_mask") == (plan.hot if hot else 0), what
                            assert s.info("last_executed_passes") == plan.executed, what
                        del keys, pay
            s.set_option("debug_max_ctas", 0)
            del x, bits, want, order


# ---- row sort --------------------------------------------------------------------------------------------------------------
def row_inputs(rng, num_rows, row_len, t):
    """(label, rows of bits, descending): sorted rows sorted both ways, reversed rows, runs of 31 / 32 / 33 equal keys, and
    rows whose keys are all equal but one, at the first or the last position (every third row has no such key)"""
    c = rows.TYPES[t][1]
    base = rows.random_bits(rng, num_rows * row_len, t).reshape(num_rows, row_len)
    up = np.take_along_axis(base, np.argsort(rows.radix(base, t), axis=-1, kind="stable"), axis=-1)
    out = [("sorted", up, False), ("sorted, sorted descending", up, True), ("reversed", up[:, ::-1].copy(), False)]
    for R in (31, 32, 33):
        pool = rows.random_bits(rng, num_rows * (row_len // R + 1), t).reshape(num_rows, -1)
        out.append((f"runs of {R}", pool[:, np.arange(row_len) // R].copy(), False))
    v = np.repeat(rows.random_bits(rng, num_rows, t)[:, None], row_len, axis=1)
    flip = c(1) << rng.integers(0, 8 * np.dtype(c).itemsize, num_rows).astype(c)  # the differing digit varies by row
    r = np.arange(num_rows)
    v[r % 3 == 0, 0] ^= flip[r % 3 == 0]
    v[r % 3 == 1, -1] ^= flip[r % 3 == 1]
    out += [("all equal but one", v, False), ("all equal but one, descending", v, True)]
    return out


@pytest.mark.parametrize("t", ["bf16", "f32", "i64"])
def test_rows_structured(g, t):
    rng = np.random.default_rng(["bf16", "f32", "i64"].index(t))
    with g.OneSweepSorter(1, 4, 4) as s:
        for block in (0, 1):
            s.set_option("debug_rows_block", block)
            for row_len in (32, 33, 256, 257, 2048, rows.cap(t)):
                num_rows = 3 if row_len >= 2048 else 67
                for label, bits, desc in row_inputs(rng, num_rows, row_len, t):
                    rows.check(s, bits, t, desc, f"{label}, rows of {row_len}, block={block}")


# ---- segmented sort --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seg_len", [256, 2048, 16384])
def test_segmented_structured(g, seg_len):
    """sorted, reversed and one-outlier segments in the 256-, 2,048- and 16,384-key geometries (max_segment_len picks it)"""
    rng = np.random.default_rng(seg_len)
    lens = np.array([seg_len, seg_len - 1, seg_len // 2 + 1, 1, 0, 2] * 4)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    keys = rng.integers(0, 1 << 32, int(offs[-1]), dtype=np.uint64).astype(np.uint32)
    for i, (a, b) in enumerate(zip(offs[:-1], offs[1:])):
        kind = i % 4
        if kind == 0:
            keys[a:b] = np.sort(keys[a:b])
        elif kind == 1:
            keys[a:b] = np.sort(keys[a:b])[::-1]
        elif b > a:  # all equal but one, first or last
            keys[a:b] = keys[a]
            keys[a if kind == 2 else b - 1] ^= np.uint32(1) << np.uint32(rng.integers(0, 32))
    wk, wv = seg_oracle(keys, offs)
    with g.OneSweepSorter(max(int(offs[-1]), 16), 4, 4) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            tk = torch.from_numpy(keys.view(np.int32).copy()).cuda()
            tv = torch.arange(keys.size, dtype=torch.int32, device="cuda")
            s.segmented_sort(tk, torch.from_numpy(offs).cuda(), tv, max_segment_len=seg_len)
            assert np.array_equal(tk.cpu().numpy().view(np.uint32), wk), f"keys, rank_mode={mode}"
            assert np.array_equal(tv.cpu().numpy().view(np.uint32), wv), f"payloads, rank_mode={mode}"
