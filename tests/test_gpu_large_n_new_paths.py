"""Past 2^31 and 2^32 elements on the paths that compute element positions in their own code and came after
tests/test_gpu_large_n.py and tests/test_gpu_large_n_typed.py: the fused first pass of u32 keys-only sorts (DESIGN §4.12),
osb200_sort_segments and osb200_topk_rows.  A position cut to 32 bits anywhere there would go unnoticed at the sizes
their feature tests use.

- The fused first pass: at n = 2^32 - 2^20 - 3 keys the 256 regions of the alt buffer reach past element 2^32 (it falls in
  region 248), so the scatter, the gapped loads of the next pass, their re-reduction and the fallback all index past it.
  The keys are an affine permutation, key[i] = (A i + B) mod 2^32, whose sort is known without a sort (tests/bigcheck.py),
  and every output element is compared with it.
- Ragged segments of 32- and 64-bit keys whose positions pass 2^31 and 2^32 (byte offsets past 2^34), and segment ids past
  2^31 in the class lists, checked bit for bit against the numpy oracle of tests/test_gpu_sort_segments.py on windows
  framed by sentinels.
- Row top-k over batches past 2^31 and 2^32 keys, on the warp path and on the select path, with both in-place sorts of the
  [rows, k] result, checked against torch.sort(stable=True) of every row's radix image cut to k.

Inputs are generated on the device from fixed seeds (the segment windows, a few hundred thousand keys, on the host); no
n-sized array is copied to the host.  Each test computes the device memory it needs (at most about 40 GiB) and skips,
saying so, when the GPU has less free.  Every test name here contains "past_2pow": -m gpu -k "not past_2pow" leaves them
out of a quick run.  -m gpu"""
import numpy as np
import pytest
import torch

from tests import bigcheck as bc
from tests.test_fused_layout_cpu import TILE, WINDOW_N, fused_eligible, region_keys
from tests.test_gpu_large_n import release, require
from tests.test_gpu_large_n_typed import generate, rand64, rows16
from tests.test_gpu_rows import dev, host, typed_input
from tests.test_gpu_sort_segments import (GUARD, OK, SENTINEL_IDX, call, cap, framed_idx, framed_keys, offsets_of, oracle, same,
                                          sentinel_bits, shuffled_edges)

pytestmark = pytest.mark.gpu

GiB = 1 << 30
CHUNK = 1 << 26     # elements per generated chunk and per checked chunk
CHECK = 64 * CHUNK  # bytes: a bound on the temporaries of one checked chunk (int64 images, sort values and indices, gathers)
WARP_MAX = 256      # rows of at most this many keys are sorted one per warp (kRowWarpMaxLen)


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


# ---- 1. the fused first pass in the window past element 2^32 ---------------------------------------------------------------
A, B = 0x2545F491, 0x6A09E667


@pytest.mark.parametrize("case", ["kept", "abort_in_the_last_tiles", "classic", "f32_descending"])
def test_fused_first_pass_past_2pow32(g, case):
    """kept: the fused result stands.  abort_in_the_last_tiles: the last 32 full tiles sorted by their low byte put 2,048
    keys of one digit into a tile (more than T/16 = 1,024): the fused pass runs to there, aborts, and the classic path sorts.
    classic: the fused pass switched off.  f32_descending: typed keys whose radix image is the affine sequence."""
    n = WINDOW_N  # 2^32 - 2^20 - 3: 262,080 tiles, the last one ragged
    c = region_keys(n)
    assert fused_eligible(n) and 248 * c < (1 << 32) < 249 * c  # regions 249-255 start past element 2^32
    require(g, "fused u32 keys", n, 4, 0, 4 * n + CHECK, 0)
    typed = case == "f32_descending"

    def keys_of(r):  # the keys whose radix image (f32, descending) or bits (u32) are r
        return bc.from_radix32(r, "f", descending=True) if typed else bc.as_int32(r)

    t = torch.empty(n, dtype=torch.int32, device="cuda")
    for a in range(0, n, CHUNK):
        b = min(a + CHUNK, n)
        t[a:b] = keys_of(bc.affine_keys(A, B, a, b, device="cuda"))
    if case == "abort_in_the_last_tiles":
        lo = (n // TILE - 32) * TILE
        bc.sort_by_low_byte(t[lo:lo + 32 * TILE])
    s = g.OneSweepSorter(n, 4, 0)
    try:
        if case == "classic":
            s.set_option("fused_histogram", 0)
        if typed:
            s.sort_keys_typed(t.view(torch.float32), "f32", descending=True)
        else:
            s.sort_keys(t)
        kept, skip, passes = s.info("last_fused_kept"), s.info("last_skip_mask"), s.info("last_executed_passes")
    finally:
        torch.cuda.synchronize()
        s.close()
    print(f"\n{case}: last_fused_kept={kept} last_skip_mask={skip} last_executed_passes={passes}")
    assert kept == (1 if case in ("kept", "f32_descending") else 0)
    assert skip == 0 and passes == 4  # place 1 ran, through the gapped loads when the fused result stood
    gaps = bc.affine_gaps(A, B, n, device="cuda")
    try:
        for a in range(0, n, CHUNK):
            b = min(a + CHUNK, n)
            bc._require(t[a:b] == keys_of(bc.affine_sorted(gaps, a, b)), f"{case}: output differs from the sort", a)
    finally:
        del t, gaps
        release()


# ---- 2. ragged segments of 32- and 64-bit keys ---------------------------------------------------------------------------
FRAME = 1000  # sentinels before and after each window


def window(rng, t, first):
    """offsets of segments of every class edge, in a random order, led by one of the cap's length that starts at `first`"""
    L = np.concatenate([[cap(t)], shuffled_edges(rng, t, extra=40)])
    return offsets_of(L, start=first)


def framed_window(x, ix, rng, t, off):
    """writes random keys over [off[0], off[-1]) and sentinels over the FRAME positions on each side (indices: sentinels
    throughout); returns (lo, hi, bits) of the framed window"""
    lo, hi = int(off[0]) - FRAME, int(off[-1]) + FRAME
    bits = typed_input(rng, hi - lo, t)
    bits[:FRAME] = bits[-FRAME:] = sentinel_bits(t)
    x[lo:hi] = dev(bits, t)
    if ix is not None:
        ix[lo:hi] = SENTINEL_IDX - (1 << 32)
    return lo, hi, bits


def check_window(x, ix, lo, hi, off, bits, t, descending, base_idx, what):
    """keys (and indices, unless ix is None) of [lo, hi) against the oracle of the in-place sort of its segments"""
    want_k, want_i = oracle(bits, off - lo, hi - lo, cap(t), t, descending, bits, base_idx)
    same(host(x[lo:hi], t), want_k, f"{what}: keys")
    if ix is not None:
        same(ix[lo:hi].cpu().numpy().view(np.uint32), want_i, f"{what}: indices")
    return want_k, want_i


def test_segments32_past_2pow31_and_2pow32(g):
    """f32, descending, in place with indices: one window whose first segment straddles 2^31 and one whose first segment
    straddles 2^32, joined by one segment of about 2^31 keys, longer than max_segment_len, that must be left as it is; then
    the same buffer sorted again keys-only as u32, which must not write the indices"""
    t = "f32"
    n = (1 << 32) + (1 << 20)
    require(g, "f32 segments", 1, 4, 0, 8 * n + GiB, 0)  # keys and indices
    rng = np.random.default_rng(23)
    off1 = window(rng, t, (1 << 31) - cap(t) // 2)
    off2 = window(rng, t, (1 << 32) - cap(t) // 2)
    off = np.concatenate([off1, off2])  # [off1[-1], off2[0]): the long segment
    assert off1[0] < (1 << 31) < off1[1] and off2[0] < (1 << 32) < off2[1]
    assert off2[0] - off1[-1] > (1 << 31) - (1 << 20) and off2[-1] + FRAME <= n
    x = torch.empty(n, dtype=torch.float32, device="cuda")
    ix = torch.empty(n, dtype=torch.int32, device="cuda")
    frames = [(o,) + framed_window(x, ix, rng, t, o) for o in (off1, off2)]
    off_t = torch.from_numpy(off).cuda()
    sentinel_idx = np.full(max(hi - lo for _, lo, hi, _ in frames), SENTINEL_IDX, np.uint32)
    try:
        with g.OneSweepSorter(1 << 12, 4, 4) as s:
            assert call(s, x.data_ptr(), x.data_ptr(), ix.data_ptr(), n, off_t, off.size - 1, cap(t), t, True) == OK
            torch.cuda.synchronize()
            firsts = [check_window(x, ix, lo, hi, o, bits, t, True, sentinel_idx[:hi - lo], f"f32 window at {lo}")
                      for o, lo, hi, bits in frames]
            assert call(s, x.data_ptr(), x.data_ptr(), None, n, off_t, off.size - 1, cap("u32"), "u32", False) == OK
            torch.cuda.synchronize()
        for (o, lo, hi, _), (bits, idx) in zip(frames, firsts):
            check_window(x, None, lo, hi, o, bits, "u32", False, idx, f"u32 window at {lo}")
            same(ix[lo:hi].cpu().numpy().view(np.uint32), idx, f"u32 window at {lo}: indices of the keys-only sort")
    finally:
        del x, ix
        release()


def test_segments64_past_2pow31(g):
    """i64, ascending, in place with indices: a window whose first segment straddles 2^31, byte offsets past 2^34"""
    t = "i64"
    n = (1 << 31) + (1 << 20)
    require(g, "i64 segments", 1, 4, 0, 12 * n + GiB, 0)
    rng = np.random.default_rng(29)
    off = window(rng, t, (1 << 31) - cap(t) // 2)
    assert off[0] < (1 << 31) < off[1] and off[-1] + FRAME <= n
    x = torch.empty(n, dtype=torch.int64, device="cuda")
    ix = torch.empty(n, dtype=torch.int32, device="cuda")
    lo, hi, bits = framed_window(x, ix, rng, t, off)
    try:
        with g.OneSweepSorter(1 << 12, 4, 4) as s:
            assert call(s, x.data_ptr(), x.data_ptr(), ix.data_ptr(), n, torch.from_numpy(off).cuda(), off.size - 1, cap(t), t,
                        False) == OK
            torch.cuda.synchronize()
        check_window(x, ix, lo, hi, off, bits, t, False, np.full(hi - lo, SENTINEL_IDX, np.uint32), "i64 window")
    finally:
        del x, ix
        release()


def test_segment_ids_past_2pow31(g):
    """2^31 + 4,099 segments of 16-bit keys, all empty but the last few hundred, which cover every length class: their ids
    lie past 2^31 in the warp list and in the block list (stored from the list's far end, at positions past 2^31 too)"""
    t = "u16"
    num_segments = (1 << 31) + 4099
    rng = np.random.default_rng(31)
    tail = offsets_of(shuffled_edges(rng, t, extra=100))
    first = num_segments - (tail.size - 1)  # the first segment that is not [0, 0)
    n = int(tail[-1])
    assert first > 1 << 31
    # the offsets (16 GiB) and a workspace whose alt key buffer holds the class lists (one u32 per segment)
    require(g, f"{num_segments} segments", num_segments, 4, 0, 8 * (num_segments + 1), 0)
    off = torch.zeros(num_segments + 1, dtype=torch.int64, device="cuda")
    off[first:] = torch.from_numpy(tail).cuda()
    bits = typed_input(rng, n, t)
    src = framed_keys(bits, t)
    out = framed_keys(bits, t, np.full(n, sentinel_bits(t), dtype=bits.dtype))
    ix = framed_idx(n)
    try:
        with g.OneSweepSorter(num_segments, 4, 0) as s:
            assert call(s, src.ptr, out.ptr, ix.ptr, n, off, num_segments, cap(t), t, True) == OK
            torch.cuda.synchronize()
        want_k, want_i = oracle(bits, tail, n, cap(t), t, True, np.full(n, sentinel_bits(t), dtype=bits.dtype),
                                np.full(n, SENTINEL_IDX, np.uint32))
        gk, gi = out.host(), ix.host()
        same(gk[GUARD:-GUARD], want_k, "keys")
        same(gi[GUARD:-GUARD], want_i, "indices")
        for what, guard, fill in (("keys", gk, sentinel_bits(t)), ("indices", gi, SENTINEL_IDX)):
            same(np.concatenate([guard[:GUARD], guard[-GUARD:]]), np.full(2 * GUARD, fill, dtype=guard.dtype),
                 f"guards of the {what}")
        same(src.host()[GUARD:-GUARD], bits, "input modified")
    finally:
        del off, src, out, ix
        release()


# ---- 3. row top-k over batches past 2^31 and 2^32 keys ------------------------------------------------------------------------
def pooled(width, seed):
    """make(gen, m) for float keys of `width` (32 or 64) bits whose radix images are half uniform and half from a pool of 64
    values, 32 near the top and 32 near the bottom: the boundary of a row's k largest, and of its k smallest, falls among
    hundreds of equal keys"""
    pg = torch.Generator(device="cuda").manual_seed(seed)
    near = torch.randint(0, 1 << 20, (64,), generator=pg, device="cuda", dtype=torch.int64)
    top = (1 << width) - 1 if width == 32 else -1  # the largest image, in its container
    pool = torch.cat([top - near[:32], near[32:]])

    def make(gen, m):
        if width == 32:
            r = torch.randint(0, 1 << 32, (m,), generator=gen, device="cuda", dtype=torch.int64)
        else:
            r = rand64(gen, m)
        tied = torch.rand(m, generator=gen, device="cuda") < 0.5
        r = torch.where(tied, pool[torch.randint(0, 64, (m,), generator=gen, device="cuda")], r)
        return bc.from_radix32(r, "f") if width == 32 else bc.from_radix64(r, "f")

    return make


def topk_and_check(g, rows, row_len, dtype, key_type, seed, make, runs):
    """topk_rows for each (k, largest, sorted) of `runs`, checked against the stable sort of every row; the input must be
    left as it was"""
    x = torch.empty(rows, row_len, dtype=dtype, device="cuda")
    generate(x, seed, make)
    try:
        with g.OneSweepSorter(1, 4, 0) as s:
            for k, largest, srt in runs:
                vals, idx = s.topk_rows(x, k, key_type, largest, srt)
                torch.cuda.synchronize()
                assert vals.shape == idx.shape == (rows, k)
                bc.check_topk_rows(vals, idx, x, bc.key_radix(key_type, largest), k, srt, CHUNK)
                del vals, idx
        generate(x, seed, make, compare=True, what="top-k input")
    finally:
        del x
        release()


def test_topk_warp_path_past_2pow32(g):
    """bf16 rows of 4 keys: the input bases pass 2^32, the output bases pass 2^31 for k = 2 and 2^32 for k = 4"""
    rows, row_len = (1 << 30) + 3, 4
    assert row_len <= WARP_MAX  # one warp per row, the first k stored from the registers
    assert (rows - 1) * row_len > 1 << 32 and (rows - 1) * 2 > 1 << 31 and (rows - 1) * 4 > 1 << 32
    n = rows * row_len
    require(g, "bf16 rows of 4", 1, 4, 0, 2 * n + 6 * n + CHECK, 0)  # input; keys and indices of k = 4
    topk_and_check(g, rows, row_len, torch.bfloat16, "bf16", 91, rows16,
                   [(2, True, True), (2, False, True), (2, True, False), (4, True, True), (4, False, True)])


def test_topk_select_path_f32_past_2pow32(g):
    """f32 rows of 50,000 keys, beyond the 16,384 held in shared memory (the first levels read global memory), 85,900 rows:
    more than 2^32 keys.  k = 1,024 is sorted by topk_sort_kernel, k = 50 by topk_warp_kernel"""
    rows, row_len = 85_900, 50_000
    assert row_len > 16384 and rows * row_len > 1 << 32
    n = rows * row_len
    require(g, "f32 rows of 50,000", 1, 4, 0, 4 * n + CHECK, 0)
    topk_and_check(g, rows, row_len, torch.float32, "f32", 92, pooled(32, 93),
                   [(1024, True, True), (50, True, True), (50, False, True), (50, True, False)])


def test_topk_select_path_f64_past_2pow31(g):
    """f64 rows of 9,000 keys, beyond the 8,192 held in shared memory, 240,000 rows: more than 2^31 keys.  k = 300 is sorted
    by the 64-bit topk_sort_kernel"""
    rows, row_len = 240_000, 9_000
    assert row_len > 8192 and rows * row_len > 1 << 31
    n = rows * row_len
    require(g, "f64 rows of 9,000", 1, 4, 0, 8 * n + CHECK, 0)
    topk_and_check(g, rows, row_len, torch.float64, "f64", 94, pooled(64, 95), [(300, True, True), (300, False, False)])


def test_topk_output_past_2pow31(g):
    """u16, k = 16,384 of rows of 16,400 keys, 131,073 rows: the [rows, k] output that topk_sort_kernel sorts in place holds
    more than 2^31 elements"""
    rows, row_len, k = 131_073, 16_400, 16_384
    assert row_len > WARP_MAX and (rows - 1) * k >= 1 << 31
    n = rows * row_len
    require(g, "u16 top 16,384", 1, 4, 0, 2 * n + 6 * rows * k + CHECK, 0)
    topk_and_check(g, rows, row_len, torch.uint16, "u16", 96, rows16, [(k, False, True)])
