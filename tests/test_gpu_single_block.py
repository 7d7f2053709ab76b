"""The single-block shared-memory sort (segment_sort_kernel) in its instantiations: three geometries (256, 2,048 and 16,384
keys; 8,192 for 64-bit keys) for keys, pairs and 64-bit keys, the argsort form, each in both rank modes.  It runs every
osb200_segmented_sort_u32 call and every sort of at most one tile (n <= 16,384; 8,192 for 64-bit keys).

The cases: every geometry with segment lengths at the geometry boundaries; many more segments than the grid has blocks, so
that every block sorts several segments in the same shared memory; segments longer than max_segment_len, which must be
left as they are; keys whose radix image is all ones, which tie with the all-ones padding of the single-block kernel and
of the multi-kernel path's ragged last tile; 64-bit keys with ties in one word only; and segments at element offsets past
2^31 and 2^32.

Every comparison is element by element against a numpy stable sort of the radix key (tests.oraclelib.to_radix), with
payload = input index wherever the entry point takes payloads.  In-place sorts get a guard region after n, which must come
back unchanged.  The past-2^32 case needs about 46 GiB of free device memory and skips, saying so, when there is less;
-k "not past_2pow" leaves it out.  -m gpu"""
import gc

import numpy as np
import pytest
import torch

from tests.oraclelib import from_radix, to_radix

pytestmark = pytest.mark.gpu

GiB = 1 << 30
CAPS = (256, 2048, 16384)  # keys per geometry, 32-bit keys
KINDS = {"u32": "u", "i32": "i", "f32": "f", "u64": "u", "i64": "i", "f64": "f"}
GUARD = 1 << 16  # elements after n that an in-place sort must not write (more than any tile)


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def rank_modes(s):
    return [0, 1] if s.info("atomic_order_ok") else [1]


def dev(a):
    return torch.from_numpy(a.view(np.int32 if a.dtype == np.uint32 else np.int64).copy()).cuda()


def host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


def random_bits(rng, n, dtype=np.uint32):
    if dtype == np.uint32:
        return rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    return rng.integers(0, np.iinfo(np.uint64).max, n, dtype=np.uint64, endpoint=True)


# ---- segmented sort ----------------------------------------------------------------------------------------------------
def layout(lens, before=5, after=7):
    """offsets of segments of the given lengths, with `before` and `after` elements outside every segment"""
    offs = before + np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return offs, int(offs[-1]) + after


def seg_reference(keys, offs, max_len):
    """(keys, payloads) after a segmented sort of uint32 keys with payload = input index: one stable lexsort in which every
    segment of at most max_len keys is one group and every other element (outside the segments, or in a longer segment)
    is a group of its own, so it keeps its position"""
    n = keys.size
    lens = np.diff(offs)
    group = np.arange(n, dtype=np.int64)
    inside = group[offs[0]:offs[-1]]
    inside[:] = np.where(np.repeat(lens <= max_len, lens), np.repeat(offs[:-1], lens), inside)
    order = np.lexsort((keys, group))
    return keys[order], order.astype(np.uint32)


def check_segmented(s, keys, offs, max_len, what):
    """segmented_sort of the uint32 keys over offs, keys only and with payloads, in every rank mode of s"""
    wk, wv = seg_reference(keys, offs, max_len)
    to = torch.from_numpy(offs).cuda()
    for mode in rank_modes(s):
        s.set_option("rank_mode", mode)
        for pairs in (False, True):
            tk = dev(keys)
            tv = torch.arange(keys.size, dtype=torch.int32, device="cuda") if pairs else None
            s.segmented_sort(tk, to, tv, max_segment_len=max_len)
            tag = f"{what}, rank_mode={mode}, pairs={pairs}"
            assert np.array_equal(host(tk), wk), f"keys: {tag}"
            if pairs:
                assert np.array_equal(host(tv), wv), f"payloads: {tag}"


BOUNDARY_LENS = [0, 1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 16383, 16384]


@pytest.mark.parametrize("max_len", [2, 255, 256, 257, 2047, 2048, 2049, 16383, 16384])
def test_every_geometry(g, max_len):
    """max_segment_len picks the geometry; segments of every boundary length up to it and random ones, with full 32-bit
    keys, 8-bit keys (ties) and all-equal keys (the identity permutation)"""
    rng = np.random.default_rng(max_len)
    lens = np.array([x for x in BOUNDARY_LENS if x <= max_len] + [max_len] + list(rng.integers(0, max_len + 1, 24)))
    rng.shuffle(lens)
    offs, n = layout(lens)
    full = random_bits(rng, n)
    with g.OneSweepSorter(n, 4, 4) as s:
        check_segmented(s, full, offs, max_len, f"max_segment_len={max_len}, full keys")
        check_segmented(s, full & np.uint32(0xFF), offs, max_len, f"max_segment_len={max_len}, 8-bit keys")
        equal = np.full(n, 0x9E3779B9, dtype=np.uint32)
        assert np.array_equal(seg_reference(equal, offs, max_len)[1], np.arange(n))
        check_segmented(s, equal, offs, max_len, f"max_segment_len={max_len}, equal keys")


def test_tiny_segments_in_the_largest_geometry(g):
    """max_segment_len 16,384 with segments of at most 40 keys: the 16,384-key geometry, almost all of it padding"""
    rng = np.random.default_rng(40)
    lens = rng.integers(0, 41, 3000)
    offs, n = layout(lens)
    keys = random_bits(rng, n) & np.uint32(0xF00F)
    with g.OneSweepSorter(n, 4, 4) as s:
        check_segmented(s, keys, offs, 16384, "segments of <= 40 keys, max_segment_len=16384")


@pytest.mark.parametrize("max_len,count", [(256, 20000), (2048, 20000), (16384, 2000)])
def test_many_segments_per_block(g, max_len, count):
    """many more segments than the grid has blocks (8 per SM in the two small geometries, 2 in the largest): every block
    sorts several segments one after the other in the same shared memory"""
    rng = np.random.default_rng(count + max_len)
    lens = rng.integers(0, max_len + 1, count)
    offs, n = layout(lens)
    keys = random_bits(rng, n)
    tied = rng.random(n) < 0.5
    keys[tied] = random_bits(rng, 256)[rng.integers(0, 256, int(tied.sum()))]
    with g.OneSweepSorter(n, 4, 4) as s:
        blocks = s.info("sm_count") * (2 if max_len > 2048 else 8)
        assert count >= 4 * blocks, "fewer segments than intended per block"
        check_segmented(s, keys, offs, max_len, f"{count} segments of <= {max_len} keys")


@pytest.mark.parametrize("max_len,cap", [(200, 256), (1000, 2048), (5000, 16384)])
def test_segments_longer_than_max_segment_len_are_left_untouched(g, max_len, cap):
    """max_segment_len below the capacity of the geometry it selects: segments of up to max_len keys are sorted, longer
    ones (up to the capacity and at it) keep their keys and values bit for bit"""
    rng = np.random.default_rng(max_len)
    long = [max_len + 1, max_len + 2, cap - 1, cap] + list(rng.integers(max_len + 1, cap + 1, 8))
    short = [0, 1, 2, max_len - 1, max_len] + list(rng.integers(0, max_len + 1, 20))
    lens = np.array(long + short)
    rng.shuffle(lens)
    offs, n = layout(lens)
    keys = random_bits(rng, n)
    with g.OneSweepSorter(n, 4, 4) as s:
        check_segmented(s, keys, offs, max_len, f"max_segment_len={max_len}, full keys")
        check_segmented(s, keys & np.uint32(0xFF), offs, max_len, f"max_segment_len={max_len}, 8-bit keys")


# ---- keys that sort like the padding -----------------------------------------------------------------------------------
def all_ones(dtype):
    return np.array([np.iinfo(dtype).max], dtype=dtype)


def padlike_mask(rng, n):
    """about half of n positions: a run at the end (the tail of the last tile, next to the padding), a run in the middle
    and single positions scattered in between"""
    hit = rng.random(n) < 0.3
    run = max(1, n // 8)
    hit[n - run:] = True
    hit[n // 3:n // 3 + run] = True
    return hit


def padlike_bits(rng, n, like, dtype=np.uint32):
    """n random keys of which about half (padlike_mask) are `like`"""
    bits = random_bits(rng, n, dtype)
    bits[padlike_mask(rng, n)] = like
    return bits


def run_entry(s, entry, key_type, descending, bits, rng, bit_range=None, pairs=False):
    """one call of `entry` on the keys `bits`, compared element by element with numpy's stable sort (payload = input
    index).  In-place sorts run on buffers of n + GUARD elements; the guard must come back unchanged."""
    n, dt = bits.size, bits.dtype
    if bit_range is not None:
        b, e = bit_range
        mask = (1 << (e - b)) - 1
        radix = (bits >> dt.type(b)) & dt.type(mask)
        what = f"{entry} bits [{b}, {e}) pairs={pairs} n={n}"
    else:
        radix = to_radix(bits, KINDS[key_type], descending)
        what = f"{entry} {key_type} descending={descending} n={n}"
    order = np.argsort(radix, kind="stable")
    if entry == "argsort":
        kin = dev(bits)
        before = kin.clone()
        out, idx = s.argsort(kin, key_type, descending)
        torch.cuda.synchronize()
        assert torch.equal(kin, before), f"the input was modified: {what}"
        assert np.array_equal(host(idx), order), f"indices: {what}"
        assert np.array_equal(host(out), bits[order]), f"keys: {what}"
        return
    guard = random_bits(rng, GUARD, dt)
    tk = dev(np.concatenate([bits, guard]))
    pairs = pairs or entry in ("sort_pairs", "sort_pairs_typed")
    if pairs:
        vguard = random_bits(rng, GUARD)
        tv = dev(np.concatenate([np.arange(n, dtype=np.uint32), vguard]))
    if entry == "sort_pairs":
        s.sort_pairs(tk, tv, n=n)
    elif entry == "sort_pairs_typed":
        s.sort_pairs_typed(tk, tv, key_type, descending, n=n)
    elif entry == "sort_keys":
        s.sort_keys(tk, n=n)
    elif entry == "sort_keys_typed":
        s.sort_keys_typed(tk, key_type, descending, n=n)
    elif entry == "sort_bits":
        s.sort_bits(tk, b, e, tv if pairs else None, n=n)
    got = host(tk, dt)
    assert np.array_equal(got[:n], bits[order]), f"keys: {what}"
    assert np.array_equal(got[n:], guard), f"keys written past n: {what}"
    if pairs:
        gv = host(tv)
        assert np.array_equal(gv[:n], order.astype(np.uint32)), f"payloads: {what}"
        assert np.array_equal(gv[n:], vguard), f"payloads written past n: {what}"


PAD_SIZES = [3, 255, 257, 2047, 2049, 16383, 16384]


def sweep(s, body):
    """body(n) for every rank mode: on the single-block path at PAD_SIZES, then on the multi-kernel path at the same sizes
    and at 3 tiles + 17 keys (a ragged last tile)"""
    ragged = 3 * s.info("tile_keys") + 17
    for mode in rank_modes(s):
        s.set_option("rank_mode", mode)
        for small in (1, 0):
            s.set_option("small_path", small)
            for n in PAD_SIZES + ([ragged] if not small else []):
                body(n)
    s.set_option("small_path", 1)


PADLIKE = [("sort_pairs", "u32", (False,)), ("sort_pairs_typed", "i32", (False, True)),
           ("sort_pairs_typed", "f32", (False, True)), ("argsort", "u32", (False, True)), ("argsort", "i32", (False, True)),
           ("argsort", "f32", (False, True)), ("sort_keys_typed", "i64", (False, True)),
           ("sort_keys_typed", "f64", (False, True))]


@pytest.mark.parametrize("entry,key_type,orders", PADLIKE, ids=[f"{e}-{k}" for e, k, _ in PADLIKE])
def test_keys_that_sort_like_the_padding(g, entry, key_type, orders):
    """about half the keys have the all-ones radix image of the requested type and order (u32 0xFFFFFFFF, INT_MAX
    ascending / INT_MIN descending, the all-ones-payload NaN of the sign that sorts last, and their 64-bit analogues):
    they tie with the padding, and must rank before it and all be stored"""
    wide = key_type.endswith("64")
    dt = np.uint64 if wide else np.uint32
    rng = np.random.default_rng(PADLIKE.index((entry, key_type, orders)))
    with g.OneSweepSorter(max(PAD_SIZES) + 4 * 16384 + GUARD, 8 if wide else 4, 0 if wide else 4) as s:
        for descending in orders:
            like = from_radix(all_ones(dt), KINDS[key_type], descending)[0]
            sweep(s, lambda n: run_entry(s, entry, key_type, descending, padlike_bits(rng, n, like, dt), rng))


@pytest.mark.parametrize("pairs", [False, True])
def test_sort_bits_keys_that_sort_like_the_padding(g, pairs):
    """sort_bits where about half the keys have all ones in the bit range and the bits outside it vary; ranges whose last
    digit has at most 5 bits run the few-bins scatter, which takes the padding out of the pad digit's run; a range that
    starts at bit 0 also sees the lowest bit of the padding"""
    rng = np.random.default_rng(70 + pairs)
    with g.OneSweepSorter(max(PAD_SIZES) + 4 * 16384 + GUARD, 4, 4 if pairs else 0) as s:
        for b, e in [(0, 13), (3, 16), (8, 12), (31, 32), (4, 28)]:
            ones = np.uint32(((1 << (e - b)) - 1) << b)

            def body(n):
                bits = random_bits(rng, n)
                bits[padlike_mask(rng, n)] |= ones  # the range all ones, the other bits random
                run_entry(s, "sort_bits", None, False, bits, rng, bit_range=(b, e), pairs=pairs)

            sweep(s, body)


def test_keys_that_sort_like_the_padding_in_hot_passes(g):
    """n = 2^22 + 4099 with about half the keys like the padding: the padding's digit is the hot bin of every pass (the
    HOT instantiation), and the last tile is ragged"""
    n = (1 << 22) + 4099
    rng = np.random.default_rng(80)
    with g.OneSweepSorter(n + GUARD, 4, 4) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for entry, key_type, descending in (("sort_pairs", "u32", False), ("argsort", "f32", True),
                                                ("argsort", "i32", False)):
                like = from_radix(all_ones(np.uint32), KINDS[key_type], descending)[0]
                run_entry(s, entry, key_type, descending, padlike_bits(rng, n, like), rng)
                assert s.info("last_hot_mask") != 0, f"{entry} {key_type}: no hot pass"


@pytest.mark.parametrize("max_len", CAPS)
def test_segments_of_keys_like_the_padding(g, max_len):
    """segments made entirely of 0xFFFFFFFF next to segments in which about half the keys are, in every geometry"""
    rng = np.random.default_rng(90 + max_len)
    lens = np.array([max_len, max_len - 1, 1, 2, 33] + list(rng.integers(0, max_len + 1, 40)))
    offs, n = layout(lens)
    keys = padlike_bits(rng, n, np.uint32(0xFFFFFFFF))
    for i in range(0, lens.size, 2):
        keys[offs[i]:offs[i + 1]] = 0xFFFFFFFF
    with g.OneSweepSorter(n, 4, 4) as s:
        check_segmented(s, keys, offs, max_len, f"max_segment_len={max_len}, keys like the padding")


# ---- 64-bit keys on the single-block path ------------------------------------------------------------------------------
N64 = [2, 255, 256, 257, 2047, 2048, 2049, 8191, 8192]


def keys64(rng, n, ties):
    """random 64-bit keys; "high" / "low": that word is drawn from 16 values, the other one is random"""
    hi, lo = random_bits(rng, n).astype(np.uint64), random_bits(rng, n).astype(np.uint64)
    pool = random_bits(rng, 16).astype(np.uint64)
    if ties == "high":
        hi = pool[rng.integers(0, 16, n)]
    elif ties == "low":
        lo = pool[rng.integers(0, 16, n)]
    return (hi << np.uint64(32)) | lo


@pytest.mark.parametrize("key_type", ["u64", "i64", "f64"])
def test_u64_single_block(g, key_type):
    rng = np.random.default_rng(["u64", "i64", "f64"].index(key_type) + 100)
    with g.OneSweepSorter(8192, 8, 0) as s:
        assert s.info("small_path_max_n") == 8192
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for n in N64:
                for ties in ("none", "high", "low"):
                    if key_type == "u64":
                        run_entry(s, "sort_keys", "u64", False, keys64(rng, n, ties), rng)
                    else:
                        for descending in (False, True):
                            run_entry(s, "sort_keys_typed", key_type, descending, keys64(rng, n, ties), rng)


def test_u64_sort_bits_single_block(g):
    rng = np.random.default_rng(110)
    with g.OneSweepSorter(8192, 8, 0) as s:
        for mode in rank_modes(s):
            s.set_option("rank_mode", mode)
            for n in N64:
                for bit_range in [(0, 64), (17, 49), (60, 64), (7, 8)]:
                    run_entry(s, "sort_bits", None, False, keys64(rng, n, "high"), rng, bit_range=bit_range)


# ---- segments past 2^31 and 2^32 ---------------------------------------------------------------------------------------
CHUNK = 1 << 28  # elements per torch op


def pattern(a, b, salt):
    """int64 words in [0, 2^32), a hash of the element index: the buffers' contents, regenerated for the check"""
    h = (torch.arange(a, b, dtype=torch.int64, device="cuda") * 0x9E3779B1 + salt) & 0xFFFFFFFF
    h = ((h ^ (h >> 15)) * 0x2C1B3C6D) & 0xFFFFFFFF
    return h ^ (h >> 12)


def as_i32(h):
    return (h - ((h >> 31) << 32)).to(torch.int32)


def key_words(a, b):
    return as_i32(pattern(a, b, 7) & 0xF0F0F00F)  # 4,096 values spread over the four bytes: ties in every segment


def value_words(a, b):
    return as_i32(torch.arange(a, b, dtype=torch.int64, device="cuda") & 0xFFFFFFFF)


def test_segments_past_2pow31_and_2pow32(g):
    """one buffer of 2^32 + 2^20 keys and one of values; segments that straddle element offsets 2^31 and 2^32 and that
    sit just past them, separated by segments longer than max_segment_len.  The sorted segments are compared exactly, and
    every other element with the index pattern it was filled with"""
    A, B = 1 << 31, 1 << 32
    total = B + (1 << 20)
    offs = np.array([A - 9000, A + 1, A + 16385, B - 16383, B + 1, B + 5001, B + 5003, total - 50], np.int64)
    gc.collect()
    torch.cuda.empty_cache()
    need = 8 * total + 12 * GiB  # keys and values, plus the int64 temporaries of one chunk of the fill and the check
    free, _ = torch.cuda.mem_get_info()
    if free < need + 4 * GiB:
        pytest.skip(f"needs {need / GiB:.1f} GiB (+4 GiB headroom), {free / GiB:.1f} GiB free")
    keys = torch.empty(total, dtype=torch.int32, device="cuda")
    vals = torch.empty(total, dtype=torch.int32, device="cuda")
    for a in range(0, total, CHUNK):
        b = min(a + CHUNK, total)
        keys[a:b] = key_words(a, b)
        vals[a:b] = value_words(a, b)
    sorted_segs = {}
    for lo, hi in zip(offs[:-1].tolist(), offs[1:].tolist()):
        if hi - lo <= 16384:
            k = key_words(lo, hi).cpu().numpy().view(np.uint32)
            order = np.argsort(k, kind="stable")
            sorted_segs[(lo, hi)] = (k[order], ((lo + order) & 0xFFFFFFFF).astype(np.uint32))
    with g.OneSweepSorter(1 << 16, 4, 4) as s:
        s.segmented_sort(keys, torch.from_numpy(offs).cuda(), vals, max_segment_len=16384)
        torch.cuda.synchronize()
    for (lo, hi), (wk, wv) in sorted_segs.items():
        assert np.array_equal(host(keys[lo:hi]), wk), f"keys of segment [{lo}, {hi})"
        assert np.array_equal(host(vals[lo:hi]), wv), f"values of segment [{lo}, {hi})"
    for a in range(0, total, CHUNK):
        b = min(a + CHUNK, total)
        wk, wv = key_words(a, b), value_words(a, b)
        for (lo, hi), (sk, sv) in sorted_segs.items():
            x, y = max(lo, a), min(hi, b)
            if x < y:
                wk[x - a:y - a] = torch.from_numpy(sk[x - lo:y - lo].view(np.int32)).cuda()
                wv[x - a:y - a] = torch.from_numpy(sv[x - lo:y - lo].view(np.int32)).cuda()
        assert torch.equal(keys[a:b], wk), f"keys in [{a}, {b})"
        assert torch.equal(vals[a:b], wv), f"values in [{a}, {b})"
        del wk, wv
    del keys, vals
    gc.collect()
    torch.cuda.empty_cache()
