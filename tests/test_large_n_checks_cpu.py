"""The chunked checkers of tests/bigcheck.py, on CPU tensors: their torch radix images equal the numpy ones the other tests
use, they accept the stable sort, and they reject each way a large sort could be subtly wrong -- payloads of equal keys
swapped, a payload off by 2^32 or past n, a key changed, an inversion exactly at a chunk border, a value replaced by its
neighbour (still sorted, but not a permutation), and a row whose indices are unstable.  The affine permutation's known
sort equals np.sort at a small modulus, and the top-k checker names the first bad row of each planted defect: a swapped
pair, a tie taken at a higher position, an index off by one, a key that is not src[idx], an unsorted output passed as
sorted and a pair missing from an unsorted output.  No GPU needed."""
import numpy as np
import pytest
import torch

from tests import bigcheck as bc
from tests.oraclelib import from_radix, to_radix
from tests.test_gpu_keys16 import from_radix16 as np_from_radix16
from tests.test_gpu_keys16 import radix16 as np_radix16
from tests.test_gpu_keys16 import specials as specials16
from tests.test_gpu_pairs64 import specials as specials64

CHUNK = 64
TYPES64 = ["u64", "i64", "f64"]
TYPES16 = ["u16", "i16", "f16", "bf16"]


def np_radix(bits, key_type, descending):
    if key_type in TYPES64:
        return to_radix(bits, key_type[0], descending)
    return np_radix16(bits, key_type, descending)


def as_torch(bits):
    """uint16 / uint64 numpy bits as an int16 / int64 tensor"""
    return torch.from_numpy(bits.view(np.int16 if bits.dtype == np.uint16 else np.int64).copy())


def random_bits(rng, n, key_type):
    """random patterns, a third of them from 8 values (runs of equal keys); floats contain every special value"""
    if key_type in TYPES64:
        bits, sp = rng.integers(0, 1 << 64, n, dtype=np.uint64), specials64()
    else:
        bits, sp = rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16), specials16(key_type)
    tied = rng.random(n) < 0.35
    bits[tied] = bits[rng.integers(0, 8, int(tied.sum()))]
    if key_type in ("f16", "bf16", "f64"):
        bits[rng.choice(n, sp.size, replace=False)] = sp
    return bits


# ---- radix images --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("key_type", TYPES64 + TYPES16)
def test_radix_images_match_numpy(key_type, descending):
    rng = np.random.default_rng(1)
    if key_type in TYPES64:
        bits = np.concatenate([rng.integers(0, 1 << 64, 4096, dtype=np.uint64), specials64(),
                               np.array([0, 1, 1 << 63, (1 << 64) - 1], dtype=np.uint64)])
        got = bc.to_radix64(as_torch(bits), key_type[0], descending)
        assert got.dtype == torch.int64
        np.testing.assert_array_equal(got.numpy().view(np.uint64), to_radix(bits, key_type[0], descending))
        back = bc.from_radix64(got, key_type[0], descending)
        np.testing.assert_array_equal(back.numpy().view(np.uint64), bits)
        np.testing.assert_array_equal(back.numpy().view(np.uint64),
                                      from_radix(to_radix(bits, key_type[0], descending), key_type[0], descending))
    else:
        bits = np.concatenate([np.arange(1 << 16, dtype=np.uint32).astype(np.uint16),  # every pattern, specials included
                               specials16("f16"), specials16("bf16")])
        got = bc.radix16(as_torch(bits), key_type, descending)
        assert got.dtype == torch.int32 and int(got.min()) >= 0 and int(got.max()) < (1 << 16)
        want = np_radix16(bits, key_type, descending)
        np.testing.assert_array_equal(got.numpy(), want.astype(np.int32))
        back = bc.from_radix16(got, key_type, descending)
        assert back.dtype == torch.int16
        np.testing.assert_array_equal(back.numpy().view(np.uint16), bits)
        np.testing.assert_array_equal(back.numpy().view(np.uint16), np_from_radix16(want, key_type, descending))


@pytest.mark.parametrize("key_type", TYPES64 + TYPES16)
def test_ordered_radix_sorts_like_numpy(key_type):
    """ordered(radix image) sorted as a signed tensor gives numpy's stable order of the unsigned image"""
    rng = np.random.default_rng(2)
    bits = random_bits(rng, 5000, key_type)
    for descending in (False, True):
        want = np.argsort(np_radix(bits, key_type, descending), kind="stable")
        got = torch.sort(bc.ordered(bc.key_radix(key_type, descending)(as_torch(bits))), stable=True).indices
        np.testing.assert_array_equal(got.numpy(), want)


# ---- sorted with payload = position --------------------------------------------------------------------------------------
def pairs_case(key_type, descending, n=1000, payload_dtype=torch.int32):
    rng = np.random.default_rng(3)
    bits = random_bits(rng, n, key_type)
    order = np.argsort(np_radix(bits, key_type, descending), kind="stable")
    return as_torch(bits), as_torch(bits[order]), torch.from_numpy(order).to(payload_dtype)


def first_tie(out):
    return int(torch.nonzero(out[1:] == out[:-1])[0, 0])


def border_with_distinct_neighbours(out, chunk):
    c = next(c for c in range(chunk, out.numel(), chunk) if out[c - 1] != out[c])
    return c


@pytest.mark.parametrize("payload_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("key_type,descending", [("f64", True), ("i64", False), ("u64", True), ("i16", False),
                                                 ("bf16", True), ("f16", False)])
def test_check_sorted_by_position(key_type, descending, payload_dtype):
    radix = bc.key_radix(key_type, descending)
    src, out, pay = pairs_case(key_type, descending, payload_dtype=payload_dtype)
    n = src.numel()
    bc.check_sorted_by_position(out, pay, src, radix, CHUNK)
    bc.check_sorted_by_position(out, pay, src, radix, n)  # one chunk
    bc.check_sorted_by_position(out, pay, src, radix, 1)  # one element per chunk

    def rejects(o, p, match):
        with pytest.raises(AssertionError, match=match):
            bc.check_sorted_by_position(o, p, src, radix, CHUNK)

    i = first_tie(out)  # two equal keys with their payloads swapped
    p = pay.clone()
    p[i], p[i + 1] = pay[i + 1], pay[i]
    rejects(out, p, f"payloads do not ascend inside a run of equal keys: first at output element {i}")
    for bad in (n, (1 << 32) - 1):  # a payload past n (as uint32 in an int32 container)
        p = pay.clone()
        p[77] = bad if payload_dtype == torch.int64 or bad < (1 << 31) else bad - (1 << 32)
        rejects(out, p, "payload outside")
    if payload_dtype == torch.int64:  # a payload plus 2^32: a position truncated to 32 bits the other way round
        p = pay.clone()
        p[500] += 1 << 32
        rejects(out, p, "payload outside")
    o = out.clone()  # one key changed
    o[300] ^= 1
    rejects(o, pay, None)
    c = border_with_distinct_neighbours(out, CHUNK)  # an inversion exactly at a chunk border, keys and payloads moved
    o, p = out.clone(), pay.clone()
    o[c - 1], o[c] = out[c], out[c - 1]
    p[c - 1], p[c] = pay[c], pay[c - 1]
    rejects(o, p, f"radix image descends: first at output element {c - 1}")
    j = border_with_distinct_neighbours(out, 7)  # a key replaced by its neighbour: still sorted
    o = out.clone()
    o[j - 1] = out[j]
    rejects(o, pay, rf"src\[payload\] != out: first at output element {j - 1}")


def test_positions_read_int32_as_unsigned():
    p = torch.tensor([0, -1, -(1 << 31), (1 << 31) - 1], dtype=torch.int32)
    assert bc.positions(p).tolist() == [0, (1 << 32) - 1, 1 << 31, (1 << 31) - 1]
    assert bc.positions(torch.tensor([1 << 32], dtype=torch.int64)).tolist() == [1 << 32]  # int64: as they are


# ---- 16-bit keys only: order and histogram -------------------------------------------------------------------------------
@pytest.mark.parametrize("key_type,descending", [("bf16", True), ("f16", False), ("i16", False), ("u16", True)])
def test_check_sorted_keys16(key_type, descending):
    radix = bc.key_radix(key_type, descending)
    src, out, _ = pairs_case(key_type, descending, n=3000)
    bc.check_sorted_keys16(out, src, radix, CHUNK)
    bc.check_sorted_keys16(out, src, radix, src.numel())

    def rejects(o, match):
        with pytest.raises(AssertionError, match=match):
            bc.check_sorted_keys16(o, src, radix, CHUNK)

    o = out.clone()  # one key changed
    o[1234] ^= 1
    rejects(o, None)
    c = border_with_distinct_neighbours(out, CHUNK)  # an inversion exactly at a chunk border: the same histogram
    o = out.clone()
    o[c - 1], o[c] = out[c], out[c - 1]
    rejects(o, f"radix image descends: first at output element {c - 1}")
    j = border_with_distinct_neighbours(out, 5)  # a value replaced by its neighbour: still sorted
    o = out.clone()
    o[j - 1] = out[j]
    assert bool((bc.ordered(radix(o))[1:] >= bc.ordered(radix(o))[:-1]).all())
    rejects(o, "radix value .* in the input")


# ---- rows ----------------------------------------------------------------------------------------------------------------
def rows_case(key_type, descending, rows, row_len):
    rng = np.random.default_rng(4)
    bits = random_bits(rng, rows * row_len, key_type).reshape(rows, row_len)
    order = np.argsort(np_radix(bits, key_type, descending), axis=-1, kind="stable")
    out = np.take_along_axis(bits, order, axis=-1)
    return as_torch(bits), as_torch(out), torch.from_numpy(order.astype(np.int32))


@pytest.mark.parametrize("key_type,descending", [("bf16", True), ("f16", False), ("u16", False), ("f64", True),
                                                 ("i64", False)])
@pytest.mark.parametrize("row_len", [5, 200])
def test_check_rows(key_type, descending, row_len):
    radix = bc.key_radix(key_type, descending)
    rows = 3 * CHUNK // row_len + 7 if row_len < CHUNK else 9
    src, out, idx = rows_case(key_type, descending, rows, row_len)
    bc.check_rows(out, idx, src, radix, CHUNK)
    bc.check_rows(out, None, src, radix, CHUNK)
    bc.check_rows(out, idx, src, radix, 1)  # one row per step
    step = max(1, CHUNK // row_len)

    def rejects(o, i, match):
        with pytest.raises(AssertionError, match=match):
            bc.check_rows(o, i, src, radix, CHUNK)

    r = next(r for r in range(rows) if bool((out[r, 1:] == out[r, :-1]).any()))  # a row whose indices are unstable
    c = int(torch.nonzero(out[r, 1:] == out[r, :-1])[0, 0])
    i = idx.clone()
    i[r, c], i[r, c + 1] = idx[r, c + 1], idx[r, c]
    rejects(out, i, f"indices differ .*: first at output row {r}, column {c}")
    o = out.clone()  # one key changed
    o[rows - 1, row_len // 2] ^= 1
    rejects(o, idx, f"keys differ .*: first at output row {rows - 1}")
    rejects(o, None, f"keys differ .*: first at output row {rows - 1}")
    o, fo = out.clone(), out.reshape(-1)  # an inversion exactly at the border of two steps: last and first key swapped
    b = step * row_len
    o.reshape(-1)[b - 1], o.reshape(-1)[b] = fo[b], fo[b - 1]
    if fo[b - 1] != fo[b]:
        rejects(o, idx, f"keys differ .*: first at output row {step - 1}, column {row_len - 1}")
    r = next(r for r in range(rows) if bool((out[r, 1:] != out[r, :-1]).any()))  # a key replaced by its neighbour
    c = int(torch.nonzero(out[r, 1:] != out[r, :-1])[0, 0])
    o = out.clone()
    o[r, c] = out[r, c + 1]
    rejects(o, idx, f"keys differ .*: first at output row {r}, column {c}")
    rejects(out[:-1], idx[:-1], "shapes")


# ---- 32-bit radix images -------------------------------------------------------------------------------------------------
SPECIALS32 = np.array([0, 1, 0x7FFFFFFF, 0x80000000, 0x80000001, 0xFFFFFFFF, 0x7F800000, 0xFF800000, 0x7FC00000,
                       0xFFC00000, 0x7F800001, 0xFF800001, 0x00000001, 0x80000001, 0x3F800000, 0xBF800000], dtype=np.uint32)


@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("kind", ["u", "i", "f"])
def test_radix32_images_match_numpy(kind, descending):
    """NaNs of both signs, +-0, +-inf and the extremes of every kind included"""
    rng = np.random.default_rng(5)
    bits = np.concatenate([rng.integers(0, 1 << 32, 4096, dtype=np.uint64).astype(np.uint32), SPECIALS32])
    got = bc.to_radix32(torch.from_numpy(bits.view(np.int32).copy()), kind, descending)
    assert got.dtype == torch.int64 and int(got.min()) >= 0 and int(got.max()) <= 0xFFFFFFFF
    want = to_radix(bits, kind, descending)
    np.testing.assert_array_equal(got.numpy().astype(np.uint32), want)
    back = bc.from_radix32(got, kind, descending)
    assert back.dtype == torch.int32
    np.testing.assert_array_equal(back.numpy().view(np.uint32), bits)
    back = bc.from_radix32(torch.from_numpy(want.astype(np.int64)), kind, descending)
    np.testing.assert_array_equal(back.numpy().view(np.uint32), from_radix(want, kind, descending))
    # the images sort like numpy's, through ordered() and through key_radix
    order = torch.sort(bc.ordered(bc.key_radix(kind + "32", descending)(torch.from_numpy(bits.view(np.int32).copy()))),
                       stable=True).indices
    np.testing.assert_array_equal(order.numpy(), np.argsort(want, kind="stable"))


# ---- the affine permutation's sort -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", [False, True])
@pytest.mark.parametrize("a,b", [(0x2545F491, 0x9E3779B9), (1, 0), (0x7FFFFFFF, 12345)])
def test_affine_sorted_is_the_sort(a, b, window):
    """at modulus 2^20 with n = 2^20 - 37 (37 values left out), with and without a window of keys sorted by their low byte"""
    bits, n = 20, (1 << 20) - 37
    keys = bc.affine_keys(a, b, 0, n, bits)
    assert torch.unique(keys).numel() == n
    assert bool((torch.bincount((keys[:n // 256 * 256] & 0xFF).reshape(-1, 256)[7], minlength=256) == 1).all())
    if window:
        lo, hi = 8192, 8192 + 4096
        bc.sort_by_low_byte(keys[lo:hi])
        assert bool((keys[lo:lo + 16] & 0xFF == 0).all()) and bool((keys[hi - 16:hi] & 0xFF == 255).all())
        assert torch.equal(torch.sort(keys).values, torch.sort(bc.affine_keys(a, b, 0, n, bits)).values)
    gaps = bc.affine_gaps(a, b, n, bits)
    assert gaps.numel() == 37 and bool((gaps[1:] >= gaps[:-1]).all())
    want = np.sort(keys.numpy())
    np.testing.assert_array_equal(bc.affine_sorted(gaps, 0, n).numpy(), want)
    for lo, hi in ((0, 1), (1000, 5000), (n - 77, n)):  # any chunk
        np.testing.assert_array_equal(bc.affine_sorted(gaps, lo, hi).numpy(), want[lo:hi])


def test_affine_gaps_names_the_left_out_values():
    a, b, bits, n = 0x2545F491, 77, 12, 4000
    gaps = bc.affine_gaps(a, b, n, bits)
    left_out = np.setdiff1d(np.arange(1 << bits), bc.affine_keys(a, b, 0, n, bits).numpy())
    np.testing.assert_array_equal(gaps.numpy() + np.arange(left_out.size), left_out)


# ---- row top-k -----------------------------------------------------------------------------------------------------------
def topk_case(key_type, largest, rows, row_len, k, seed=6):
    """(src, vals, idx) of the stable top k, sorted; a third of the keys come from 8 values, and every row has equal keys on
    both sides of its boundary"""
    rng = np.random.default_rng(seed)
    if key_type == "f32":
        bits = rng.integers(0, 1 << 32, rows * row_len, dtype=np.uint64).astype(np.uint32)
        tied = rng.random(bits.size) < 0.35
        bits[tied] = bits[rng.integers(0, 8, int(tied.sum()))]
        bits[rng.choice(bits.size, SPECIALS32.size, replace=False)] = SPECIALS32
    else:
        bits = random_bits(rng, rows * row_len, key_type)

    def image(bits):
        return to_radix(bits, "f", largest) if key_type == "f32" else np_radix(bits, key_type, largest)

    # a tie across the boundary of every row: the first key left out becomes a copy of the last one taken
    b2 = bits.reshape(rows, row_len)
    order = np.argsort(image(bits).reshape(rows, row_len), axis=-1, kind="stable")
    b2[np.arange(rows), order[:, k]] = b2[np.arange(rows), order[:, k - 1]]
    order = np.argsort(image(bits).reshape(rows, row_len), axis=-1, kind="stable")[:, :k]
    src = (torch.from_numpy(bits.view(np.int32).copy()) if key_type == "f32" else as_torch(bits)).reshape(rows, row_len)
    vals = torch.gather(src, 1, torch.from_numpy(order))
    return src, vals, torch.from_numpy(order.astype(np.int32))


def shuffled_rows(vals, idx, seed=7):
    """every row's pairs in another order (the same one for keys and positions)"""
    perm = torch.argsort(torch.from_numpy(np.random.default_rng(seed).random(tuple(idx.shape))), dim=-1)
    return torch.gather(vals, 1, perm), torch.gather(idx, 1, perm)


@pytest.mark.parametrize("key_type,largest", [("f32", True), ("f32", False), ("bf16", True), ("u16", False),
                                              ("f64", True), ("i64", False)])
@pytest.mark.parametrize("row_len,k", [(4, 2), (300, 50)])
def test_check_topk_rows(key_type, largest, row_len, k):
    radix = bc.key_radix(key_type, largest)
    rows = 3 * CHUNK // row_len + 7 if row_len < CHUNK else 9
    src, vals, idx = topk_case(key_type, largest, rows, row_len, k)
    uv, ui = shuffled_rows(vals, idx)
    for chunk in (CHUNK, 1, rows * row_len):
        bc.check_topk_rows(vals, idx, src, radix, k, True, chunk)
        bc.check_topk_rows(vals, idx, src, radix, k, False, chunk)
        bc.check_topk_rows(uv, ui, src, radix, k, False, chunk)
    r0 = rows - 2  # the planted defects go into a row of a later step than the first

    def rejects(v, i, srt, match):
        with pytest.raises(AssertionError, match=match):
            bc.check_topk_rows(v, i, src, radix, k, srt, CHUNK)

    bits = bc.bits_of(src)
    img = bc.ordered(radix(src))
    # a swapped pair: two columns of different keys exchanged, keys and positions
    vb = bc.bits_of(vals)
    r = next(r for r in range(r0, rows) if bool((vb[r, 1:] != vb[r, :-1]).any()))
    c = int(torch.nonzero(vb[r, 1:] != vb[r, :-1])[0, 0])
    v, i = vals.clone(), idx.clone()
    v[r, c], v[r, c + 1] = vals[r, c + 1], vals[r, c]
    i[r, c], i[r, c + 1] = idx[r, c + 1], idx[r, c]
    rejects(v, i, True, f"positions differ .*: first at output row {r}, column {c}")
    # a tie taken at a higher position: the last key taken has an equal key behind the first k, which replaces it
    found = None
    for r in range(r0, rows):
        last = img[r, int(idx[r, k - 1])]
        later = torch.nonzero(img[r] == last).reshape(-1)
        later = later[later > int(idx[r, k - 1])]
        taken = set(idx[r].tolist())
        later = [p for p in later.tolist() if p not in taken]
        if later:
            found = (r, later[0])
            break
    assert found is not None, "no row of the last step has a tie at its boundary"
    r, p = found
    for srt, (v0, i0) in ((True, (vals, idx)), (False, (uv, ui))):
        v, i = v0.clone(), i0.clone()
        c = int(torch.nonzero(i0[r] == idx[r, k - 1])[0, 0])
        i[r, c] = p
        bc.bits_of(v)[r, c] = bits[r, p]
        rejects(v, i, srt, f"positions differ .*: first at output row {r}")
    # an index off by one
    for srt, (v0, i0) in ((True, (vals, idx)), (False, (uv, ui))):
        i = i0.clone()
        i[r0, k // 2] += 1 if int(i0[r0, k // 2]) + 1 < row_len else -1
        rejects(v0, i, srt, f"positions differ .*: first at output row {r0}")
    # a key that is not src[idx]
    for srt, (v0, i0) in ((True, (vals, idx)), (False, (uv, ui))):
        v = v0.clone()
        bc.bits_of(v)[r0, k - 1] ^= 1
        rejects(v, i0, srt, f"keys differ .*: first at output row {r0}")
    # an unsorted output passed as sorted: the first row whose order the shuffle changed is named
    r = next(r for r in range(rows) if not torch.equal(ui[r], idx[r]))
    rejects(uv, ui, True, f"positions differ .*: first at output row {r},")
    # one element missing from an unsorted output: a pair of the row written twice
    v, i = uv.clone(), ui.clone()
    v[r0, 0], i[r0, 0] = uv[r0, 1], ui[r0, 1]
    rejects(v, i, False, f"positions differ .*: first at output row {r0}")
    rejects(vals[:-1], idx[:-1], True, "shapes")
