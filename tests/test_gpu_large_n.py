"""Sorts past 2^31 and 2^32 elements: the element indices, tile bases and digit offsets of the default kernel must be 64-bit
all the way (the 38-bit descriptor value field allows n up to 2^34 per sorter; the reference stops at 2^30).

No CPU sort of 16 GiB: the keys-only outputs are compared element by element with torch.sort, bucket by bucket.  The
input is regenerated with the deterministic InitRandom; its histogram of the top key byte gives every bucket's slice of
the output; each bucket's input keys are gathered, sorted and compared with that slice.  Keys of 20 bits, whose buckets
would be too uneven for that, are checked through their full histogram instead: an ascending output with the input's
count of every one of the 2^20 values is the sorted input.  Pairs are checked through payload
= input index: the output is sorted, every payload points at an input element with the same key, and indices ascend
inside every run of equal keys -- together, exactly the stable sort.  No torch op sees more than 2^28 elements.

Each test computes the device memory it needs (about 46 GiB for the largest) and skips, saying so, when the GPU has less
free.  Every test name here contains "past_2pow": -m gpu -k "not past_2pow" leaves them out of a quick run.  -m gpu"""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu

GiB = 1 << 30
CHUNK = 1 << 28        # elements per torch op
GROUP = 1 << 27        # most elements one torch.sort of gathered buckets sees
VERIFY_EXTRA = 10 * GiB  # temporaries of one bucket group: gather masks and parts, int64 copies, sort values and indices
HEADROOM = 4 * GiB


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def require(g, what, n, key_bytes, value_bytes, own_bytes, verify_bytes):
    """skip unless the free device memory covers the sort (workspace + the test's tensors) and the check after it"""
    gc.collect()
    torch.cuda.empty_cache()
    ws = g.lib.osb200_workspace_bytes(n, key_bytes, value_bytes)
    need = max(ws + own_bytes, verify_bytes)
    free, _ = torch.cuda.mem_get_info()
    if free < need + HEADROOM:
        pytest.skip(f"{what}: needs {need / GiB:.1f} GiB (+{HEADROOM // GiB} GiB headroom), {free / GiB:.1f} GiB free")


def release():
    gc.collect()
    torch.cuda.empty_cache()


def check_by_buckets(out, src, bucket_of, sortable):
    """out must equal the ascending sort of src.  bucket_of(x): integer bucket 0..255 that is monotone in the key order;
    sortable(x): int64 whose signed order is the key order (out and src are never sorted or reordered whole)."""
    n = src.numel()
    assert out.numel() == n
    hist = torch.zeros(256, dtype=torch.int64, device=src.device)
    for a in range(0, n, CHUNK):
        hist += torch.bincount(bucket_of(src[a:a + CHUNK]).long(), minlength=256)
    ends = torch.cumsum(hist, 0).tolist()
    starts = [0] + ends[:-1]
    b = 0
    while b < 256:
        e = b + 1  # a group of consecutive buckets of at most GROUP keys (a bucket larger than that is its own group)
        while e < 256 and ends[e] - starts[b] <= GROUP:
            e += 1
        lo, hi = starts[b], ends[e - 1]
        if hi > lo:
            parts = []
            for a in range(0, n, CHUNK):
                bk = bucket_of(src[a:a + CHUNK])
                parts.append(src[a:a + CHUNK][(bk >= b) & (bk < e)])
                del bk
            want = torch.sort(sortable(torch.cat(parts))).values
            del parts
            got = sortable(out[lo:hi])
            assert want.numel() == hi - lo and torch.equal(got, want), f"buckets [{b}, {e}): output slice [{lo}, {hi})"
            del want, got
        b = e


def in_chunks(t, fn):
    for a in range(0, t.numel(), CHUNK):
        fn(t[a:a + CHUNK])


def check_full_keys_u32(out, src):
    # int32 containers: >> is an arithmetic shift, hence the mask
    check_by_buckets(out, src, lambda x: (x >> 24) & 0xFF, lambda x: x.to(torch.int64) & 0xFFFFFFFF)


def check_20bit_keys(out, src):
    bins = 1 << 20
    h_in = torch.zeros(bins, dtype=torch.int64, device=src.device)
    h_out = torch.zeros_like(h_in)
    n = src.numel()
    for a in range(0, n, CHUNK):
        h_in += torch.bincount(src[a:a + CHUNK].long(), minlength=bins)
        h_out += torch.bincount(out[a:a + CHUNK].long(), minlength=bins)
        o = out[a:a + CHUNK + 1]  # one element of overlap with the next chunk
        assert bool((o[1:] >= o[:-1]).all()), f"output not ascending in [{a}, {a + o.numel()})"
    assert torch.equal(h_in, h_out), "output is not a permutation of the input"


@pytest.mark.parametrize("and_count,mask,skip,hot,check", [
    (0, None, 0b0000, 0b0000, check_full_keys_u32),
    (2, 0xFFFFF, 0b1000, 0b0111, check_20bit_keys),  # AND of 3 words, 20 bits: top pass skipped, three hot ones, copy-back
], ids=["full_entropy", "20bit_low_entropy"])
def test_keys_u32_past_2pow32(g, and_count, mask, skip, hot, check):
    n = (1 << 32) + (1 << 20) + 7  # a ragged last tile
    require(g, "u32 keys", n, 4, 0, 4 * n, 8 * n + VERIFY_EXTRA)
    t = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(t, and_count, 12)
    if mask is not None:
        in_chunks(t, lambda c: c.bitwise_and_(mask))
    s = g.OneSweepSorter(n, 4, 0)
    try:
        s.sort_keys(t)
        assert s.info("last_skip_mask") == skip and s.info("last_hot_mask") == hot
        assert s.validate(t) == 0
    finally:
        s.close()
    src = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(src, and_count, 12)
    if mask is not None:
        in_chunks(src, lambda c: c.bitwise_and_(mask))
    try:
        check(t, src)
    finally:
        del t, src
        release()


def test_pairs_u32_past_2pow31(g):
    n = (1 << 31) + 4099
    # sort: keys + payloads; check: keys, payloads, the regenerated input and one chunk of int64 indices, gathered keys, masks
    require(g, "u32 pairs", n, 4, 4, 8 * n, 12 * n + 4 * CHUNK * 8)
    k = torch.empty(n, dtype=torch.int32, device="cuda")
    v = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(k, 0, 13, payload=v, payload_is_index=True)
    in_chunks(k, lambda c: c.bitwise_and_(0xFFFFF))  # ~2048 copies of every key value: stability is observable
    s = g.OneSweepSorter(n, 4, 4)
    try:
        s.sort_pairs(k, v)
        assert s.validate(k) == 0
    finally:
        s.close()
    kin = torch.empty(n, dtype=torch.int32, device="cuda")
    g.init_random(kin, 0, 13)
    in_chunks(kin, lambda c: c.bitwise_and_(0xFFFFF))
    try:
        for a in range(0, n, CHUNK):
            b = min(a + CHUNK, n)
            idx = v[a:b].to(torch.int64) & 0xFFFFFFFF  # indices >= 2^31 are negative in the int32 container
            assert torch.equal(kin[idx], k[a:b]), f"payload round trip, output [{a}, {b})"
            del idx
            e = min(b + 1, n)  # one element of overlap: runs of equal keys cross chunk borders
            ks, vs = k[a:e], v[a:e].to(torch.int64) & 0xFFFFFFFF
            assert bool(((vs[1:] > vs[:-1]) | (ks[1:] != ks[:-1])).all()), f"stability, output [{a}, {e})"
            del ks, vs
    finally:
        del k, v, kin
        release()


def test_keys_u64_past_2pow31(g):
    n = (1 << 31) + 12345
    require(g, "u64 keys", n, 8, 0, 8 * n, 16 * n + VERIFY_EXTRA)
    w = torch.empty(2 * n, dtype=torch.int32, device="cuda")
    g.init_random(w, 0, 14)  # low and high words are consecutive draws
    t = w.view(torch.int64)
    s = g.OneSweepSorter(n, 8, 0)
    try:
        s.sort_keys(t)
        assert s.validate(t) == 0
    finally:
        s.close()
    ws = torch.empty(2 * n, dtype=torch.int32, device="cuda")
    g.init_random(ws, 0, 14)
    sign = -(1 << 63)
    try:
        # buckets: the top byte of the high word; sort as int64 with the sign bit flipped (signed order = unsigned order)
        check_by_buckets(t, ws.view(torch.int64), lambda x: (x >> 56) & 0xFF, lambda x: x ^ sign)
    finally:
        del w, t, ws
        release()
