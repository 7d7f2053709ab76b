"""Sorts past 2^31 and 2^32 elements through the paths that compute element positions in their own code: the 64-bit keys
pairs pass (payloads stored through per-digit pointers, one CTA per 8,192-pair tile), the argsorts' copy-back of 16- and
64-bit keys (indices generated there when no pass or an odd number of passes executes) and their first pass (payloads
generated from tile bases), the 16-bit keys histogram and passes, and the row sort's row bases.  A position truncated to
32 bits anywhere there would go unnoticed at the sizes the feature tests use.

Inputs are generated on the device, chunk by chunk, from fixed seeds, and regenerated to check the outputs (and that the
argsorts leave their input as it was).  The checkers (tests/bigcheck.py, themselves tested on the CPU by
tests/test_large_n_checks_cpu.py) prove the stable sort through payload = input position, or through the histogram of
16-bit keys, or through torch.sort of whole rows; no torch op sees more than CHUNK elements of an output.

Each test computes the device memory it needs (about 70 GiB for the largest) and skips, saying so, when the GPU has less
free.  Every test name here contains "past_2pow": -m gpu -k "not past_2pow" leaves them out of a quick run.  -m gpu"""
import pytest
import torch

from tests import bigcheck as bc
from tests.test_gpu_large_n import release, require

pytestmark = pytest.mark.gpu

CHUNK = 1 << 26   # elements per generated chunk and per checked chunk
CHECK = 48 * CHUNK  # bytes: a bound on the temporaries of one checked chunk (int64 radix images, positions, gathers)
GUARD = 64
SIZE = -2  # OSB200_ERR_SIZE
F16 = 2    # OSB200_KEY16_F16


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


def s64(x: int) -> int:
    """a 64-bit pattern as the int64 that holds it"""
    return x - (1 << 64) if x >= (1 << 63) else x


# ---- inputs: one generator per input, consumed chunk by chunk, so the same call regenerates the same values ------------------
def generate(t, seed, make, compare=False, what="input"):
    """t (flattened, as its integer container) = make(gen, m) chunk by chunk; compare=True asserts it still holds that"""
    flat = bc.bits_of(t).reshape(-1)
    gen = torch.Generator(device=t.device).manual_seed(seed)
    for a in range(0, flat.numel(), CHUNK):
        m = min(CHUNK, flat.numel() - a)
        if compare:
            assert torch.equal(flat[a:a + m], make(gen, m)), f"{what} changed in [{a}, {a + m})"
        else:
            flat[a:a + m] = make(gen, m)


def rand64(gen, m):
    hi = torch.randint(-(1 << 31), 1 << 31, (m,), generator=gen, device="cuda", dtype=torch.int64)
    return hi * (1 << 32) | torch.randint(0, 1 << 32, (m,), generator=gen, device="cuda", dtype=torch.int64)


def rand16(gen, m):
    """uniform 16-bit patterns, as int32 0 .. 65535"""
    return torch.randint(0, 1 << 16, (m,), generator=gen, device="cuda", dtype=torch.int32)


def as_int16(u):
    return ((u ^ 0x8000) - 0x8000).to(torch.int16)


def positions_mod_2pow32(t):
    """t[i] = i mod 2^32, as int32 (payload = input position; positions >= 2^31 read as negative)"""
    for a in range(0, t.numel(), CHUNK):
        x = torch.arange(a, min(a + CHUNK, t.numel()), device=t.device, dtype=torch.int64) & 0xFFFFFFFF
        t[a:a + x.numel()] = ((x ^ 0x80000000) - 0x80000000).to(torch.int32)


def assert_positions(idx, what):
    """idx[i] == i mod 2^32"""
    for a in range(0, idx.numel(), CHUNK):
        b = min(a + CHUNK, idx.numel())
        want = torch.arange(a, b, device=idx.device, dtype=torch.int64) & 0xFFFFFFFF
        assert torch.equal(bc.positions(idx[a:b]), want), f"{what}: indices in [{a}, {b}) are not the positions"


# ---- 64-bit keys with uint32 payloads ----------------------------------------------------------------------------------------
def spread20(gen, m):
    """f64 keys whose radix images (descending) are 20-bit values spread over all 8 bytes: ~2^11 copies of each"""
    v = torch.randint(0, 1 << 20, (m,), generator=gen, device="cuda", dtype=torch.int64)
    r = v | (v << 20) | (v << 40) | ((v & 7) << 60)  # the low 20 bits are v: one image per value
    r = torch.where((v & 8) != 0, r | bc.SIGN64, r)
    return bc.from_radix64(r, "f", descending=True)


def test_pairs64_past_2pow31(g):
    n = (1 << 31) + 4099
    # sort: workspace, keys and payloads; check: keys, payloads, the regenerated input and one chunk's temporaries
    require(g, "(8, 4) pairs", n + GUARD, 8, 4, 12 * (n + GUARD), 20 * (n + GUARD) + CHECK)
    k = torch.empty(n + GUARD, dtype=torch.float64, device="cuda")
    v = torch.empty(n + GUARD, dtype=torch.int32, device="cuda")
    generate(k, 31, spread20)
    positions_mod_2pow32(v)
    s = g.OneSweepSorter(n + GUARD, 8, 4)
    try:
        s.sort_pairs_typed(k, v, "f64", descending=True, n=n)
        assert s.info("last_executed_passes") == 8
    finally:
        torch.cuda.synchronize()
        s.close()
    src = torch.empty(n + GUARD, dtype=torch.float64, device="cuda")
    generate(src, 31, spread20)
    try:
        assert torch.equal(bc.bits_of(k[n:]), bc.bits_of(src[n:])), "key guard after n"
        assert torch.equal(bc.positions(v[n:]), torch.arange(n, n + GUARD, device="cuda")), "payload guard after n"
        bc.check_sorted_by_position(k[:n], v[:n], src[:n], bc.key_radix("f64", True), CHUNK)
    finally:
        del k, v, src
        release()


ARGSORT64_FILL = 0x5AA5C33C0FF01EE1
BYTES_036 = 0x00FF0000FF0000FF


def i64_bytes_036(gen, m):
    """i64 keys whose radix images vary only in bytes 0, 3 and 6; 35 % of them are one value (a hot bin in every pass)"""
    r = (rand64(gen, m) & BYTES_036) | (ARGSORT64_FILL & ~BYTES_036)
    tied = torch.rand(m, generator=gen, device="cuda") < 0.35
    return bc.from_radix64(torch.where(tied, s64(0x5A77C33C11F01E99), r), "i")


def i64_all_bytes(gen, m):
    """random i64 keys, 5 % of them one value"""
    r = rand64(gen, m)
    return torch.where(torch.rand(m, generator=gen, device="cuda") < 0.05, s64(0xC0FFEE0123456789), r)


def i64_equal(gen, m):
    return torch.full((m,), -12345678901, device="cuda", dtype=torch.int64)


def test_argsort64_past_2pow31(g):
    n = (1 << 31) + 12345
    # the sorter stays open for three inputs: workspace, input, output keys, indices and one checked chunk's temporaries
    require(g, "(8, 4) argsort", n, 8, 4, 20 * n + CHECK, 0)
    kin = torch.empty(n, dtype=torch.int64, device="cuda")
    radix = bc.key_radix("i64")
    s = g.OneSweepSorter(n, 8, 4)
    try:
        for seed, make, passes, hot in ((41, i64_bytes_036, 3, 0x49), (42, i64_all_bytes, 8, None), (43, i64_equal, 0, 0)):
            what = make.__name__
            generate(kin, seed, make)
            out, idx = s.argsort(kin, "i64")
            torch.cuda.synchronize()
            assert s.info("last_executed_passes") == passes, what
            if hot is not None:
                assert s.info("last_hot_mask") == hot, what
            generate(kin, seed, make, compare=True, what=f"argsort input, {what}")
            if passes == 0:  # the copy-back generates every index: out is the input, idx the positions
                generate(out, seed, make, compare=True, what=f"argsort keys, {what}")
                assert_positions(idx, what)
            bc.check_sorted_by_position(out, idx, kin, radix, CHUNK)
            del out, idx
    finally:
        torch.cuda.synchronize()
        s.close()
        del kin
        release()


# ---- 16-bit keys -----------------------------------------------------------------------------------------------------------
def test_keys16_past_2pow32(g):
    n = (1 << 32) + 12345
    # sort: workspace and keys; check: keys, the regenerated input and one chunk's temporaries
    require(g, "(4, 0) keys16", n + GUARD, 4, 0, 2 * (n + GUARD), 4 * (n + GUARD) + CHECK)

    def make(gen, m):
        return as_int16(rand16(gen, m))

    k = torch.empty(n + GUARD, dtype=torch.bfloat16, device="cuda")
    generate(k, 51, make)
    s = g.OneSweepSorter(n + GUARD, 4, 0)
    try:
        s.sort_keys16(k, "bf16", descending=True, n=n)
        assert s.info("last_executed_passes") == 2
    finally:
        torch.cuda.synchronize()
        s.close()
    src = torch.empty(n + GUARD, dtype=torch.bfloat16, device="cuda")
    generate(src, 51, make)
    try:
        assert torch.equal(bc.bits_of(k[n:]), bc.bits_of(src[n:])), "guard after n"
        bc.check_sorted_keys16(k[:n], src[:n], bc.key_radix("bf16", True), CHUNK)
    finally:
        del k, src
        release()


def test_pairs16_past_2pow32(g):
    head = 1 << 32
    tail = 12345
    n = head + tail

    def make(gen, m):  # never -32768: the tail's key, whose payloads (positions mod 2^32) are 0 .. 12344
        return torch.randint(-32767, 32768, (m,), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)

    def inputs(t):
        generate(t[:head], 61, make)
        t[head:].fill_(-32768)

    # sort: workspace, keys and payloads; check: keys, payloads, the regenerated input and one chunk's temporaries
    require(g, "(4, 4) pairs16", n, 4, 4, 6 * n, 8 * n + CHECK)
    k = torch.empty(n, dtype=torch.int16, device="cuda")
    v = torch.empty(n, dtype=torch.int32, device="cuda")
    inputs(k)
    positions_mod_2pow32(v)
    s = g.OneSweepSorter(n, 4, 4)
    try:
        s.sort_pairs16(k, v, "i16")
        assert s.info("last_executed_passes") == 2
    finally:
        torch.cuda.synchronize()
        s.close()
    src = torch.empty(n, dtype=torch.int16, device="cuda")
    inputs(src)
    try:
        assert bool((k[:tail] == -32768).all()), "the smallest key, only in the last 12,345 positions, does not lead"
        assert torch.equal(v[:tail], torch.arange(tail, dtype=torch.int32, device="cuda")), \
            "payloads of the last 12,345 positions (2^32 + j, stored as j)"
        # every other payload p names position p < 2^32
        bc.check_sorted_by_position(k[tail:], v[tail:], src[:head], bc.key_radix("i16"), CHUNK)
    finally:
        del k, v, src
        release()


def f16_random(gen, m):
    return as_int16(rand16(gen, m))


def f16_low_byte(gen, m):
    return bc.from_radix16((rand16(gen, m) & 0xFF) | 0xBC00, "f16")


def f16_equal(gen, m):
    return torch.full((m,), 0x4248, device="cuda", dtype=torch.int16)


def test_argsort16_past_2pow31_at_the_2pow32_limit(g):
    n = 1 << 32
    # the sorter stays open for three inputs: workspace, input, output keys, indices and one checked chunk's temporaries
    require(g, "(4, 4) argsort16", n + 1, 4, 4, 8 * n + CHECK, 0)
    kin = torch.empty(n, dtype=torch.float16, device="cuda")
    radix = bc.key_radix("f16")
    s = g.OneSweepSorter(n + 1, 4, 4)
    try:
        for seed, make, passes in ((71, f16_random, 2), (72, f16_low_byte, 1), (73, f16_equal, 0)):
            what = make.__name__
            generate(kin, seed, make)
            out, idx = s.argsort16(kin, "f16")
            torch.cuda.synchronize()
            assert s.info("last_executed_passes") == passes, what
            generate(kin, seed, make, compare=True, what=f"argsort16 input, {what}")
            if passes == 0:  # the copy-back generates every index, the last one 2^32 - 1
                generate(out, seed, make, compare=True, what=f"argsort16 keys, {what}")
                assert_positions(idx, what)
                assert int(idx[-1]) == -1, "the last index, 0xFFFFFFFF"
            bc.check_sorted_by_position(out, idx, kin, radix, CHUNK)
            if passes == 0:  # one more key does not fit the 32-bit indices
                assert g.lib.osb200_argsort16(s._h, kin.data_ptr(), out.data_ptr(), idx.data_ptr(), n + 1, F16, 0,
                                              None) == SIZE
            del out, idx
    finally:
        torch.cuda.synchronize()
        s.close()
        del kin
        release()


# ---- the row sort ----------------------------------------------------------------------------------------------------------
def rows16(gen, m):
    """16-bit patterns, half of them from 64 values: many equal keys in every row"""
    u = rand16(gen, m)
    return as_int16(torch.where(torch.rand(m, generator=gen, device="cuda") < 0.5, u & 0xC107, u))


def rows64(gen, m):
    """64-bit patterns, half of them from 64 values: many equal keys in every row"""
    u = rand64(gen, m)
    return torch.where(torch.rand(m, generator=gen, device="cuda") < 0.5, u & s64(0x8000010000010007), u)


def sort_and_check_rows(g, rows, row_len, dtype, key_type, descending, seed, make):
    """sort_rows with indices, out of place; checked against torch.sort of every row of the (untouched) input"""
    x = torch.empty(rows, row_len, dtype=dtype, device="cuda")
    generate(x, seed, make)
    with g.OneSweepSorter(1, 4, 0) as s:
        out, idx = s.sort_rows(x, key_type, descending)
        torch.cuda.synchronize()
    try:
        generate(x, seed, make, compare=True, what="sort_rows input")
        bc.check_rows(out, idx, x, bc.key_radix(key_type, descending), CHUNK)
    finally:
        del x, out, idx
        release()


def test_rows_past_2pow32_warp_path(g):
    row_len, rows = 200, (1 << 32) // 200 + 1
    n = rows * row_len
    require(g, "bf16 rows of 200", 1, 4, 0, 8 * n + CHECK, 0)  # input, output keys, indices
    sort_and_check_rows(g, rows, row_len, torch.bfloat16, "bf16", True, 81, rows16)


def test_rows_past_2pow32_block_path(g):
    row_len, rows = 16384, (1 << 18) + 1
    n = rows * row_len
    require(g, "f16 rows of 16,384", 1, 4, 0, 8 * n + CHECK, 0)
    sort_and_check_rows(g, rows, row_len, torch.float16, "f16", False, 82, rows16)
    # in place, without indices: checked against the regenerated input
    x = torch.empty(rows, row_len, dtype=torch.uint16, device="cuda")
    generate(x, 83, rows16)
    with g.OneSweepSorter(1, 4, 0) as s:
        s.sort_rows(x, "u16", return_indices=False, inplace=True)
        torch.cuda.synchronize()
    src = torch.empty_like(x)
    generate(src, 83, rows16)
    try:
        bc.check_rows(x, None, src, bc.key_radix("u16"), CHUNK)
    finally:
        del x, src
        release()


def test_rows_past_2pow31_8byte(g):
    for row_len, rows, dtype, key_type, descending, seed in (
            (8192, (1 << 18) + 1, torch.float64, "f64", True, 84),  # the block path
            (256, (1 << 23) + 1, torch.int64, "i64", False, 85)):   # the warp path
        n = rows * row_len
        require(g, f"{key_type} rows of {row_len}", 1, 4, 0, 20 * n + CHECK, 0)
        sort_and_check_rows(g, rows, row_len, dtype, key_type, descending, seed, rows64)
