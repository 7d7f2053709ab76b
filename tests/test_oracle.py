"""The oracle (oracle/oracle.c) against numpy and against the golden fixtures produced by the reference's own
CUDA kernels (tests/golden/ref_onesweep_golden.json).  Runs on CPU."""
import json
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_onesweep_golden.json")


def test_generator_known_values(oracle):
    # InitRandom(seed=10, andCount=0): values pinned by the reference kernel run recorded in the golden file
    k = oracle.init_random_u32(1 << 17, 0, 10)
    assert [hex(x) for x in k[:4]] == ["0xffeb2900", "0x88b92968", "0x11876dd0", "0x9a57ca38"]
    assert [hex(x) for x in k[65536:65538]] == ["0x145cb47f", "0x6766deee"]


def test_generator_entropy_presets_and(oracle):
    # AND-ing more draws can only clear bits; population count must fall monotonically (Thearling-Smith)
    pops = []
    for andc in range(5):
        k = oracle.init_random_u32(1 << 16, andc, 10)
        pops.append(int(np.unpackbits(k.view(np.uint8)).sum()))
    assert all(a > b for a, b in zip(pops, pops[1:]))
    assert abs(pops[0] / (32 * (1 << 16)) - 0.5) < 0.01


@pytest.mark.parametrize("n", [0, 1, 2, 255, 256, 257, 7680, 7681, 100003, 1 << 20])
def test_sort_keys_u32_matches_numpy(oracle, n):
    k = oracle.init_random_u32(n, 0, 10 + n) if n else np.empty(0, np.uint32)
    assert np.array_equal(oracle.sort_keys(k), np.sort(k, kind="stable"))


@pytest.mark.parametrize("andc", [0, 2, 4])
def test_sort_pairs_is_stable(oracle, andc):
    n = 200003
    k = oracle.init_random_u32(n, andc, 77) & np.uint32(0x3FF)  # many duplicate keys
    v = np.arange(n, dtype=np.uint32)
    sk, sv = oracle.sort_pairs(k, v)
    order = np.argsort(k, kind="stable").astype(np.uint32)
    assert np.array_equal(sv, order) and np.array_equal(sk, k[order])
    # std::stable_sort baseline agrees
    k2, v2 = k.copy(), v.copy()
    oracle.lib.orc_std_stable_sort_pairs_u32(k2.ctypes.data, v2.ctypes.data, n)
    assert np.array_equal(k2, sk) and np.array_equal(v2, sv)


def test_sort_keys_u64_matches_numpy(oracle):
    k = oracle.init_random_u64(150001, 0, 10)
    assert np.array_equal(oracle.sort_keys(k), np.sort(k))
    assert len(np.unique(k >> np.uint64(32))) > 100000  # hi words are independent draws


def test_histogram_scan_and_single_pass(oracle):
    k = oracle.init_random_u32(123457, 0, 5)
    h = oracle.global_histogram(k)
    for p in range(4):
        assert np.array_equal(h[p], np.bincount((k >> (8 * p)) & 255, minlength=256).astype(np.uint64))
    ex = oracle.scan_exclusive(h)
    assert np.array_equal(ex[2], np.concatenate([[0], np.cumsum(h[2])[:-1]]).astype(np.uint64))
    out = oracle.binning_pass(k, 8)
    order = np.argsort((k >> 8) & 255, kind="stable")
    assert np.array_equal(out, k[order])


def test_parallel_port_equals_serial(oracle):
    k = oracle.init_random_u32(1 << 20, 0, 3)
    want = oracle.sort_keys(k)
    for threads in (1, 3, 0):
        got = k.copy()
        assert oracle.sort_parallel_inplace(got, threads=threads) == 0
        assert np.array_equal(got, want)
    v = np.arange(k.size, dtype=np.uint32)
    kk, vv = (k & np.uint32(0xFFF)).copy(), v.copy()
    oracle.sort_parallel_inplace(kk, vv, threads=0)
    assert np.array_equal(vv, np.argsort(k & np.uint32(0xFFF), kind="stable").astype(np.uint32))


def test_validate_counts_inversions(oracle):
    k = np.array([1, 2, 2, 5, 4, 4, 9, 0], np.uint32)
    assert oracle.validate(k) == 2
    assert oracle.validate(np.sort(k)) == 0
    std = k.copy()
    oracle.lib.orc_std_sort_u32(std.ctypes.data, std.size)
    assert np.array_equal(std, np.sort(k))


@pytest.mark.parametrize("ftype,utype", [(np.float32, np.uint32), (np.float64, np.uint64)])
def test_to_radix_is_ieee_total_order(ftype, utype):
    """The typed-key transform the GPU tests compare with, checked against numpy's float order and the IEEE 754 totalOrder
    cases numpy cannot express (signed zeros, NaNs of both signs and several payloads)."""
    from tests.oraclelib import from_radix, to_radix

    rng = np.random.default_rng(11)
    fi = np.finfo(ftype)
    nb = np.dtype(utype).itemsize * 8
    sign = 1 << (nb - 1)
    # distinct magnitudes (numpy calls -0.0 == +0.0; total order does not), specials included
    mags = np.concatenate([rng.standard_normal(3000) * 1e3, rng.standard_normal(500) * 1e-3,
                           [fi.max, fi.tiny, fi.tiny * fi.eps, fi.tiny - fi.tiny * fi.eps, np.inf, 0.0, 1.0]]).astype(ftype)
    mags = np.unique(np.abs(mags))
    vals = mags * np.where(rng.random(mags.size) < 0.5, -1, 1).astype(ftype)
    vals = vals[rng.permutation(vals.size)]
    bits = vals.view(utype)
    assert np.array_equal(np.argsort(to_radix(bits, "f"), kind="stable"), np.argsort(vals, kind="stable"))

    u = lambda x: np.array([x], dtype=utype)  # noqa: E731
    qnan, exp_all = 1 << (fi.nmant - 1), ((1 << (nb - 1 - fi.nmant)) - 1) << fi.nmant  # quiet bit, all-ones exponent
    pinf, top = exp_all, (1 << fi.nmant) - 1
    # ascending IEEE totalOrder of these bit patterns
    chain = [sign | exp_all | top, sign | exp_all | qnan, sign | exp_all | 1, sign | pinf,   # -NaNs (payload large..small), -inf
             sign | fi.max.view(utype).item(), sign | 1, sign, 0, 1, fi.max.view(utype).item(),  # -max, -min subnormal, -0, +0, ...
             pinf, exp_all | 1, exp_all | qnan, exp_all | top]                                 # +inf, +NaNs (payload small..large)
    keys = np.concatenate([to_radix(u(c), "f") for c in chain])
    assert np.all(keys[1:] > keys[:-1])
    shuffled = np.array(chain, dtype=utype)[rng.permutation(len(chain))]
    assert np.array_equal(shuffled[np.argsort(to_radix(shuffled, "f"), kind="stable")], np.array(chain, dtype=utype))

    # descending: the reverse order of the keys, equal keys (many ties here) keep their input order
    for kind in ("u", "i", "f"):
        b = rng.integers(0, 40, 2000).astype(np.int64) - 20
        b = (b.astype(ftype) if kind == "f" else b.astype(np.int32 if nb == 32 else np.int64)).view(utype)
        asc = to_radix(b, kind)
        want = sorted(range(b.size), key=lambda i: -int(asc[i]))  # Python's sort is stable
        assert np.array_equal(np.argsort(to_radix(b, kind, True), kind="stable"), want)
        if kind != "u":
            typed = b.view(ftype if kind == "f" else (np.int32 if nb == 32 else np.int64))
            assert np.array_equal(np.argsort(to_radix(b, kind, True), kind="stable"), np.argsort(-typed, kind="stable"))
        for desc in (False, True):
            assert np.array_equal(from_radix(to_radix(b, kind, desc), kind, desc), b)
    nans = np.array([c for c in chain if (c & exp_all) == exp_all and (c & top)], dtype=utype)
    for desc in (False, True):
        assert np.array_equal(from_radix(to_radix(nans, "f", desc), "f", desc), nans)


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="golden fixture not generated yet")
def test_oracle_reproduces_reference_golden_vectors(oracle):
    """Pins the oracle to the reference: inputs, sorted outputs, payloads and histograms produced by the
    reference's own CUDA kernels on the GPU (see tests/golden/make_ref_golden.py)."""
    cases = json.load(open(GOLDEN))["cases"]
    assert len(cases) >= 10
    for c in cases:
        n = c["n"]
        k = oracle.init_random_u32(n, c["and_count"], c["seed"])
        assert [int(x) for x in k[:8]] == c["input_head"]
        assert oracle.digest(k) == c["input_digest"]
        assert c["ref_validate_errors"] == 0
        if c["pairs"]:
            sk, sv = oracle.sort_pairs(k, k.copy())  # the reference sets payload = key
            assert oracle.digest(sv) == c["payload_digest"]
        else:
            sk = oracle.sort_keys(k)
        assert [int(x) for x in sk[:8]] == c["sorted_head"]
        assert [int(x) for x in sk[-8:]] == c["sorted_tail"]
        assert oracle.digest(sk) == c["sorted_digest"]
        assert oracle.digest(oracle.global_histogram(k).reshape(-1)) == c["global_hist_digest"]
