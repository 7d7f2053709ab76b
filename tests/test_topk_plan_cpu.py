"""CPU checks of tests/topk_plan.py, the numpy restatement of the row top-k's radix select that tests/test_gpu_topk.py builds its
boundary inputs from: the selection it describes is the first k columns of the stable sort, and each boundary input holds
the number of candidates its test claims at the level it claims."""
import numpy as np
import pytest

from tests.topk_plan import candidates_row, plan, select


def stable_first_k(images, k):
    return np.argsort(images, kind="stable")[:k]


@pytest.mark.parametrize("bits", [16, 32, 64])
def test_select_is_the_stable_sorts_first_k_columns(bits):
    rng = np.random.default_rng(bits)
    dt = {16: np.uint16, 32: np.uint32, 64: np.uint64}[bits]
    for row_len in (1, 2, 33, 257, 3000):
        for draw in ("uniform", "few", "equal", "sorted", "reversed"):
            u = rng.integers(0, np.iinfo(dt).max, row_len, dtype=dt, endpoint=True)
            if draw == "few":
                u = u[:3][rng.integers(0, min(3, row_len), row_len)]
            elif draw == "equal":
                u = np.full(row_len, u[0], dtype=dt)
            elif draw == "sorted":
                u = np.sort(u)
            elif draw == "reversed":
                u = np.sort(u)[::-1].copy()
            for k in sorted({min(1, row_len), min(2, row_len), min(50, row_len), row_len}):
                got = select(u, k, bits)
                assert got.size == k, (row_len, draw, k)
                # the kernel's output order, sorted stable by key, is the stable sort's first k columns: equal keys come in
                # position order
                again = got[np.argsort(u[got], kind="stable")]
                assert np.array_equal(again, stable_first_k(u, k)), (row_len, draw, k)


def test_plan_reads_a_row_at_most_digits_plus_one_times():
    rng = np.random.default_rng(5)
    for bits, dt in ((16, np.uint16), (32, np.uint32), (64, np.uint64)):
        for row_len, k in ((300, 1), (5000, 50), (20000, 1024)):
            u = rng.integers(0, 4, row_len).astype(dt)  # every level's bucket mostly ties
            p = plan(u, k, bits, 16384)
            assert len(p) <= bits // 8 + 1
            assert p[-1]["last"] and not any(e["last"] for e in p[:-1])
            # a row that fits is read from global memory once
            if row_len <= 16384:
                assert [e["source"] for e in p] == ["global"] + ["smem"] * (len(p) - 1)


@pytest.mark.parametrize("level", [1, 2])
@pytest.mark.parametrize("bits", [32, 64])
def test_candidates_row_holds_n_candidates_after_its_level(level, bits):
    rng = np.random.default_rng(level * 10 + bits)
    cap = 300
    for n in (cap, cap + 1):
        for k in (1, 50, 256):
            u = candidates_row(rng, 3000, k, n, level, bits)
            p = plan(u, k, bits, cap)
            assert p[level]["candidates"] == n
            assert all(e["source"] == "global" for e in p[:level + 1])
            assert p[level]["compact"] == (n <= cap) and not p[level]["last"]
            assert p[level + 1]["source"] == ("smem" if n <= cap else "global")
            assert np.array_equal(np.sort(select(u, k, bits)), np.sort(stable_first_k(u, k)))
