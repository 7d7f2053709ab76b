"""CPU checks of tests/select_plan.py, the numpy restatement of the row select's split path: the grouped multi-rank select
finds the columns of the stable sort at the ranks, counts every key at most once per level, and the workspace bound it states
(the header's) is the Python package's and fits every handle with max_n >= num_rows * row_len for rows above the row sort's
capacity."""
import numpy as np
import pytest

from tests.select_plan import select, workspace_words


def rows_for(rng, bits, row_len):
    dt = {16: np.uint16, 32: np.uint32, 64: np.uint64}[bits]
    u = rng.integers(0, np.iinfo(dt).max, row_len, dtype=dt, endpoint=True)
    top = dt(0x5A) << dt(bits - 8)
    return {
        "uniform": u,
        "few": u[:3][rng.integers(0, min(3, row_len), row_len)],
        "equal": np.full(row_len, u[0], dtype=dt),
        "constant_top_byte": (u >> dt(8)) | top,
        "last_digit_only": top | (u & dt(0xFF)),
        "sorted": np.sort(u),
        "reversed": np.sort(u)[::-1].copy(),
    }


@pytest.mark.parametrize("bits", [16, 32, 64])
def test_select_is_the_stable_sorts_columns(bits):
    rng = np.random.default_rng(bits)
    for row_len in (1, 2, 33, 257, 5000):
        for name, u in rows_for(rng, bits, row_len).items():
            order = np.argsort(u, kind="stable")
            for ranks in ({0}, {row_len - 1}, {(row_len - 1) // 2},
                          {round(i * (row_len - 1) / 15) for i in range(16)}, set(range(min(16, row_len)))):
                ranks = sorted(ranks)
                v, pos, levels = select(u, ranks, bits)
                assert np.array_equal(pos, order[ranks]), (name, row_len, ranks)
                assert np.array_equal(v, u[order[ranks]].astype(np.uint64)), (name, row_len, ranks)
                assert len(levels[0]["groups"]) == 1  # one group at level 0
                for lv in levels:
                    assert lv["counted"] <= row_len  # no key is counted twice in a level
                    assert len(lv["groups"]) <= len(ranks)


def test_groups_part_at_the_last_level():
    rng = np.random.default_rng(1)
    u = (np.uint32(0xA5B6C700) | rng.integers(0, 256, 4000).astype(np.uint32))
    ranks = [round(i * 3999 / 15) for i in range(16)]
    _, _, levels = select(u, ranks, 32)
    assert [len(lv["groups"]) for lv in levels[:3]] == [1, 1, 1]
    assert len(levels[3]["groups"]) == 1 and len({p[0] for p in levels[3]["picks"]}) > 1


def test_workspace_bound_from_shapes():
    import gpusorting_b200 as g

    for num_rows in (1, 3, 1000):
        for row_len in (2, 8193, 16385, 151_936, 1 << 26):
            for r in (1, 3, 16):
                for pos in (False, True):
                    assert workspace_words(num_rows, row_len, r, pos) == g.select_workspace_words(num_rows, row_len, r, pos)
    # a quantile over 2^30 keys: about 17 KB of row state, 8 MiB of tile counts and 2 KiB of chunk sums
    assert workspace_words(1, 1 << 30, 16) * 4 < 17_000 + 8 * 2**20 + 2048 + 64
    # every handle with max_n >= n (alternate keys of at least 4 bytes per key) has the room above the row sort's capacity
    for cap in (8192, 16384):
        for row_len in (cap + 1, cap + 2, 2 * cap, 65_536, 151_936, (1 << 32) - 1):
            for num_rows in (1, 2, 7, 1000):
                assert workspace_words(num_rows, row_len, 16) <= num_rows * row_len
