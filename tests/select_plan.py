"""A numpy restatement of the row select's split path (osb200_select_rows; the LongRowGeo instantiations of
select_count_kernel, select_pick_kernel, select_eq_count_kernel and select_locate_kernel), over one row's radix images
(unsigned keys whose ascending order is the library's order), and of the workspace bound the header states.
tests/test_select_plan_cpu.py checks it against a stable argsort.

Every rank r_i has a state: the prefix v_i of its key's top t digits and taken_i, the keys below v_i's range.  At level t the
ranks whose prefixes are equal form a group (contiguous, the ranks increasing); each key matches at most one group's prefix
and is counted by digit t into that group's 256 bins.  Each rank of a group takes the bucket b holding its (r_i - taken_i)-th
candidate, taken_i grows by the candidates below b and b is appended to v_i.  After the last level v_i is the key, and its
position is occurrence r_i - taken_i of that key in row order."""
import numpy as np


def select(images, ranks, key_bits):
    """(values, positions, levels) of one row: levels[t] = {"groups": [(prefix, first rank, last rank + 1)], "counted": keys
    counted at level t, "picks": [(bucket, below, in bucket)] per rank}"""
    u = np.asarray(images).astype(np.uint64)
    ranks = list(ranks)
    assert ranks and all(b > a for a, b in zip(ranks, ranks[1:])) and ranks[-1] < u.size
    v, taken = [0] * len(ranks), [0] * len(ranks)
    levels = []
    for t in range(key_bits // 8):
        shift = key_bits - 8 * (t + 1)
        mask = ((1 << (8 * t)) - 1) << (key_bits - 8 * t) if t else 0
        groups, i = [], 0
        while i < len(ranks):
            j = i + 1
            while j < len(ranks) and v[j] == v[i]:
                j += 1
            groups.append((v[i], i, j))
            i = j
        counted, picks = 0, [None] * len(ranks)
        for prefix, i, j in groups:
            members = u[(u & np.uint64(mask)) == np.uint64(prefix)]
            counted += members.size
            hist = np.bincount(((members >> np.uint64(shift)) & np.uint64(0xFF)).astype(np.int64), minlength=256)
            excl = np.concatenate([[0], np.cumsum(hist)[:-1]])
            for q in range(i, j):
                need = ranks[q] - taken[q]
                b = int(np.flatnonzero((excl <= need) & (need < excl + hist))[0])
                picks[q] = (b, int(excl[b]), int(hist[b]))
                v[q] |= b << shift
                taken[q] += int(excl[b])
        levels.append({"groups": groups, "counted": counted, "picks": picks})
    positions = [int(np.flatnonzero(u == np.uint64(v[q]))[ranks[q] - taken[q]]) for q in range(len(ranks))]
    return np.array(v, dtype=np.uint64), np.array(positions, dtype=np.int64), levels


TILE, CHUNK = 8192, 4096  # the long rows' tile and scan chunk (counts per chunk)


def workspace_words(num_rows, row_len, num_ranks, positions=True):
    """the 32-bit words of the alternate keys the split path needs (include/onesweep_b200.h, select_layout)"""
    def round4(w):
        return (w + 3) // 4 * 4
    tiles = -(-row_len // TILE)
    words = round4(16 + num_rows * num_ranks * (4 + 256))
    if positions:
        words += round4(num_rows * num_ranks * tiles)
        chunks = -(-num_ranks * tiles // CHUNK)
        if chunks > 1:
            words += round4(num_rows * chunks)
    return words
