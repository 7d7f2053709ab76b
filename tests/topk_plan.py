"""A numpy restatement of the row top-k's radix select (osb200_topk_rows, topk_select_kernel), over one row's radix images
(unsigned keys whose ascending order is the requested order).  It is the level plan the boundary tests of
tests/test_gpu_topk.py are built from, and tests/test_topk_plan_cpu.py checks it against a stable sort.

Pass t (t = 0 .. D, D digit places) reads the candidates S_t, the keys whose t top digits equal the prefix chosen so far.
It selects the keys of S_{t-1} in the buckets below the one chosen at level t - 1, counts digit t of S_t, and picks the
bucket b holding the k'-th candidate.  When b holds exactly k' keys, or after the last digit, the next pass is the last:
it also selects the keys equal to the prefix, the first k' of them in position order.  A pass that reads the row from global
memory while |S_t| <= cap compacts S_t into shared memory; later passes read only that."""
import numpy as np


def plan(images, k, key_bits, cap):
    """[{t, source, candidates, compact, last, bucket, below, in_bucket}] of one row: one entry per pass.  source is "global"
    or "smem", candidates = |S_t|; bucket / below / in_bucket are those picked by the pass (None on the last pass)."""
    images = np.asarray(images)
    u = images.astype(np.uint64)
    digits = key_bits // 8
    mask = value = 0  # S_t = {x : x & mask == value}
    need, cand, in_smem, last = k, u.size, False, False
    out = []
    for t in range(digits + 1):
        compact = not last and not in_smem and cand <= cap
        entry = {"t": t, "source": "smem" if in_smem else "global", "candidates": cand, "compact": compact, "last": last,
                 "bucket": None, "below": None, "in_bucket": None}
        out.append(entry)
        if last:
            break
        if compact:
            in_smem = True
        shift = key_bits - 8 * (t + 1)
        members = u[(u & np.uint64(mask)) == np.uint64(value)]
        hist = np.bincount(((members >> np.uint64(shift)) & np.uint64(0xFF)).astype(np.int64), minlength=256)
        excl = np.concatenate([[0], np.cumsum(hist)[:-1]])
        b = int(np.flatnonzero((hist > 0) & (excl < need) & (need <= excl + hist))[0])
        entry.update(bucket=b, below=int(excl[b]), in_bucket=int(hist[b]))
        need -= int(excl[b])
        cand = int(hist[b])
        mask |= 0xFF << shift
        value |= b << shift
        last = cand == need or t + 1 == digits
    return out


def select(images, k, key_bits):
    """the positions the kernel writes for one row, in its output order (pass by pass, row order within a pass)"""
    u = np.asarray(images).astype(np.uint64)
    digits = key_bits // 8
    mprev = vprev = mcur = vcur = 0
    need, written = k, []
    pos = np.arange(u.size)
    for t in range(digits + 1):
        in_prev = (u & np.uint64(mprev)) == np.uint64(vprev)
        sel = in_prev & ((u & np.uint64(mcur)) < np.uint64(vcur))
        eq = (u & np.uint64(mcur)) == np.uint64(vcur)
        last = t > 0 and (cand == need or t == digits)
        if last:
            keep = eq & (np.cumsum(eq) <= need)
            written += list(pos[sel | keep])
            break
        written += list(pos[sel])
        shift = key_bits - 8 * (t + 1)
        hist = np.bincount(((u[eq] >> np.uint64(shift)) & np.uint64(0xFF)).astype(np.int64), minlength=256)
        excl = np.concatenate([[0], np.cumsum(hist)[:-1]])
        b = int(np.flatnonzero((hist > 0) & (excl < need) & (need <= excl + hist))[0])
        need -= int(excl[b])
        cand = int(hist[b])
        mprev, vprev = mcur, vcur
        mcur |= 0xFF << shift
        vcur |= b << shift
    return np.array(written, dtype=np.int64)


def candidates_row(rng, row_len, k, n, level, key_bits=32):
    """u32 (or u64) radix images of one row in which exactly n candidates are left after `level` levels (1 or 2): the k-th
    smallest key lies in a bucket of n keys at that level and in larger buckets at the levels above.  Keys are drawn so that
    fewer than k lie below the chosen bucket at each level; the rest of the row lies above it."""
    assert level in (1, 2) and k <= n < row_len
    dt = np.uint64 if key_bits == 64 else np.uint32
    top = key_bits - 8
    low_bits = key_bits - 8 * level
    b = [0x80, 0x40][:level]
    prefix = 0
    for i, d in enumerate(b):
        prefix |= d << (key_bits - 8 * (i + 1))
    below = int(rng.integers(0, k)) if k > 1 else 0
    rest = row_len - n - below
    bucket = prefix | rng.integers(0, 1 << min(low_bits, 62), n, dtype=np.uint64).astype(np.uint64)
    lo = rng.integers(0, 0x80, below, dtype=np.uint64) << np.uint64(top)  # below the bucket at level 1
    if level == 2:
        # the rest of the level-1 bucket (so S_1 > n): above the level-2 bucket
        hi = (np.uint64(0x80 << top) | (rng.integers(0x41, 0x100, rest, dtype=np.uint64) << np.uint64(top - 8))
              | rng.integers(0, 1 << (top - 8), rest, dtype=np.uint64))
    else:
        hi = rng.integers(0x81, 0x100, rest, dtype=np.uint64) << np.uint64(top)
    row = np.concatenate([lo, bucket, hi]).astype(dt)
    return row[rng.permutation(row_len)]
