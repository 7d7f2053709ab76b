"""Inputs structured by position: sorted runs, single-digit tiles, lone outliers and tile-local hot digits.

The DigitBinningPass's data-dependent work is per tile (its digit counts, its hot digit, its few-bins scatter runs, the
lookback over its predecessors' counts), and inputs drawn independently per position give every tile the global digit
histogram.  These generators put chosen digits at chosen positions instead.

Every input is built as a radix image: the unsigned key whose ascending order is the requested order
(tests.oraclelib.to_radix), held in an int64 tensor (16- and 32-bit images as non-negative values, 64-bit ones in two's
complement); to_bits turns it into the typed bits a sort takes.  A generator puts its structure into the digits of ONE
digit place p and holds every other place constant, so p is the only pass the plan executes and that pass (the first
executed one: it encodes typed keys and makes an argsort's indices) sees the structure as generated.  whole_keys
structures whole keys instead, and every place executes.

A generator takes n, the tile size T, the layout of the digit places, the place p and a seed, and returns the image and
the plan it promises: the places the scan kernel skips (all n keys share the digit), the places it calls hot (n >= 2^22
and one bin holds at least n/8 keys) and the number of executed passes.  expected_plan restates the scan kernel's rule
from the global histogram; tests/test_structured_inputs_cpu.py checks that both agree and that every input has the
tile-level property it claims."""
from typing import NamedTuple

import torch

from tests import bigcheck

HOT_MIN_N = 1 << 22  # the scan kernel calls no pass hot below this n
# tile size T of a DigitBinningPass -> keys per thread K (a warp's row of the tile holds 32 K keys):
# 16,384 = u32 keys, 12,288 = 16-bit keys, 8,192 = u32 pairs and argsort, u64 keys, 16-bit pairs, 64-bit pairs
KEYS_PER_THREAD = {16384: 32, 12288: 24, 8192: 16}


class Layout(NamedTuple):
    width: int     # key bits: 16, 32 or 64
    places: tuple  # (shift, bits) of every digit place, least significant first


class Plan(NamedTuple):
    skip: int      # bit p: place p is skipped
    hot: int       # bit p: place p runs in the HOT kernel (when hot passes are on)
    executed: int  # number of executed passes


def layout(width, begin=0, end=None):
    """the digit places of the bit range [begin, end): 8-bit places from begin, the last one narrower when the range is
    not a multiple of 8 bits"""
    end = width if end is None else end
    return Layout(width, tuple((b, min(8, end - b)) for b in range(begin, end, 8)))


def digit(image, place):
    shift, bits = place
    return (image >> shift) & ((1 << bits) - 1)


def expected_plan(image, places):
    """scan_kernel's plan: a place whose bins hold all n keys in one is skipped; otherwise it is hot when n >= 2^22 and a
    bin holds at least n/8 keys"""
    n = image.numel()
    skip = hot = 0
    for p, place in enumerate(places):
        c = int(torch.bincount(digit(image, place), minlength=1 << place[1]).max())
        if c == n:
            skip |= 1 << p
        elif n >= HOT_MIN_N and 8 * c >= n:
            hot |= 1 << p
    return Plan(skip, hot, len(places) - bin(skip).count("1"))


def to_bits(image, width, kind, descending=False):
    """the typed bits (an int16, int32 or int64 tensor) whose radix image is `image`; kind "u", "i" or "f" (16-bit
    floats: bfloat16 and float16 order their bits alike)"""
    if width == 64:
        return bigcheck.from_radix64(image, kind, descending)
    if width == 16:
        return bigcheck.from_radix16(image.to(torch.int32), kind + "16", descending)
    u = image ^ 0xFFFFFFFF if descending else image  # oraclelib.from_radix for 32-bit images
    if kind == "i":
        u = u ^ 0x80000000
    elif kind == "f":
        u = torch.where(u >= 0x80000000, u ^ 0x80000000, u ^ 0xFFFFFFFF)
    return ((u ^ 0x80000000) - 0x80000000).to(torch.int32)


def ordered(image, width):
    """a tensor whose signed order is the image's unsigned order"""
    return bigcheck.ordered(image) if width == 64 else image


# ---- sizes ---------------------------------------------------------------------------------------------------------------
def hot_n(T):
    """past 2^22 (the HOT kernel's threshold) by three tiles and a ragged remainder"""
    return HOT_MIN_N + 3 * T + T // 3 + 1


def whole_tiles_n(T):
    """the least n >= 2^22 that is a multiple of 8 T: whole tiles, and n/8 is whole tiles too"""
    return -(-HOT_MIN_N // (8 * T)) * 8 * T


def run_lengths(T):
    """one key, around a warp's 32, a warp's row of the tile (32 K), T/8 (the hot-digit threshold), around a tile, 3T/2"""
    return [1, 31, 32, 33, 32 * KEYS_PER_THREAD[T], T // 8, T - 1, T, T + 1, 3 * T // 2]


# ---- building blocks -----------------------------------------------------------------------------------------------------
def _rng(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def _randint(g, hi, size):
    return torch.randint(0, hi, (size,), generator=g, device=g.device, dtype=torch.int64)


def _s64(v):
    return v - (1 << 64) if v >= 1 << 63 else v


def _words(g, n, width):
    if width == 64:
        return (_randint(g, 1 << 32, n) << 32) | _randint(g, 1 << 32, n)
    return _randint(g, 1 << width, n)


def _bins(lay, p):
    return 1 << lay.places[p][1]


def _avoiding(g, n, nbins, avoid):
    """n digits drawn uniformly from the bins other than the (distinct) ones in `avoid`"""
    r = _randint(g, nbins - len(avoid), n)
    for a in sorted(avoid):
        r += (r >= a).long()
    return r


def _two(g, nbins):
    a = int(_randint(g, nbins, 1))
    return a, int(_avoiding(g, 1, nbins, [a]))


def tile_ranks(n, T, g):
    """a random order of the positions inside every tile: rank[i] in [0, keys of i's tile)"""
    tile = torch.arange(n, device=g.device) // T
    by = torch.argsort(tile.double() + torch.rand(n, generator=g, device=g.device, dtype=torch.float64))
    rank = torch.empty(n, dtype=torch.int64, device=g.device)
    rank[by] = torch.arange(n, device=g.device) - tile[by] * T
    return rank, tile


def compose(d, lay, p, g):
    """the image whose place p holds the digits d and every other place one random constant digit; bits outside the
    places are random (bit ranges: they ride along, and show stability)"""
    img = _words(g, d.numel(), lay.width)
    for q, (shift, bits) in enumerate(lay.places):
        img &= ~_s64(((1 << bits) - 1) << shift)
        if q == p:
            img |= d.to(torch.int64) << shift
        else:
            img |= _s64(int(_randint(g, 1 << bits, 1)) << shift)
    return img


def _single(d, lay, p, g, hot):
    every = (1 << len(lay.places)) - 1
    return compose(d, lay, p, g), Plan(every & ~(1 << p), (1 << p) if hot else 0, 1)


def _hot(n):
    return n >= HOT_MIN_N


def _ceil(a, b):
    return -(-a // b)


# ---- generators: structure in place p ------------------------------------------------------------------------------------
RUN_ORDERS = ("asc", "desc", "random")


def runs(n, T, lay, p, seed, R, order, device="cpu"):
    """digit (i // R) mod bins: ascending ("asc"), descending ("desc"), or one random digit per run ("random").  Hot only
    when the digit has at most 8 bins (then some bin holds n/8 keys)."""
    g = _rng(seed, device)
    nb = _bins(lay, p)
    j = torch.arange(n, device=device) // R
    if order == "asc":
        d = j % nb
    elif order == "desc":
        d = nb - 1 - j % nb
    else:
        rd = _randint(g, nb, int(j[-1]) + 2)
        rd[1] = (rd[0] + 1) % nb  # the first two runs differ: the place is never constant
        d = rd[j]
    return _single(d, lay, p, g, _hot(n) and nb <= 8)


def tile_blocks(n, T, lay, p, seed, device="cpu"):
    """every tile holds one digit, drawn at random; a quarter of the tiles repeat the digit of the tile before"""
    g = _rng(seed, device)
    nb = _bins(lay, p)
    tiles = -(-n // T)
    td = _randint(g, nb, tiles)
    repeat = torch.rand(tiles, generator=g, device=device) < 0.25
    repeat[0] = False
    src = torch.where(repeat, 0, torch.arange(tiles, device=device)).cummax(0).values
    return _single(td[src][torch.arange(n, device=device) // T], lay, p, g, _hot(n) and nb <= 8)


def outlier(n, T, lay, p, seed, pos, above, device="cpu"):
    """one digit everywhere but at `pos`: there a digit above the common one (common 0, outlier 1), or below it (common:
    the top bin, the digit of the ragged tile's all-ones padding; outlier the bin below).  Executed, and hot from 2^22."""
    g = _rng(seed, device)
    nb = _bins(lay, p)
    common, odd = (0, 1) if above else (nb - 1, nb - 2)
    d = torch.full((n,), common, dtype=torch.int64, device=device)
    d[pos] = odd
    return _single(d, lay, p, g, _hot(n))


def hot_block(n, T, lay, p, seed, extra, device="cpu"):
    """the first ceil(n/8) + extra keys share one digit h, the rest are uniform: the pass is hot, while the tiles after the
    block have no digit of T/8 keys"""
    g = _rng(seed, device)
    nb = _bins(lay, p)
    d = _randint(g, nb, n)
    d[: -(-n // 8) + extra] = int(_randint(g, nb, 1))
    return _single(d, lay, p, g, _hot(n))


def local_hot_counts(T):
    """the count of a tile's own majority digit in tile_local_hot, tile by tile (cycled): from the threshold to all T"""
    return [T // 8, T // 8 + 1, T // 2, T - 1, T]


def tile_local_hot(n, T, lay, p, seed, device="cpu"):
    """a global hot block of digit h in the leading whole tiles (at least ceil(n/8) keys); every later tile has its own
    majority digit m != h with local_hot_counts(T) keys at random positions, the rest uniform over the digits but m"""
    g = _rng(seed, device)
    nb = _bins(lay, p)
    tiles = _ceil(n, T)
    h = int(_randint(g, nb, 1))
    m = _avoiding(g, tiles, nb, [h])
    counts = torch.tensor(local_hot_counts(T), device=device)[torch.arange(tiles, device=device) % 5]
    rank, tile = tile_ranks(n, T, g)
    rest = _randint(g, nb - 1, n)
    rest += (rest >= m[tile]).long()
    d = torch.where(rank < counts[tile], m[tile], rest)
    d[: _ceil(_ceil(n, 8), T) * T] = h
    return _single(d, lay, p, g, _hot(n))


def tile_threshold(n, T, lay, p, seed, k, lead, device="cpu"):
    """every tile holds exactly k keys of one digit m at random positions, the others uniform over the digits but m and h
    (n a multiple of T: with k = T/8 m's global bin is exactly n/8).  lead: the first n/8 keys (whole tiles) hold another
    digit h instead, which makes the pass hot for either k."""
    assert n % T == 0 and (not lead or n % (8 * T) == 0)
    g = _rng(seed, device)
    nb = _bins(lay, p)
    m, h = _two(g, nb)
    rank, _ = tile_ranks(n, T, g)
    d = torch.where(rank < k, m, _avoiding(g, n, nb, [m, h]))
    if lead:
        d[: n // 8] = h
    return _single(d, lay, p, g, _hot(n) and (lead or 8 * k >= T))


def tie_counts(T):
    """the equal counts of tile_tie's two digits, tile by tile (cycled)"""
    return [T // 8, T // 4, T // 2]


def tile_tie(n, T, lay, p, seed, device="cpu"):
    """every tile holds two digits a < b with equal counts (tie_counts(T)) at random positions, the rest uniform over the
    other digits (n a multiple of T); a holds at least n/8 keys, so the pass is hot"""
    assert n % T == 0
    g = _rng(seed, device)
    nb = _bins(lay, p)
    a, b = sorted(_two(g, nb))
    rank, tile = tile_ranks(n, T, g)
    c = torch.tensor(tie_counts(T), device=device)[tile % 3]
    d = torch.where(rank < c, a, torch.where(rank < 2 * c, b, _avoiding(g, n, nb, [a, b])))
    return _single(d, lay, p, g, _hot(n))


def global_boundary(n, T, lay, p, seed, c, device="cpu"):
    """exactly c keys of one digit h at random positions, the rest uniform over the other digits: hot when n >= 2^22 and
    8c >= n"""
    g = _rng(seed, device)
    nb = _bins(lay, p)
    h = int(_randint(g, nb, 1))
    d = _avoiding(g, n, nb, [h])
    d[torch.randperm(n, generator=g, device=device)[:c]] = h
    return _single(d, lay, p, g, _hot(n) and 8 * c >= n)


# ---- whole keys: every place executes ------------------------------------------------------------------------------------
WHOLE_SHAPES = ["sorted", "reversed", "nearly", "runs8", "organ"]


def _sorted(v, width, descending=False):
    return v[torch.sort(ordered(v, width), descending=descending, stable=True).indices]


def whole_keys(n, T, lay, seed, shape, device="cpu"):
    """uniform keys arranged as a whole: sorted, reversed, nearly sorted (n // 100 disjoint random transpositions), 8
    concatenated sorted runs, or organ pipe (the first half ascending, the second descending).  No place is constant or
    hot."""
    g = _rng(seed, device)
    v = _sorted(_words(g, n, lay.width), lay.width)
    if shape == "reversed":
        v = v.flip(0)
    elif shape == "nearly":
        m = n // 100
        sel = torch.randperm(n, generator=g, device=device)[: 2 * m]
        perm = torch.arange(n, device=device)
        perm[sel[:m]], perm[sel[m:]] = sel[m:], sel[:m]
        v = v[perm]
    elif shape == "runs8":
        v = v[torch.randperm(n, generator=g, device=device)]
        for k in range(8):
            v[k * n // 8:(k + 1) * n // 8] = _sorted(v[k * n // 8:(k + 1) * n // 8], lay.width)
    elif shape == "organ":
        v = v[torch.randperm(n, generator=g, device=device)]
        v[: n // 2] = _sorted(v[: n // 2], lay.width)
        v[n // 2:] = _sorted(v[n // 2:], lay.width, descending=True)
    return v, Plan(0, 0, len(lay.places))


# ---- checks shared by the CPU tests --------------------------------------------------------------------------------------
def tile_counts(d, T, nbins):
    """[tiles, nbins] digit counts of every tile (the ragged last one counts its live keys only)"""
    tile = torch.arange(d.numel(), device=d.device) // T
    return torch.bincount(tile * nbins + d, minlength=(-(-d.numel() // T)) * nbins).view(-1, nbins)
