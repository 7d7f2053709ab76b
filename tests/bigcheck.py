"""Chunked checks for sorts too large to sort again or copy to the host: every check walks the output `chunk` elements
(or whole rows) at a time, so no torch op sees more than `chunk` elements of it.

Keys are compared through their radix image: the unsigned key whose ascending order is the requested order of the typed
value (tests.oraclelib.to_radix and tests.test_gpu_keys16.radix16, restated here in torch so they run on the device).  A
64-bit image is kept in an int64 container, a 32-bit one in int64 (0 .. 2^32 - 1) and a 16-bit one in int32 (0 .. 65535);
ordered() turns any of them into a tensor whose signed order is the key order.  Every checker reads keys as raw bits
(float NaNs compare unequal to themselves)."""
import torch

SIGN64 = -(1 << 63)
MASK32 = 0xFFFFFFFF
_INT_OF_WIDTH = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def bits_of(t: torch.Tensor) -> torch.Tensor:
    """the same memory as the signed integer container of its width"""
    return t.view(_INT_OF_WIDTH[t.element_size()])


# ---- radix images --------------------------------------------------------------------------------------------------------
def to_radix64(bits: torch.Tensor, kind: str, descending: bool = False) -> torch.Tensor:
    """oraclelib.to_radix for 64-bit containers: kind "u", "i" or "f"; the uint64 image in an int64 container"""
    u = bits_of(bits)
    if kind == "i":
        u = u ^ SIGN64
    elif kind == "f":
        u = torch.where(u < 0, ~u, u | SIGN64)
    return ~u if descending else u


def from_radix64(r: torch.Tensor, kind: str, descending: bool = False) -> torch.Tensor:
    """inverse of to_radix64: the int64 bits whose radix image is `r`"""
    u = ~r if descending else r
    if kind == "i":
        u = u ^ SIGN64
    elif kind == "f":
        u = torch.where(u < 0, u ^ SIGN64, ~u)
    return u


def as_int32(u: torch.Tensor) -> torch.Tensor:
    """32-bit patterns held as int64 0 .. 2^32 - 1, as the int32 container of the same bits"""
    return ((u ^ 0x80000000) - 0x80000000).to(torch.int32)


def to_radix32(bits: torch.Tensor, kind: str, descending: bool = False) -> torch.Tensor:
    """oraclelib.to_radix for 32-bit containers: kind "u", "i" or "f"; the uint32 image as int64 (0 .. 2^32 - 1)"""
    u = bits_of(bits).to(torch.int64) & MASK32
    if kind == "i":
        u = u ^ 0x80000000
    elif kind == "f":
        u = torch.where(u >= 0x80000000, u ^ MASK32, u | 0x80000000)
    return u ^ MASK32 if descending else u


def from_radix32(r: torch.Tensor, kind: str, descending: bool = False) -> torch.Tensor:
    """inverse of to_radix32: the int32 bits whose radix image is `r` (int64, 0 .. 2^32 - 1)"""
    u = r ^ MASK32 if descending else r
    if kind == "i":
        u = u ^ 0x80000000
    elif kind == "f":
        u = torch.where(u >= 0x80000000, u ^ 0x80000000, u ^ MASK32)
    return as_int32(u)


def radix16(bits: torch.Tensor, key_type: str, descending: bool = False) -> torch.Tensor:
    """test_gpu_keys16.radix16 for 16-bit containers (key_type "u16", "i16", "f16" or "bf16"): the image as int32"""
    u = bits_of(bits).to(torch.int32) & 0xFFFF
    if key_type == "i16":
        u = u ^ 0x8000
    elif key_type in ("f16", "bf16"):
        u = torch.where(u >= 0x8000, u ^ 0xFFFF, u | 0x8000)
    return u ^ 0xFFFF if descending else u


def from_radix16(r: torch.Tensor, key_type: str, descending: bool = False) -> torch.Tensor:
    """inverse of radix16: the int16 bits whose radix image is `r` (int32, 0 .. 65535)"""
    u = r ^ 0xFFFF if descending else r
    if key_type == "i16":
        u = u ^ 0x8000
    elif key_type in ("f16", "bf16"):
        u = torch.where(u >= 0x8000, u ^ 0x8000, u ^ 0xFFFF)
    return ((u ^ 0x8000) - 0x8000).to(torch.int16)


def key_radix(key_type: str, descending: bool = False):
    """the radix image function of a key type ("u16" .. "bf16", "u32", "i32", "f32", "u64", "i64", "f64")"""
    if key_type in ("u64", "i64", "f64"):
        return lambda bits: to_radix64(bits, key_type[0], descending)
    if key_type in ("u32", "i32", "f32"):
        return lambda bits: to_radix32(bits, key_type[0], descending)
    return lambda bits: radix16(bits, key_type, descending)


def ordered(r: torch.Tensor) -> torch.Tensor:
    """a radix image as a tensor whose signed order is its unsigned order (16-bit images in int32 already are, and 32-bit
    ones in int64 keep their order with the sign bit set)"""
    return r ^ SIGN64 if r.dtype == torch.int64 else r


# ---- an affine permutation of 32-bit keys and its sort ---------------------------------------------------------------------
# key[i] = (a i + b) mod 2^bits, a odd, for i < n <= 2^bits: n distinct keys, and the keys of consecutive positions run
# through every residue of the low byte, so every 256 aligned positions hold each low byte once.  The ascending sort is
# known without a sort: with M the m = 2^bits - n values left out (those of i = n .. 2^bits - 1), sorted, output position
# p holds the p-th value not in M, which is p + #{j : M[j] - j <= p}.
def affine_keys(a: int, b: int, lo: int, hi: int, bits: int = 32, device=None) -> torch.Tensor:
    """the keys of positions [lo, hi) as int64 (0 .. 2^bits - 1); a < 2^31, so that a i fits int64 for every i < 2^32"""
    assert a % 2 == 1 and 0 < a < (1 << 31)
    i = torch.arange(lo, hi, dtype=torch.int64, device=device)
    return (a * i + b) & ((1 << bits) - 1)


def affine_gaps(a: int, b: int, n: int, bits: int = 32, device=None) -> torch.Tensor:
    """M[j] - j (non-decreasing) for the sorted values M that the n keys leave out"""
    m = torch.sort(affine_keys(a, b, n, 1 << bits, bits, device)).values
    return m - torch.arange(m.numel(), dtype=torch.int64, device=device)


def affine_sorted(gaps: torch.Tensor, lo: int, hi: int) -> torch.Tensor:
    """positions [lo, hi) of the ascending sort of the n keys, as int64"""
    p = torch.arange(lo, hi, dtype=torch.int64, device=gaps.device)
    return p + torch.searchsorted(gaps, p, right=True)


def sort_by_low_byte(t: torch.Tensor) -> None:
    """reorders the keys of `t` in place, stable, by their low byte: a window of such keys concentrates each digit of place 0"""
    t.copy_(t[torch.sort(t & 0xFF, stable=True).indices])


# ---- checkers ------------------------------------------------------------------------------------------------------------
def _require(ok: torch.Tensor, what: str, first: int = 0, row_len: int = 0) -> None:
    """fails naming the first element where `ok` is false; `first`: the position of ok's first element in the output"""
    if bool(ok.all()):
        return
    i = first + int(torch.nonzero(~ok.reshape(-1))[0, 0])
    where = f"row {i // row_len}, column {i % row_len}" if row_len else f"element {i}"
    raise AssertionError(f"{what}: first at output {where}")


def positions(payload: torch.Tensor) -> torch.Tensor:
    """payloads as int64 positions: int32 containers hold unsigned 32-bit words (positions >= 2^31 read as negative)"""
    return payload.long() & 0xFFFFFFFF if payload.dtype == torch.int32 else payload.long()


def check_sorted_by_position(out: torch.Tensor, payload: torch.Tensor, src: torch.Tensor, radix, chunk: int) -> None:
    """`out` with `payload` must be exactly the stable sort of `src` with payload = input position.  It is when the radix
    image of `out` ascends, every payload p is in [0, n), src[p] == out, and payloads strictly ascend inside every run of
    equal keys: payloads of different keys differ because their keys do, those of equal keys because they ascend, so the n
    payloads are a permutation of 0 .. n-1, and the order of equal keys is the input's.  Chunks overlap by one element, so
    the order and runs of equal keys are also checked across chunk borders."""
    n = src.numel()
    assert out.numel() == n and payload.numel() == n, f"{out.numel()} keys and {payload.numel()} payloads for {n} inputs"
    out, src = bits_of(out), bits_of(src)
    for a in range(0, n, chunk):
        b = min(a + chunk, n)
        e = min(b + 1, n)
        r = ordered(radix(out[a:e]))
        _require(r[1:] >= r[:-1], "radix image descends", a)
        p = positions(payload[a:e])
        _require((p >= 0) & (p < n), f"payload outside [0, {n})", a)
        _require(src[p[:b - a]] == out[a:b], "src[payload] != out", a)
        _require((p[1:] > p[:-1]) | (r[1:] != r[:-1]), "payloads do not ascend inside a run of equal keys", a)
        del r, p


def check_sorted_keys16(out: torch.Tensor, src: torch.Tensor, radix, chunk: int) -> None:
    """`out` must be the sort of `src` (16-bit keys): its radix image ascends (chunks overlap by one element) and holds
    every one of the 65,536 radix values as often as the input does"""
    n = src.numel()
    assert out.numel() == n, f"{out.numel()} output keys for {n} inputs"
    h_in = torch.zeros(1 << 16, dtype=torch.int64, device=src.device)
    h_out = torch.zeros_like(h_in)
    for a in range(0, n, chunk):
        b = min(a + chunk, n)
        e = min(b + 1, n)
        r = radix(out[a:e])
        _require(r[1:] >= r[:-1], "radix image descends", a)
        h_out += torch.bincount(r[:b - a], minlength=1 << 16)
        h_in += torch.bincount(radix(src[a:b]), minlength=1 << 16)
        del r
    bad = torch.nonzero(h_in != h_out)
    if bad.numel():
        v = int(bad[0, 0])
        raise AssertionError(f"radix value {v:#06x}: {int(h_in[v])} in the input, {int(h_out[v])} in the output "
                             f"({bad.numel()} values differ)")


def check_topk_rows(vals: torch.Tensor, idx: torch.Tensor, src: torch.Tensor, radix, k: int, sorted: bool,
                    chunk: int) -> None:
    """`vals` and `idx` ([rows, k]) must be the first k columns of torch.sort(stable=True) of every row's radix image in `src`
    ([rows, row_len]): the positions in that order when `sorted`, else the same positions in any order (each row's pairs
    are sorted by position first, and compared with the reference's first k sorted by position); and every key must be the
    bits of src at its position.  Whole rows at a time (at least one row per step)."""
    row_len = src.shape[-1]
    s2 = bits_of(src).reshape(-1, row_len)
    v2, i2 = bits_of(vals).reshape(-1, k), idx.reshape(-1, k)
    assert k <= row_len and v2.shape == i2.shape == (s2.shape[0], k), f"shapes {vals.shape}, {idx.shape} and {src.shape}"
    rows = s2.shape[0]
    step = max(1, chunk // row_len)
    for a in range(0, rows, step):
        b = min(a + step, rows)
        want = torch.sort(ordered(radix(s2[a:b])), dim=-1, stable=True).indices[:, :k]
        got_i, got_v = positions(i2[a:b]), v2[a:b]
        if not sorted:
            got_i, by_pos = torch.sort(got_i, dim=-1)
            got_v = torch.gather(got_v, 1, by_pos)
            want = torch.sort(want, dim=-1).values
        _require(got_i == want, "positions differ from the stable sort of the row cut to k", a * k, k)
        _require(got_v == torch.gather(s2[a:b], 1, want), "keys differ from the row's keys at those positions", a * k, k)
        del want, got_i, got_v


def check_rows(out: torch.Tensor, idx, src: torch.Tensor, radix, chunk: int) -> None:
    """every row of `out` (and of `idx`, unless None) must be torch.sort(stable=True) of that row's radix image in `src`,
    compared bit for bit, whole rows at a time (at least one row per step)"""
    row_len = src.shape[-1]
    s2, o2 = bits_of(src).reshape(-1, row_len), bits_of(out).reshape(-1, row_len)
    i2 = idx.reshape(-1, row_len) if idx is not None else None
    assert o2.shape == s2.shape and (i2 is None or i2.shape == s2.shape), f"shapes {out.shape} and {src.shape}"
    rows = s2.shape[0]
    step = max(1, chunk // row_len)
    for a in range(0, rows, step):
        b = min(a + step, rows)
        want = torch.sort(ordered(radix(s2[a:b])), dim=-1, stable=True)
        _require(ordered(radix(o2[a:b])) == want.values, "keys differ from the stable sort of the row", a * row_len,
                 row_len)
        if i2 is not None:
            _require(i2[a:b].long() == want.indices, "indices differ from the stable sort of the row", a * row_len,
                     row_len)
        del want
