"""Chunked checks for sorts too large to sort again or copy to the host: every check walks the output `chunk` elements
(or whole rows) at a time, so no torch op sees more than `chunk` elements of it.

Keys are compared through their radix image: the unsigned key whose ascending order is the requested order of the typed
value (tests.oraclelib.to_radix and tests.test_gpu_keys16.radix16, restated here in torch so they run on the device).  A
64-bit image is kept in an int64 container and a 16-bit one in int32 (0 .. 65535); ordered() turns either into a tensor
whose signed order is the key order.  Every checker reads keys as raw bits (float NaNs compare unequal to themselves)."""
import torch

SIGN64 = -(1 << 63)
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
    """the radix image function of a key type of 16 or 64 bits ("u16" .. "bf16", "u64", "i64", "f64")"""
    if key_type in ("u64", "i64", "f64"):
        return lambda bits: to_radix64(bits, key_type[0], descending)
    return lambda bits: radix16(bits, key_type, descending)


def ordered(r: torch.Tensor) -> torch.Tensor:
    """a radix image as a tensor whose signed order is its unsigned order (16-bit images in int32 already are)"""
    return r ^ SIGN64 if r.dtype == torch.int64 else r


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
