"""One sorter handle shared by every entry point, eagerly, inside one CUDA graph and beside other work.  -m gpu

The module calls send argsort, argsort16, sort_rows, topk, sort_segments and topk_segments through one cached (4, 4)
handle per stream, and the call families use the same parts of a handle in different ways: the alternate key buffer
(ping-pong keys, the fused pass's 256 gapped regions, the segment calls' class lists), the control block (global
histogram, tickets 0-3 of the passes, the fused ticket and abort word in slots 4-5, the scratch words of validate and of
the segment calls' class counts, the device plan), the epoch-stamped descriptors (cleared by captured sorts over their own
tiles: 16,384 keys for u32 keys, 12,288 for 16-bit keys, 8,192 for pairs, argsorts and 64-bit keys) and the compact
reductions.  Here each call directly follows one that used the same state differently:
  1. about 40 eager calls of every family on one (4, 4) handle, first with a host sync and a plan check after each call,
     then all enqueued before the first check, in both rank modes;
  2. the same on a (8, 4) handle with 64-bit sorts, rows, top-k and segments of every width, and a refused argsort16;
  3. one graph holding a fused sort, argsort16, pairs, segment top-k, segment sort and row top-k, replayed with new
     contents and offsets, eager calls of other families between replays, and eager sorts at the captured epochs and
     across the epoch wrap-around;
  4. one handle and stream per family, three rounds enqueued at once beside a loop of matmuls;
  5. the module calls: six functions on one cached handle, and a cache that grows under a live graph.

Every output is compared element by element with the stable sort of the radix image (numpy, or torch.sort(stable=True) on
sign-flipped keys from 2^20 keys): keys bit for bit, payloads and indices exactly, argsort inputs bit-identical, top-k
padding exactly, and sentinel-filled positions outside every segment untouched."""
import numpy as np
import pytest
import torch

from tests.test_fused_layout_cpu import region_keys
from tests.test_gpu_fused_first_pass import WINDOW, with_place0_bin
from tests.test_gpu_graphs_and_streams import radix_inputs
from tests.test_gpu_large_n import GiB, release, require
from tests.test_gpu_rows import TYPES, dev, host, radix, random_bits, same, typed_input
from tests.test_gpu_sort_segments import GUARD, SENTINEL_IDX, call as sort_segments_call, framed_idx, framed_keys
from tests.test_gpu_sort_segments import oracle as sort_segments_oracle, sentinel_bits
from tests.test_gpu_topk import from_radix
from tests.test_gpu_topk_segments import oracle as topk_segments_oracle

pytestmark = pytest.mark.gpu

INVALID_ARG = -1
EPOCH_MAX = (1 << 24) - 1
DEVICE_ORACLE_MIN = 1 << 20
SIGNED = {2: torch.int16, 4: torch.int32, 8: torch.int64}
F = 1 << 21                  # fused u32 keys sorts: 128 tiles of 16,384 keys
NB = (1 << 21) + 4099        # the larger sorts: 257 tiles of 8,192, 171 of 12,288, 129 of 16,384
NS = (1 << 20) + 77          # the smaller ones
SLACK = 1 << 16              # every handle holds more than its largest sort


@pytest.fixture(scope="module")
def g():
    import gpusorting_b200 as g

    return g


# ---- references -------------------------------------------------------------------------------------------------------
def order_of(bits, t, descending=False):
    """the stable order of the radix image: numpy below 2^20 keys, torch.sort(stable=True) on sign-flipped keys above"""
    r = radix(bits, t, descending)
    if r.size < DEVICE_ORACLE_MIN:
        return np.argsort(r, kind="stable")
    w = r.dtype.itemsize * 8
    signed = (r ^ r.dtype.type(1 << (w - 1))).view(f"int{w}")
    return torch.sort(torch.from_numpy(signed).cuda(), stable=True)[1].cpu().numpy()


def device_order(x, t, descending=False):
    """the same on the device, for a device tensor x: the order and x's keys in its signed integer view"""
    b = x.view(SIGNED[x.element_size()])
    lo, hi = torch.iinfo(b.dtype).min, torch.iinfo(b.dtype).max
    kind = TYPES[t][3]
    s = b ^ lo if kind == "u" else torch.where(b < 0, b ^ hi, b) if kind == "f" else b
    if descending:
        s = ~s
    return torch.sort(s, stable=True)[1], b


def idx_host(idx):
    return idx.cpu().numpy().view(np.uint32)


def uniform(rng, n, t="u32"):
    return random_bits(rng, n, t)


def with_low_byte(rng, n, t, const_low):
    """bits whose radix image has a constant low byte (const_low) or a constant top byte (otherwise)"""
    c = TYPES[t][1]
    w = np.dtype(c).itemsize * 8
    r = random_bits(rng, n, t)
    top = c(0xFF << (w - 8))
    r = (r & ~c(0xFF)) | c(0x5A) if const_low else (r & ~top) | c(0x5A << (w - 8))
    return from_radix(r, t)


def ragged(rng, kind, n_target):
    """segment lengths: log-uniform up to 2^15, short (1-300), or runs of empty segments between short and long ones"""
    if kind == "log-uniform":
        return np.exp(rng.uniform(0, np.log(1 << 15), max(1, n_target // 3000))).astype(np.int64)
    if kind == "short":
        return rng.integers(2, 257, n_target // 128)
    lens = rng.integers(0, 3000, n_target // 1500)
    lens[rng.random(lens.size) < 0.5] = 0
    return lens


def offsets_of(lens, start=0):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + start


# ---- the calls: each enqueues on the current stream and returns the check of its result -----------------------------------
def keys_u32(bits):
    def enqueue(s):
        t = dev(bits, "u32")
        s.sort_keys(t)
        return lambda: same(host(t, "u32"), np.sort(bits), "keys")
    return enqueue


def keys_typed(bits, t, descending):
    def enqueue(s):
        x = dev(bits, t)
        s.sort_keys_typed(x, t, descending)
        return lambda: same(host(x, t), bits[order_of(bits, t, descending)], "keys")
    return enqueue


def sort_bits(bits, begin, end):
    def enqueue(s):
        x = dev(bits, "u32")
        s.sort_bits(x, begin, end)
        part = (bits >> np.uint32(begin)) & np.uint32((1 << (end - begin)) - 1)
        return lambda: same(host(x, "u32"), bits[order_of(part, "u32")], "keys")
    return enqueue


def pairs(bits, t="u32", descending=False, typed=False):
    def enqueue(s):
        x = dev(bits, t)
        v = torch.arange(bits.size, dtype=torch.int32, device="cuda")
        s.sort_pairs_typed(x, v, t, descending) if typed else s.sort_pairs(x, v)

        def check():
            o = order_of(bits, t, descending)
            same(host(x, t), bits[o], "keys")
            same(idx_host(v), o, "payloads")
        return check
    return enqueue


def argsort(bits, t, descending=False):
    def enqueue(s):
        x = dev(bits, t)
        out, idx = s.argsort(x, t, descending)

        def check():
            o = order_of(bits, t, descending)
            same(host(x, t), bits, "input modified")
            same(host(out, t), bits[o], "keys")
            same(idx_host(idx), o, "indices")
        return check
    return enqueue


def keys16(bits, t, descending=False):
    def enqueue(s):
        x = dev(bits, t)
        s.sort_keys16(x, t, descending)
        return lambda: same(host(x, t), bits[order_of(bits, t, descending)], "keys")
    return enqueue


def pairs16(bits, t, descending=False):
    def enqueue(s):
        x = dev(bits, t)
        v = torch.arange(bits.size, dtype=torch.int32, device="cuda")
        s.sort_pairs16(x, v, t, descending)

        def check():
            o = order_of(bits, t, descending)
            same(host(x, t), bits[o], "keys")
            same(idx_host(v), o, "payloads")
        return check
    return enqueue


def argsort16(bits, t, descending=False):
    def enqueue(s):
        x = dev(bits, t)
        out, idx = s.argsort16(x, t, descending)

        def check():
            o = order_of(bits, t, descending)
            same(host(x, t), bits, "input modified")
            same(host(out, t), bits[o], "keys")
            same(idx_host(idx), o, "indices")
        return check
    return enqueue


def rows(bits2d, t, descending=False):
    def enqueue(s):
        x = dev(bits2d, t)
        vals, idx = s.sort_rows(x, t, descending)

        def check():
            o = np.argsort(radix(bits2d, t, descending), axis=-1, kind="stable")
            same(host(x, t), bits2d, "input modified")
            same(host(vals, t), np.take_along_axis(bits2d, o, axis=-1), "keys")
            same(idx_host(idx), o, "indices")
        return check
    return enqueue


def topk_rows(bits2d, t, k, largest):
    def enqueue(s):
        x = dev(bits2d, t)
        vals, idx = s.topk_rows(x, k, t, largest, True)

        def check():
            o = np.argsort(radix(bits2d, t, largest), axis=-1, kind="stable")[:, :k]
            same(host(vals, t), np.take_along_axis(bits2d, o, axis=-1), "keys")
            same(idx_host(idx), o, "indices")
        return check
    return enqueue


def topk_segments(bits, off, t, k, largest):
    def enqueue(s):
        x, offs = dev(bits, t), torch.from_numpy(off).cuda()
        vals, idx = s.topk_segments(x, offs, k, t, largest, True)

        def check():
            wk, wi = topk_segments_oracle(bits, off, k, t, largest)  # padding columns included
            same(host(vals, t), wk, "keys")
            same(idx_host(idx), wi, "indices")
        return check
    return enqueue


def sort_segments_framed(bits, off, t, descending, max_len):
    """through the C entry point into sentinel-filled, guarded outputs: positions outside every segment stay untouched"""
    def enqueue(s):
        src = framed_keys(bits, t)
        out = framed_keys(bits, t, np.full(bits.size, sentinel_bits(t), dtype=TYPES[t][1]))
        ix = framed_idx(bits.size)
        off_t = torch.from_numpy(off).cuda()
        assert sort_segments_call(s, src.ptr, out.ptr, ix.ptr, bits.size, off_t, off.size - 1, max_len, t, descending) == 0

        def check():
            keep = (off_t, src)  # noqa: F841  (alive until the call has run)
            sk = np.full(bits.size + 2 * GUARD, sentinel_bits(t), dtype=TYPES[t][1])
            si = np.full(bits.size + 2 * GUARD, SENTINEL_IDX, dtype=np.uint32)
            wk, wi = sort_segments_oracle(bits, off, bits.size, max_len, t, descending, sk[GUARD:-GUARD], si[GUARD:-GUARD])
            sk[GUARD:-GUARD], si[GUARD:-GUARD] = wk, wi
            same(src.host()[GUARD:-GUARD], bits, "input modified")
            same(out.host(), sk, "keys (sentinels outside the segments)")
            same(ix.host(), si, "indices (sentinels outside the segments)")
        return check
    return enqueue


def sort_segments_method(bits, off, t, descending, max_len):
    """OneSweepSorter.sort_segments on segments that cover the whole input (every output position is written)"""
    def enqueue(s):
        x, offs = dev(bits, t), torch.from_numpy(off).cuda()
        vals, idx = s.sort_segments(x, offs, t, descending, max_segment_len=max_len)

        def check():
            wk, wi = sort_segments_oracle(bits, off, bits.size, max_len, t, descending, bits, np.zeros(bits.size, np.uint32))
            same(host(vals, t), wk, "keys")
            same(idx_host(idx), wi, "indices")
        return check
    return enqueue


def segmented_sort(bits, off, max_len):
    def enqueue(s):
        x, offs = dev(bits, "u32"), torch.from_numpy(off).cuda()
        v = torch.arange(bits.size, dtype=torch.int32, device="cuda")
        s.segmented_sort(x, offs, values=v, max_segment_len=max_len)

        def check():
            end = int(off[-1])
            seg = np.repeat(np.arange(off.size - 1), np.diff(off))
            o = np.concatenate([np.lexsort((bits[:end], seg)), np.arange(end, bits.size)])
            same(host(x, "u32"), bits[o], "keys")
            same(idx_host(v), o, "payloads")
        return check
    return enqueue


def validate(bits, t):
    def enqueue(s):
        got = s.validate(dev(bits, t))  # reads its count back: synchronises the stream
        return lambda: same(np.array([got]), np.array([int(np.count_nonzero(bits[:-1] > bits[1:]))]), "inversions")
    return enqueue


def global_histogram(bits, t):
    def enqueue(s):
        h = s.global_histogram(dev(bits, t))

        def check():
            w = bits.dtype.itemsize
            want = [np.bincount(((bits >> bits.dtype.type(8 * p)) & bits.dtype.type(0xFF)).astype(np.int64), minlength=256)
                    for p in range(w)]
            same(h.cpu().numpy(), np.stack(want), "histogram")
        return check
    return enqueue


def binning_pass(bits, shift):
    def enqueue(s):
        src, dst = dev(bits, "u32"), torch.empty(bits.size, dtype=torch.int32, device="cuda")
        sv = torch.arange(bits.size, dtype=torch.int32, device="cuda")
        dv = torch.empty_like(sv)
        s.digit_binning_pass(src, dst, shift, src_values=sv, dst_values=dv)

        def check():
            o = np.argsort((bits >> np.uint32(shift)) & np.uint32(0xFF), kind="stable")
            same(host(dst, "u32"), bits[o], "keys")
            same(idx_host(dv), o, "payloads")
        return check
    return enqueue


def sort_host(bits):
    def enqueue(s):
        a = bits.copy()
        s.sort_host(a)
        return lambda: same(a, np.sort(bits), "keys")
    return enqueue


def refused_argsort16(bits):
    def enqueue(s):
        from gpusorting_b200 import OneSweepError

        with pytest.raises(OneSweepError) as e:
            s.argsort16(dev(bits, "bf16"), "bf16")
        assert e.value.status == INVALID_ARG
        return lambda: None
    return enqueue


# ---- the programs ------------------------------------------------------------------------------------------------------------
def run_program(s, steps, synced):
    """steps: (name, enqueue, plan or None, host_call).  synced: a host sync, the check and the plan after every call;
    otherwise everything is enqueued before the first check.  A host call runs on the handle's own stream, so the stream
    is drained before it (one sort in flight per handle).  plan: (last_skip_mask, last_executed_passes, last_fused_kept)."""
    pending = []
    for name, enqueue, plan, host_call in steps:
        if host_call:
            torch.cuda.synchronize()
        check = enqueue(s)
        if synced:
            torch.cuda.synchronize()
            checked(name, check)
            if plan is not None:
                got = (s.info("last_skip_mask"), s.info("last_executed_passes"), s.info("last_fused_kept"))
                assert got == plan, f"{name}: plan (skip mask, executed passes, fused kept) {got}, want {plan}"
        else:
            pending.append((name, check))
    torch.cuda.synchronize()
    for name, check in pending:
        checked(name, check)


def checked(name, check):
    try:
        check()
    except AssertionError as e:
        raise AssertionError(f"{name}: {e}") from None


def program_44(seed, max_n):
    rng = np.random.default_rng(seed)
    c = region_keys(F)
    u = lambda n, t="u32": uniform(rng, n, t)  # noqa: E731
    ti = lambda n, t: typed_input(rng, n, t)  # noqa: E731
    # (typed_input's ties fill one place-0 bin past its region: fused sorts that must stand take normal floats)
    normal32 = lambda n: rng.standard_normal(n).astype(np.float32).view(np.uint32)  # noqa: E731
    log_off = offsets_of(ragged(rng, "log-uniform", 1 << 20))
    gap_lens = ragged(rng, "empty runs", 400_000)
    gap_off = offsets_of(gap_lens, start=17)
    gap_off[gap_off.size // 2:] += 1000  # a gap between two segments
    full_off = offsets_of(rng.integers(0, 4, max_n))  # num_segments == max_n: the class lists fill the alt buffer
    short_off = offsets_of(ragged(rng, "short", 1 << 19))
    seg_off = offsets_of(rng.integers(0, 9000, 64))
    u64_off = offsets_of(ragged(rng, "empty runs", 300_000))
    big = (0, 4, 0)
    return [
        ("fused sort, kept", keys_u32(u(F)), (0, 4, 1), False),
        ("fused sort, late overflow: fallback", keys_u32(with_place0_bin(F, c + 1, F - WINDOW, seed)), (0, 4, 0), False),
        ("fused sort, kept, after a fallback", keys_u32(u(F)), (0, 4, 1), False),
        ("topk_segments f32 after a fused sort", topk_segments(ti(int(log_off[-1]), "f32"), log_off, "f32", 50, True), None, False),
        ("validate after a segment call", validate(u(NS), "u32"), None, False),
        ("sort_segments i32 after validate", sort_segments_framed(ti(int(gap_off[-1]) + 99, "i32"), gap_off, "i32", True, 16384),
         None, False),
        ("topk_segments bf16, num_segments == max_n, after a segment call",
         topk_segments(ti(int(full_off[-1]), "bf16"), full_off, "bf16", 4, True), None, False),
        ("sort_keys_typed f32 descending (fused) after the segment calls", keys_typed(normal32(F), "f32", True), (0, 4, 1), False),
        ("argsort i32 at NS: smaller, 8,192-key tiles", argsort(ti(NS, "i32"), "i32"), big, False),
        ("sort_keys16 f16 at NB, place 0 skipped: larger, 12,288-key tiles", keys16(with_low_byte(rng, NB, "f16", True), "f16"),
         (0b01, 1, 0), False),
        ("sort_pairs at NS: 8,192-key tiles", pairs(ti(NS, "u32")), big, False),
        ("sort_bits(0, 32), fused", sort_bits(u(F), 0, 32), (0, 4, 1), False),
        ("argsort f32 at NB", argsort(ti(NB, "f32"), "f32"), big, False),
        ("sort_bits(3, 22): three places and the copy-back", sort_bits(u(NS), 3, 22), (0, 3, 0), False),
        ("sort_pairs16 i16 descending, place 1 skipped", pairs16(with_low_byte(rng, NS, "i16", False), "i16", True),
         (0b10, 1, 0), False),
        ("argsort16 bf16 at NB", argsort16(ti(NB, "bf16"), "bf16"), (0, 2, 0), False),
        ("sort_rows f32 descending, warp path", rows(ti(1000 * 200, "f32").reshape(1000, 200), "f32", True), None, False),
        ("fused sort, early overflow: fallback", keys_u32(with_place0_bin(F, c + 1, 0, seed + 1)), (0, 4, 0), False),
        ("fused sort, kept, after a fallback (2)", keys_u32(u(F)), (0, 4, 1), False),
        ("topk_rows bf16, select path", topk_rows(ti(48 * 50_000, "bf16").reshape(48, 50_000), "bf16", 100, True), None, False),
        ("sort_rows i64, block path", rows(ti(64 * 3000, "i64").reshape(64, 3000), "i64"), None, False),
        ("topk_rows u32 smallest, warp path", topk_rows(ti(4000 * 100, "u32").reshape(4000, 100), "u32", 8, False), None, False),
        ("segmented_sort with payloads", segmented_sort(u(600_000), seg_off, 16384), None, False),
        ("global_histogram", global_histogram(u(NS), "u32"), None, False),
        ("digit_binning_pass, shift 8, with payloads", binning_pass(u(NS), 8), None, False),
        ("sort_host", sort_host(u(NS)), None, True),
        ("fused sort, kept, after the host sort", keys_u32(u(F)), (0, 4, 1), False),
        ("sort_segments f16, short segments", sort_segments_method(ti(int(short_off[-1]), "f16"), short_off, "f16", False, 256),
         None, False),
        ("validate a sorted array after a segment call", validate(np.sort(u(NS)), "u32"), None, False),
        ("topk_segments i32 smallest after validate", topk_segments(ti(int(gap_off[-1]) + 5, "i32"), gap_off, "i32", 100, False),
         None, False),
        ("argsort16 u16, single block", argsort16(ti(10_000, "u16"), "u16"), None, False),
        ("sort_keys16 bf16 at NS", keys16(ti(NS, "bf16"), "bf16"), (0, 2, 0), False),
        ("fused sort, middle overflow: fallback", keys_u32(with_place0_bin(F, c + 1, F // 2, seed + 2)), (0, 4, 0), False),
        ("sort_keys_typed f32, kept, after a fallback", keys_typed(normal32(F), "f32", False), (0, 4, 1), False),
        ("sort_segments u64", sort_segments_framed(ti(int(u64_off[-1]), "u64"), u64_off, "u64", False, 8192), None, False),
        ("topk_rows f64", topk_rows(ti(100 * 1000, "f64").reshape(100, 1000), "f64", 33, True), None, False),
        ("argsort f32 descending at NB", argsort(ti(NB, "f32"), "f32", True), big, False),
        ("sort_keys16 i16, three tiles and five keys", keys16(ti(3 * 12288 + 5, "i16"), "i16"), (0, 2, 0), False),
        ("sort_pairs at NB", pairs(ti(NB, "u32")), big, False),
        ("validate", validate(u(NS), "u32"), None, False),
    ]


def program_84(seed, max_n):
    rng = np.random.default_rng(seed)
    n = NS
    ti = lambda m, t: typed_input(rng, m, t)  # noqa: E731
    full_off = offsets_of(rng.integers(0, 3, max_n))  # num_segments == max_n
    log_off = offsets_of(ragged(rng, "log-uniform", 1 << 20))
    gap_off = offsets_of(ragged(rng, "empty runs", 300_000))
    hi_const = random_bits(rng, n, "u64") & np.uint64(0xFFFFFFFF) | np.uint64(0x5A5A5A5A << 32)
    top_only = random_bits(rng, n, "u64") & np.uint64(0xFF << 56) | np.uint64(0x00A5A5A5A5A5A5A5)
    low16_const = from_radix(random_bits(rng, n, "u64") & ~np.uint64(0xFFFF) | np.uint64(0x1234), "i64")
    all8 = (0, 8, 0)
    return [
        ("u64 sort_keys", keys_typed(random_bits(rng, n, "u64"), "u64", False), all8, False),
        ("topk_segments u64 after a sort", topk_segments(ti(int(log_off[-1]), "u64"), log_off, "u64", 64, True), None, False),
        ("sort_pairs_typed f64 descending", pairs(ti(n, "f64"), "f64", True, typed=True), all8, False),
        ("argsort16 on a (8, 4) sorter: INVALID_ARG", refused_argsort16(ti(1000, "bf16")), None, False),
        ("argsort i64 after the refused call", argsort(ti(n, "i64"), "i64"), all8, False),
        ("sort_rows u16, block path", rows(ti(500 * 300, "u16").reshape(500, 300), "u16"), None, False),
        ("sort_segments f32, num_segments == max_n", sort_segments_framed(ti(int(full_off[-1]), "f32"), full_off, "f32", True, 16384),
         None, False),
        ("u64 keys, high half constant", keys_typed(hi_const, "u64", False), (0xF0, 4, 0), False),
        ("validate u64", validate(random_bits(rng, n, "u64"), "u64"), None, False),
        ("topk_rows i64, select path", topk_rows(ti(64 * 20_000, "i64").reshape(64, 20_000), "i64", 64, True), None, False),
        ("sort_keys_typed i64, low 16 bits constant", keys_typed(low16_const, "i64", False), (0b11, 6, 0), False),
        ("topk_segments f16 smallest", topk_segments(ti(int(gap_off[-1]), "f16"), gap_off, "f16", 20, False), None, False),
        ("sort_host u64", sort_host(random_bits(rng, n, "u64")), None, True),
        ("sort_pairs u64", pairs(random_bits(rng, n, "u64"), "u64"), all8, False),
        ("sort_segments i16 descending", sort_segments_framed(ti(int(gap_off[-1]), "i16"), gap_off, "i16", True, 16384), None, False),
        ("topk_rows bf16, warp path", topk_rows(ti(3000 * 200, "bf16").reshape(3000, 200), "bf16", 5, True), None, False),
        ("argsort f64 descending, a third of the size", argsort(ti(n // 3, "f64"), "f64", True), all8, False),
        ("global_histogram u64", global_histogram(random_bits(rng, n, "u64"), "u64"), None, False),
        ("u64 keys, only the top byte varies", keys_typed(top_only, "u64", False), (0x7F, 1, 0), False),
        ("argsort u64 after a one-pass sort", argsort(random_bits(rng, n, "u64"), "u64"), all8, False),
        ("sort_rows f64 descending", rows(ti(200 * 1000, "f64").reshape(200, 1000), "f64", True), None, False),
    ]


def sorter_in_rank_mode(g, max_n, kb, vb, rank_mode):
    s = g.OneSweepSorter(max_n, kb, vb)
    if rank_mode == 0 and not s.info("atomic_order_ok"):
        s.close()
        pytest.skip("the atomic rank mode failed its self-test on this device")
    s.set_option("rank_mode", rank_mode)
    return s


@pytest.mark.parametrize("rank_mode", [0, 1])
def test_eager_program_on_one_44_handle(g, rank_mode):
    max_n = NB + SLACK
    require(g, "the (4, 4) program", max_n, 4, 4, 2 * GiB, 4 * GiB)
    with sorter_in_rank_mode(g, max_n, 4, 4, rank_mode) as s:
        run_program(s, program_44(10 + rank_mode, max_n), synced=True)
        run_program(s, program_44(20 + rank_mode, max_n), synced=False)
    release()


@pytest.mark.parametrize("rank_mode", [0, 1])
def test_eager_program_on_one_84_handle(g, rank_mode):
    max_n = NS + SLACK
    require(g, "the (8, 4) program", max_n, 8, 4, 2 * GiB, 4 * GiB)
    with sorter_in_rank_mode(g, max_n, 8, 4, rank_mode) as s:
        run_program(s, program_84(30 + rank_mode, max_n), synced=True)
        run_program(s, program_84(40 + rank_mode, max_n), synced=False)
    release()


# ---- 3. one graph mixing the families ------------------------------------------------------------------------------------------
NK = (1 << 20) + 5       # the graph's fused sort: 65 tiles of 16,384
N16 = (1 << 21) + 4099   # its argsort16: 257 tiles of 8,192, beyond the 129 tiles of 16,384 that cover its keys
NP = (1 << 20) - 3       # its pairs: 128 tiles of 8,192


def inputs16(rng, n):
    """radix images in replay order, each replay's first executed place the previous one's last (as radix_inputs does for
    wider keys): (name, radix image, skip mask)"""
    u = lambda: rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16)  # noqa: E731
    return [
        ("uniform", u(), 0),
        ("top byte only", (u() & np.uint16(0xFF00)) | np.uint16(0x5A), 0b01),
        ("low byte only", (u() & np.uint16(0xFF)) | np.uint16(0xA500), 0b10),
        ("uniform", u(), 0),
        ("constant top byte", (u() & np.uint16(0xFF)) | np.uint16(0x3C00), 0b10),
        ("low byte only", (u() & np.uint16(0xFF)) | np.uint16(0xC300), 0b10),
        ("all equal", np.full(n, 0x5AA5, np.uint16), 0b11),
        ("uniform", u(), 0),
    ]


class Graph:
    """the static tensors and the graph of section 3, on one (4, 4) handle"""

    def __init__(self, s, rng):
        self.s, self.rng = s, rng
        self.keys = torch.zeros(NK, dtype=torch.int32, device="cuda")
        self.k16 = torch.zeros(N16, dtype=torch.bfloat16, device="cuda")
        self.pk = torch.zeros(NP, dtype=torch.int32, device="cuda")
        self.pv = torch.zeros(NP, dtype=torch.int32, device="cuda")
        self.segs = 3000
        self.sx = torch.zeros(1 << 20, dtype=torch.float32, device="cuda")
        self.soff = torch.zeros(self.segs + 1, dtype=torch.int64, device="cuda")
        self.rx = torch.zeros(1 << 20, dtype=torch.int16, device="cuda")
        self.roff = torch.zeros(self.segs + 1, dtype=torch.int64, device="cuda")
        self.tx = torch.zeros(64, 20_000, dtype=torch.float16, device="cuda")
        self.k = 40

    def enqueue(self):
        s = self.s
        s.sort_keys(self.keys)
        self.a16 = s.argsort16(self.k16, "bf16", True)
        s.sort_pairs(self.pk, self.pv)
        self.ts = s.topk_segments(self.sx, self.soff, self.k, "f32", True)
        self.ss = s.sort_segments(self.rx, self.roff, "i16", False, True, True, 16384)
        self.tr = s.topk_rows(self.tx, self.k, "f16", False)

    def fill(self, i, b16, pk):
        """new contents of every static tensor; returns the host copies the check needs"""
        rng = self.rng
        c = region_keys(NK)
        keys = (random_bits(rng, NK, "u32") if i % 2 == 0 else with_place0_bin(NK, c + 1, NK - WINDOW, 100 + i))
        lens = np.minimum(np.exp(rng.uniform(0, np.log(1 << 13), self.segs)).astype(np.int64), 16384)
        soff = offsets_of(lens)
        sx = typed_input(rng, 1 << 20, "f32")
        soff = np.minimum(soff, sx.size)  # the offsets change, their count stays
        rlens = rng.integers(0, 700, self.segs)
        rlens[rng.random(self.segs) < 0.2] = 0
        roff = offsets_of(rlens, start=int(rng.integers(0, 500)))
        rx = typed_input(rng, 1 << 20, "i16")
        tx = typed_input(rng, 64 * 20_000, "f16").reshape(64, 20_000)
        self.keys.copy_(dev(keys, "u32").view(torch.int32))
        self.k16.copy_(dev(b16, "bf16"))
        self.pk.copy_(dev(pk, "u32").view(torch.int32))
        self.pv.copy_(torch.arange(NP, dtype=torch.int32, device="cuda"))
        self.sx.copy_(dev(sx, "f32"))
        self.soff.copy_(torch.from_numpy(soff))
        self.rx.copy_(dev(rx, "i16"))
        self.roff.copy_(torch.from_numpy(roff))
        self.tx.copy_(dev(tx, "f16"))
        return keys, b16, pk, sx, soff, rx, roff, tx

    def check(self, what, host_in):
        keys, b16, pk, sx, soff, rx, roff, tx = host_in
        same(host(self.keys, "i32").view(np.uint32), np.sort(keys), f"{what}: fused sort")
        o = order_of(b16, "bf16", True)
        same(host(self.k16, "bf16"), b16, f"{what}: argsort16 input modified")
        same(host(self.a16[0], "bf16"), b16[o], f"{what}: argsort16 keys")
        same(idx_host(self.a16[1]), o, f"{what}: argsort16 indices")
        o = order_of(pk, "u32")
        same(host(self.pk, "i32").view(np.uint32), pk[o], f"{what}: pairs keys")
        same(idx_host(self.pv), o, f"{what}: pairs payloads")
        wk, wi = topk_segments_oracle(sx, soff, self.k, "f32", True)
        same(host(self.ts[0], "f32"), wk, f"{what}: topk_segments keys")
        same(idx_host(self.ts[1]), wi, f"{what}: topk_segments indices")
        wk, wi = sort_segments_oracle(rx, roff, rx.size, 16384, "i16", False, rx, np.zeros(rx.size, np.uint32))
        inside = np.zeros(rx.size, bool)
        inside[roff[0]:roff[-1]] = True  # the segments are contiguous: only the indices before and after them are unset
        same(host(self.rx, "i16"), wk, f"{what}: sort_segments keys (in place; the rest untouched)")
        same(idx_host(self.ss[1])[inside], wi[inside], f"{what}: sort_segments indices")
        o = np.argsort(radix(tx, "f16"), axis=-1, kind="stable")[:, :self.k]
        same(host(self.tr[0], "f16"), np.take_along_axis(tx, o, axis=-1), f"{what}: topk_rows keys")
        same(idx_host(self.tr[1]), o, f"{what}: topk_rows indices")


def eager_other_families(s, rng, i):
    """calls that leave the descriptors alone, between replays: rows, segments, validate, a single-block 16-bit sort"""
    steps = [
        ("sort_rows", rows(typed_input(rng, 300 * 257, "u32").reshape(300, 257), "u32", True)),
        ("topk_segments", topk_segments(typed_input(rng, 50_000, "bf16"), offsets_of(rng.integers(0, 300, 200)), "bf16", 17, False)),
        ("validate", validate(random_bits(rng, 100_000, "u32"), "u32")),
        ("sort_keys16, one block", keys16(typed_input(rng, 16_000, "f16"), "f16", True)),
        ("segmented_sort", segmented_sort(random_bits(rng, 200_000, "u32"), offsets_of(rng.integers(0, 3000, 60)), 16384)),
    ]
    for name, enqueue in steps[i % 2::2]:
        checked(f"eager {name} after replay {i}", enqueue(s))


def test_one_graph_mixing_families_on_one_44_handle(g):
    require(g, "the mixed graph", N16 + SLACK, 4, 4, 2 * GiB, 2 * GiB)
    rng = np.random.default_rng(50)
    ins16 = inputs16(rng, N16)
    insp = radix_inputs(rng, NP, np.uint32)
    with g.OneSweepSorter(N16 + SLACK, 4, 4) as s:
        gr = Graph(s, rng)
        host_in = gr.fill(0, from_radix(ins16[0][1], "bf16"), insp[0][1])
        gr.enqueue()  # eager, before the capture: kernels configured, and the reference for the first check
        torch.cuda.synchronize()
        gr.check("eager", host_in)
        e0 = s.info("epoch")
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            gr.enqueue()
        assert s.info("epoch") == e0 + 10  # fused sort e0+1..4, argsort16 e0+5..6, pairs e0+7..10

        def replay(i, r16, pk, what):
            # descending bf16: the complement of the radix image keeps the varying bytes where they were
            host_in = gr.fill(i, from_radix(~r16, "bf16"), pk)
            graph.replay()
            torch.cuda.synchronize()
            gr.check(what, host_in)

        for i in range(8):
            name16, r16, skip16 = ins16[i]
            namep, pk, skipp, _ = insp[i % len(insp)]
            replay(i, r16, pk, f"replay {i} (argsort16 {name16}, pairs {namep})")
            assert s.info("last_skip_mask") == skipp, f"replay {i}: pairs plan"
            eager_other_families(s, rng, i)

        # eager sorts on the captured epochs, between replays whose first and last executed passes meet theirs
        u16 = lambda: rng.integers(0, 1 << 16, N16, dtype=np.uint32).astype(np.uint16)  # noqa: E731
        replay(8, ins16[2][1], insp[3][1], "replay before the eager sorts (place 0 only)")
        s.set_option("debug_epoch", e0 + 4)
        checked("eager argsort16 on the captured epochs", argsort16(u16().view(np.uint16), "bf16", True)(s))
        assert s.info("epoch") == e0 + 6
        checked("eager sort_pairs on the captured epochs", pairs(random_bits(rng, NP, "u32"))(s))
        assert s.info("epoch") == e0 + 10
        s.set_option("debug_epoch", e0)
        checked("eager fused sort on the captured epochs", keys_u32(random_bits(rng, NK, "u32"))(s))
        assert s.info("last_fused_kept") == 1
        replay(9, ins16[1][1], insp[1][1], "replay after the eager sorts (last place only)")
        replay(10, ins16[0][1], insp[0][1], "replay, uniform")

        # across the wrap-around: a pass at epoch 1 leaves its words; the sort that wraps runs its next executed pass at 1.
        # (Eager sorts never clear, so only one eager sort may run on the epochs debug_epoch brings back.)
        s.set_option("debug_epoch", 0)
        bits = from_radix((u16() & np.uint16(0xFF)) | np.uint16(0x7700), "bf16")  # only place 0 runs, at epoch 1
        checked("argsort16, one pass at epoch 1", argsort16(bits, "bf16")(s))
        assert s.info("last_skip_mask") == 0b10
        s.set_option("debug_epoch", EPOCH_MAX - 1)
        bits = from_radix((u16() & np.uint16(0xFF00)) | np.uint16(0x66), "bf16")  # place 0 skipped at 2^24 - 1, place 1 at 1
        checked("argsort16 across the wrap-around", argsort16(bits, "bf16")(s))
        assert s.info("epoch") == 1 and s.info("last_skip_mask") == 0b01
        # its pass at epoch 1 left its words in all 257 tiles; the next sort to wrap runs its third place on them
        s.set_option("debug_epoch", EPOCH_MAX - 2)
        r = random_bits(rng, N16, "u32") & ~np.uint32(0xFFFF) | np.uint32(0x1234)  # places 0, 1 skipped, place 2 at 1
        checked("argsort i32 across the wrap-around", argsort(from_radix(r, "i32"), "i32")(s))
        assert s.info("epoch") == 2 and s.info("last_skip_mask") == 0b0011
        # the sorts that wrap after it skip the places they run before the wrap, which no other sort may reuse
        s.set_option("debug_epoch", EPOCH_MAX - 2)
        r = random_bits(rng, NP, "u32") & ~np.uint32(0xFFFF) | np.uint32(0x4321)
        checked("sort_pairs across the wrap-around", pairs(r)(s))
        assert s.info("epoch") == 2 and s.info("last_skip_mask") == 0b0011
        s.set_option("debug_epoch", EPOCH_MAX - 2)
        checked("fused sort across the wrap-around", keys_u32(random_bits(rng, NK, "u32"))(s))
        assert s.info("epoch") == 2 and s.info("last_fused_kept") == 1
        replay(11, ins16[3][1], insp[4][1], "replay after the wrap-around")
        del graph
    release()


# ---- 4. concurrency ----------------------------------------------------------------------------------------------------------
def test_families_concurrently_beside_matmuls(g):
    """one handle and one stream per family, three rounds enqueued before any check, while bf16 matmuls hold SMs"""
    require(g, "the concurrent families", 1 << 24, 4, 4, 8 * GiB, 10 * GiB)

    def rand(n, dtype, seed):
        """random bit patterns, 30 % of them drawn from 64 values (ties)"""
        gen = torch.Generator(device="cuda").manual_seed(seed)
        sd = SIGNED[torch.empty(0, dtype=dtype).element_size()]
        b = torch.randint(torch.iinfo(sd).min, torch.iinfo(sd).max, (n,), device="cuda", generator=gen, dtype=sd)
        pick = torch.rand(n, device="cuda", generator=gen) < 0.3
        b[pick] = b[:64].clone()[torch.randint(0, 64, (int(pick.sum()),), device="cuda", generator=gen)]
        return b.view(dtype)

    def uniform32(seed):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        return torch.randint(-(1 << 31), (1 << 31) - 1, (1 << 24,), device="cuda", generator=gen, dtype=torch.int32)

    def check_argsort(what, x, x0, out, idx, t, desc):
        o, b = device_order(x0, t, desc)
        assert torch.equal(x.view(b.dtype), b), f"{what}: input modified"
        assert torch.equal(out.view(b.dtype), b[o]), f"{what}: keys"
        assert torch.equal(idx.long(), o), f"{what}: indices"

    def check_pairs(what, x, x0, v, t, desc):
        o, b = device_order(x0, t, desc)
        assert torch.equal(x.view(b.dtype), b[o]), f"{what}: keys"
        assert torch.equal(v.long(), o), f"{what}: payloads"

    rounds = []
    c24 = region_keys(1 << 24)
    rng = np.random.default_rng(60)
    seg_lens = ragged(rng, "log-uniform", 1 << 22)
    seg_off = torch.from_numpy(offsets_of(seg_lens)).cuda()
    seg_n = int(seg_lens.sum())
    late = torch.from_numpy(with_place0_bin(1 << 24, c24 + 1, (1 << 24) - WINDOW, 61).view(np.int32)).cuda()
    s16 = g.OneSweepSorter(1 << 24, 4, 4)
    s64 = g.OneSweepSorter(1 << 23, 8, 4)
    s32 = g.OneSweepSorter(1 << 24, 4, 4)
    sfu = g.OneSweepSorter(1 << 24, 4, 0)
    stk = g.OneSweepSorter(1, 4, 4)
    sse = g.OneSweepSorter(seg_lens.size + 1, 4, 4)
    sorters = [s16, s64, s32, sfu, stk, sse]
    streams = [torch.cuda.Stream() for _ in sorters]
    try:
        for r in range(3):
            seed = 1000 * r
            case = {
                "a16": rand(1 << 24, torch.bfloat16, seed + 1), "p16k": rand(1 << 24, torch.int16, seed + 2),
                "f64k": rand(1 << 23, torch.float64, seed + 3), "i64": rand(1 << 23, torch.int64, seed + 4),
                "f32": rand(1 << 24, torch.float32, seed + 5),
                # one fused sort that stands and one whose last tiles overflow a region (the fallback), in either order
                "first": uniform32(seed + 6) if r != 1 else late.clone(),
                "second": late.clone() if r != 1 else uniform32(seed + 6),
                "tk": rand(256 * 151_936, torch.float32, seed + 7).view(256, 151_936),
                "seg": rand(seg_n, torch.float32, seed + 8),
            }
            case["p16v"] = torch.arange(1 << 24, dtype=torch.int32, device="cuda")
            case["f64v"] = torch.arange(1 << 23, dtype=torch.int32, device="cuda")
            case["orig"] = {k: v.clone() for k, v in case.items() if isinstance(v, torch.Tensor)}
            rounds.append(case)
        a = torch.randn(4096, 4096, dtype=torch.bfloat16, device="cuda")
        b = torch.randn(4096, 4096, dtype=torch.bfloat16, device="cuda")
        ms = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(ms):
            for _ in range(100):
                torch.mm(a, b)
        for case in rounds:
            with torch.cuda.stream(streams[0]):
                case["a16_out"] = s16.argsort16(case["a16"], "bf16")
                s16.sort_pairs16(case["p16k"], case["p16v"], "i16", True)
            with torch.cuda.stream(streams[1]):
                s64.sort_pairs_typed(case["f64k"], case["f64v"], "f64", True)
                case["i64_out"] = s64.argsort(case["i64"], "i64")
            with torch.cuda.stream(streams[2]):
                case["f32_out"] = s32.argsort(case["f32"], "f32")
            with torch.cuda.stream(streams[3]):
                sfu.sort_keys(case["first"])
                sfu.sort_keys(case["second"])
            with torch.cuda.stream(streams[4]):
                case["tk_out"] = stk.topk_rows(case["tk"], 64, "f32", True)
            with torch.cuda.stream(streams[5]):
                case["ts_out"] = sse.topk_segments(case["seg"], seg_off, 32, "f32", True)
                case["ss_out"] = sse.sort_segments(case["seg"], seg_off, "f32", True, max_segment_len=16384)
        torch.cuda.synchronize()
        for r, case in enumerate(rounds):
            o = case["orig"]
            check_argsort(f"round {r}: argsort16 bf16", case["a16"], o["a16"], *case["a16_out"], "bf16", False)
            check_pairs(f"round {r}: sort_pairs16 i16 descending", case["p16k"], o["p16k"], case["p16v"], "i16", True)
            check_pairs(f"round {r}: sort_pairs_typed f64 descending", case["f64k"], o["f64k"], case["f64v"], "f64", True)
            check_argsort(f"round {r}: argsort i64", case["i64"], o["i64"], *case["i64_out"], "i64", False)
            check_argsort(f"round {r}: argsort f32", case["f32"], o["f32"], *case["f32_out"], "f32", False)
            for name in ("first", "second"):
                want = torch.sort(o[name] ^ torch.iinfo(torch.int32).min, stable=True)[0] ^ torch.iinfo(torch.int32).min
                assert torch.equal(case[name], want), f"round {r}: the {name} fused sort"
            vals, idx = case["tk_out"]
            ordr, bb = device_order(o["tk"], "f32", True)
            ordr = ordr[:, :64]
            assert torch.equal(vals.view(torch.int32), torch.gather(bb, 1, ordr)), f"round {r}: topk_rows keys"
            assert torch.equal(idx.long(), ordr), f"round {r}: topk_rows indices"
            seg_bits = o["seg"].view(torch.int32).cpu().numpy().view(np.uint32)
            off = seg_off.cpu().numpy()
            wk, wi = topk_segments_oracle(seg_bits, off, 32, "f32", True)
            same(host(case["ts_out"][0], "f32"), wk, f"round {r}: topk_segments keys")
            same(idx_host(case["ts_out"][1]), wi, f"round {r}: topk_segments indices")
            wk, wi = sort_segments_oracle(seg_bits, off, seg_bits.size, 16384, "f32", True, seg_bits, np.zeros(seg_bits.size, np.uint32))
            inside = np.repeat(np.diff(off) <= 16384, np.diff(off))
            same(host(case["ss_out"][0], "f32")[inside], wk[inside], f"round {r}: sort_segments keys")
            same(idx_host(case["ss_out"][1])[inside], wi[inside], f"round {r}: sort_segments indices")
    finally:
        for s in sorters:
            s.close()
    release()


# ---- 5. the module calls -------------------------------------------------------------------------------------------------------
def module_calls(g, rng, stream, n):
    """the six functions that share the stream's cached (4, 4) sorter, interleaved on `stream`; returns their check"""
    f32 = typed_input(rng, n, "f32")
    b16 = typed_input(rng, n, "bf16")
    r32 = typed_input(rng, 500 * 300, "i32").reshape(500, 300)
    t16 = typed_input(rng, 40 * 5000, "f16").reshape(40, 5000)
    off = offsets_of(ragged(rng, "empty runs", 200_000))  # contiguous from 0: every output position is written
    sx = typed_input(rng, int(off[-1]), "u16")
    tx = typed_input(rng, int(off[-1]), "f32")
    offs, xa, x16, xr, xt, xs, xtk = (torch.from_numpy(off).cuda(), dev(f32, "f32"), dev(b16, "bf16"), dev(r32, "i32"),
                                      dev(t16, "f16"), dev(sx, "u16"), dev(tx, "f32"))
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        res = [
            g.topk_segments(xtk, offs, 9),
            g.argsort(xa, "f32"),
            g.sort_rows(xr, descending=True),
            g.argsort16(x16, "bf16", True),
            g.sort_segments(xs, offs, max_segment_len=16384),
            g.topk(xt, 25, largest=False),
        ]

    def check(what):
        wk, wi = topk_segments_oracle(tx, off, 9, "f32", True)
        same(host(res[0][0], "f32"), wk, f"{what}: topk_segments keys")
        same(idx_host(res[0][1]), wi, f"{what}: topk_segments indices")
        o = order_of(f32, "f32")
        same(host(xa, "f32"), f32, f"{what}: argsort input modified")
        same(host(res[1][0], "f32"), f32[o], f"{what}: argsort keys")
        same(idx_host(res[1][1]), o, f"{what}: argsort indices")
        o = np.argsort(radix(r32, "i32", True), axis=-1, kind="stable")
        same(host(res[2][0], "i32"), np.take_along_axis(r32, o, axis=-1), f"{what}: sort_rows keys")
        same(idx_host(res[2][1]), o, f"{what}: sort_rows indices")
        o = order_of(b16, "bf16", True)
        same(host(x16, "bf16"), b16, f"{what}: argsort16 input modified")
        same(host(res[3][0], "bf16"), b16[o], f"{what}: argsort16 keys")
        same(idx_host(res[3][1]), o, f"{what}: argsort16 indices")
        wk, wi = sort_segments_oracle(sx, off, sx.size, 16384, "u16", False, sx, np.zeros(sx.size, np.uint32))
        same(host(res[4][0], "u16"), wk, f"{what}: sort_segments keys")
        same(idx_host(res[4][1]), wi, f"{what}: sort_segments indices")
        o = np.argsort(radix(t16, "f16"), axis=-1, kind="stable")[:, :25]
        same(host(res[5][0], "f16"), np.take_along_axis(t16, o, axis=-1), f"{what}: topk keys")
        same(idx_host(res[5][1]), o, f"{what}: topk indices")
    return check


def test_module_calls_share_one_handle_per_stream(g):
    """the six calls interleaved on one stream, then on two: each stream gets one cached (4, 4) sorter and no other"""
    from gpusorting_b200 import onesweep

    rng = np.random.default_rng(70)
    d = torch.cuda.current_device()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    assert s1.cuda_stream != s2.cuda_stream
    before = set(onesweep._CACHE)

    def new_entries(st):
        return {k for k in onesweep._CACHE if k[3] == st.cuda_stream} - before

    torch.cuda.synchronize()
    check = module_calls(g, rng, s1, NS)
    torch.cuda.synchronize()
    check("one stream")
    assert new_entries(s1) <= {(d, 4, 4, s1.cuda_stream)} and (d, 4, 4, s1.cuda_stream) in onesweep._CACHE
    h1 = onesweep._CACHE[(d, 4, 4, s1.cuda_stream)]
    assert h1.max_n >= NS
    checks = [(module_calls(g, rng, st, NS // 2), f"stream {i + 1} of 2") for i, st in enumerate((s1, s2))]
    torch.cuda.synchronize()
    for check, what in checks:
        check(what)
    for st in (s1, s2):
        assert new_entries(st) <= {(d, 4, 4, st.cuda_stream)} and (d, 4, 4, st.cuda_stream) in onesweep._CACHE
    assert onesweep._CACHE[(d, 4, 4, s1.cuda_stream)] is h1  # large enough already: the same handle
    assert onesweep._CACHE[(d, 4, 4, s2.cuda_stream)] is not h1


def test_cache_grows_under_a_live_graph(g):
    """argsort and topk_segments captured on stream S; then eager calls on S grow the cached sorter twice.  The captured
    handle must still be open, kept by the module, before the graph is replayed."""
    from gpusorting_b200 import onesweep

    rng = np.random.default_rng(80)
    d = torch.cuda.current_device()
    S = torch.cuda.Stream()
    key = (d, 4, 4, S.cuda_stream)
    base = onesweep._CACHE[key].max_n if key in onesweep._CACHE else 0
    na = max(base, 1 << 20) + 1
    require(g, "the growing cache", 4 * na, 4, 4, 64 * na, 2 * GiB)
    xa = torch.zeros(na, dtype=torch.float32, device="cuda")
    lens = rng.integers(0, 600, 2000)
    y = torch.zeros(int(lens.sum()) + 100, dtype=torch.float32, device="cuda")
    off = torch.zeros(lens.size + 1, dtype=torch.int64, device="cuda")

    def fill():
        a = typed_input(rng, na, "f32")
        o = offsets_of(rng.permutation(lens))
        b = typed_input(rng, y.numel(), "f32")
        xa.copy_(dev(a, "f32"))
        off.copy_(torch.from_numpy(o))
        y.copy_(dev(b, "f32"))
        return a, o, b

    def check(what, a, o, b, res):
        (ak, ai), (tk, ti) = res
        w = order_of(a, "f32", True)
        same(host(ak, "f32"), a[w], f"{what}: argsort keys")
        same(idx_host(ai), w, f"{what}: argsort indices")
        wk, wi = topk_segments_oracle(b, o, 7, "f32", False)
        same(host(tk, "f32"), wk, f"{what}: topk_segments keys")
        same(idx_host(ti), wi, f"{what}: topk_segments indices")

    torch.cuda.synchronize()
    with torch.cuda.stream(S):
        a, o, b = fill()
        res = (g.argsort(xa, "f32", True), g.topk_segments(y, off, 7, largest=False))  # warm-up outside the capture
    S.synchronize()
    check("eager", a, o, b, res)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=S):
        res = (g.argsort(xa, "f32", True), g.topk_segments(y, off, 7, largest=False))
    h0 = onesweep._CACHE[key]
    # eager calls on S that need more than the captured handle holds: more segments, then more keys
    segs = h0.max_n + 1
    gl = rng.integers(0, 3, segs)
    go = offsets_of(gl)
    gb = typed_input(rng, int(go[-1]), "f32")
    with torch.cuda.stream(S):
        gk, gi = g.topk_segments(dev(gb, "f32"), torch.from_numpy(go).cuda(), 2)
    h1 = onesweep._CACHE[key]
    assert h1 is not h0 and h1.max_n >= segs
    ga = typed_input(rng, h1.max_n + 1, "f32")
    with torch.cuda.stream(S):
        ak, ai = g.argsort(dev(ga, "f32"), "f32")
    h2 = onesweep._CACHE[key]
    assert h2 is not h1 and h2.max_n >= ga.size
    S.synchronize()
    wk, wi = topk_segments_oracle(gb, go, 2, "f32", True)
    same(host(gk, "f32"), wk, "growing topk_segments keys")
    same(idx_host(gi), wi, "growing topk_segments indices")
    w = order_of(ga, "f32")
    same(host(ak, "f32"), ga[w], "growing argsort keys")
    same(idx_host(ai), w, "growing argsort indices")

    # before any replay: the captured handle is open and the module still holds it
    assert h0._h is not None and h1._h is not None, "the cache closed a sorter that a captured graph uses"
    assert any(r is h0 for r in onesweep._RETIRED) and any(r is h1 for r in onesweep._RETIRED)
    for i in range(3):
        with torch.cuda.stream(S):
            a, o, b = fill()
            graph.replay()
        torch.cuda.synchronize()
        check(f"replay {i}", a, o, b, res)

    del graph, res
    g.release_cached_sorters()
    assert h0._h is None and h1._h is None and not onesweep._RETIRED
    assert onesweep._CACHE[key] is h2 and h2._h is not None  # the sorter in use stays
    release()
