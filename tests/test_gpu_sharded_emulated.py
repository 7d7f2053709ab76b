"""The sharded sort's exchange on ONE GPU: one process plays all R ranks.  -m gpu

The fused exchange is the ordinary DigitBinningPass with no output pointer and per-bin bases that are virtual element
indices (byte address / 4) into the receive buffers; the staged exchange is the same pass into a send buffer followed by
ncclSend/ncclRecv.  Neither needs a second GPU to be checked: here R receive buffers live on the one device, every
virtual rank runs osb200_debug_digit_histogram and osb200_debug_exchange_pass with the layout the sort itself computes
(osb200_sharded_exchange_layout), and every slot of every receive buffer is compared with the stable MSD partition built
in numpy.  What this does not cover -- NCCL, CUDA IPC mapping, peer stores over NVLink and the cross-GPU barriers --
stays with tests/test_gpu_sharded.py on two or more GPUs."""
import numpy as np
import pytest
import torch

import gpusorting_b200 as g
from gpusorting_b200 import sharded
from gpusorting_b200._lib import check, lib

pytestmark = pytest.mark.gpu

SENTINEL = np.uint32(0xA5C3E1F7)
GUARD = 1000  # sentinel words around every buffer the passes write


def _stream():
    return int(torch.cuda.current_stream().cuda_stream)


def _dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32 if a.dtype == np.uint32 else np.int64).copy()).cuda()


def _host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy().view(np.uint32)


def _ptr(t: torch.Tensor, n: int):
    return t.data_ptr() if n else None


def debug_histogram(s: g.OneSweepSorter, keys: torch.Tensor, n: int) -> np.ndarray:
    out = torch.empty(256, dtype=torch.int64, device="cuda")
    check(lib.osb200_debug_digit_histogram(s._h, _ptr(keys, n), n, 24, out.data_ptr(), _stream()),
          "osb200_debug_digit_histogram")
    return out.cpu().numpy().astype(np.uint64)


def debug_pass(s: g.OneSweepSorter, keys: torch.Tensor, n: int, shift: int, hist=None, out=None, out_base=None):
    check(lib.osb200_debug_exchange_pass(s._h, _ptr(keys, n), None if out is None else out.data_ptr(), n, shift,
                                         None if hist is None else hist.data_ptr(),
                                         None if out_base is None else out_base.data_ptr(), _stream()),
          "osb200_debug_exchange_pass")


def arena(n: int, offset: int) -> tuple:
    """A buffer of n words at `offset` words into a larger allocation that is filled with sentinels."""
    a = torch.from_numpy(np.full(n + offset + GUARD, SENTINEL).view(np.int32)).cuda()
    return a, a[offset:offset + n]


def check_arena(a: torch.Tensor, offset: int, want: np.ndarray, what: str) -> None:
    got = _host(a)
    body = got[offset:offset + want.size]
    assert body.size == want.size and np.array_equal(body, want), \
        f"{what}: {int(np.count_nonzero(body != want))} of {want.size} words differ"
    outside = np.concatenate([got[:offset], got[offset + want.size:]])
    assert (outside == SENTINEL).all(), f"{what}: {int(np.count_nonzero(outside != SENTINEL))} words written outside"


def tile_keys() -> int:
    with g.OneSweepSorter(1 << 16) as s:
        return s.info("tile_keys")


def default_sizes(world: int, T: int) -> list:
    """Unequal per-rank sizes: empty, one key, less than a tile, one tile, ragged multi-tile."""
    pattern = [0, 1, T - 3, T, 3 * T + 17, 2 * T + 1, 5 * T + 4097, T // 2 + 1, 7 * T + 333]
    if world == 1:
        return [3 * T + 17]
    return [pattern[(5 * r + 1) % len(pattern)] for r in range(world)]


def make_keys(oracle, dist: str, n: int, rank: int, seed: int) -> np.ndarray:
    s = 1000 * seed + 10 + rank
    if dist.startswith("entropy"):  # reference presets 3..5: AND of 3..5 words
        return oracle.init_random_u32(n, int(dist[-1]) - 1, s)
    k = oracle.init_random_u32(n, 0, s)
    if dist == "skewed" and rank == 0:
        k &= np.uint32(0x3FFFFFFF)  # rank 0 holds only small keys
    elif dist == "quarter":
        k &= np.uint32(0x3FFFFFFF)  # every key below 2^30, over that quarter's 64 top bytes
    elif dist == "one_byte":
        k = (k & np.uint32(0x00FFFFFF)) | np.uint32(0x42000000)
    elif dist == "equal":
        k[:] = np.uint32(0x9E3779B9)
    return k


def stable_parts(keys: np.ndarray, shift: int) -> list:
    """keys split by the digit keys >> shift, each part in input order: the stable bin-major partition, as 256 parts."""
    digit = (keys >> np.uint32(shift)).astype(np.uint16)
    order = np.argsort(digit, kind="stable")
    bounds = np.concatenate([[0], np.cumsum(np.bincount(digit, minlength=256))])
    part = keys[order]
    return [part[bounds[b]:bounds[b + 1]] for b in range(256)]


def run_exchange(oracle, world, dist="uniform", mode="fused", force_fine=False, slack=50, sizes=None, options=(),
                 expect=None, seed=1):
    """R virtual ranks run the exchange; every received word, every guard word and the final sort are checked.
    Returns the layout of rank 0 (or "size")."""
    T = tile_keys()
    sizes = default_sizes(world, T) if sizes is None else sizes
    keys = [make_keys(oracle, dist, n, r, seed) for r, n in enumerate(sizes)]
    max_n = max(max(sizes), 1)
    cap = sharded.capacity(max_n, slack)
    ex = g.OneSweepSorter(max_n)
    try:
        for k, v in options:
            if k == "rank_mode" and v == 0 and ex.info("atomic_order_ok") == 0:
                pytest.skip("atomic ranking is not available on this device")
            ex.set_option(k, v)
        d_keys = [_dev(k) for k in keys]

        # 1. the sort's first step: the top-byte histogram of every rank
        hist_all = np.stack([debug_histogram(ex, d, n) for d, n in zip(d_keys, sizes)])
        for r, k in enumerate(keys):
            assert np.array_equal(hist_all[r], np.bincount(k >> np.uint32(24), minlength=256)), f"histogram of rank {r}"

        # 2. every rank's layout; fused bases point into receive buffers that start at arbitrary word offsets
        recv = offs = addrs = None
        if mode == "fused":
            offs = [37 + 5 * q for q in range(world)]
            recv = [arena(cap, o) for o in offs]
            addrs = [buf.data_ptr() for _, buf in recv]
        lays = []
        for r in range(world):
            try:
                lays.append(sharded.exchange_layout(hist_all, r, cap, force_fine, addrs))
            except g.OneSweepError as e:
                lays.append(e.status)
        if expect == "size":
            assert lays == [-2] * world, "every rank returns OSB200_ERR_SIZE together and nothing is launched"
            return "size"
        assert all(isinstance(x, dict) for x in lays), lays
        lay0 = lays[0]
        xshift, bins, dest, recv_count = lay0["xshift"], lay0["bins"], lay0["dest"], lay0["recv_count"]
        if expect == "coarse":
            assert bins == world and xshift == 32 - (world - 1).bit_length()
        elif expect == "fine":
            assert bins == 256 and xshift == 24

        # 3. before any launch: each pass scans the counts of its own digit, and every bin's range lies inside its
        #    destination buffer -- a layout error fails here and never becomes a store outside the buffers
        for r, lay in enumerate(lays):
            digit_hist = np.bincount(keys[r] >> np.uint32(xshift), minlength=256)
            assert np.array_equal(lay["pass_hist"], digit_hist), f"pass histogram of rank {r}"
            assert np.array_equal(lay["dest"], dest) and np.array_equal(lay["recv_count"], recv_count)
        assert (recv_count <= cap).all() and int(recv_count.sum()) == sum(sizes)
        if mode == "fused":
            unaligned = False
            for r, lay in enumerate(lays):
                for b in np.flatnonzero(lay["pass_hist"]):
                    q, c = int(dest[b]), int(lay["pass_hist"][b])
                    lo = int(lay["out_base"][b]) - addrs[q] // 4
                    assert 0 <= lo and lo + c <= int(recv_count[q]), f"bin {b} of rank {r} leaves buffer {q}"
                    unaligned |= int(lay["out_base"][b]) % 32 != 0
            if bins <= 32 and sum(n > 0 for n in sizes) >= 2:
                assert unaligned, "some few-bins run must start inside a 128-byte line"

        parts = [stable_parts(k, xshift) for k in keys]
        owned = [[b for b in range(bins) if dest[b] == q] for q in range(world)]
        # 4. the exchange
        if mode == "fused":
            for r in range(world):
                debug_pass(ex, d_keys[r], sizes[r], xshift, hist=_dev(lays[r]["pass_hist"]),
                           out_base=_dev(lays[r]["out_base"]))
            torch.cuda.synchronize()
            received = []
            for q in range(world):
                # bucket-major, source-minor, input order within a (bucket, source): the stable MSD partition
                want = np.concatenate([parts[r][b] for b in owned[q] for r in range(world)] + [np.empty(0, np.uint32)])
                a, buf = recv[q]
                check_arena(a, offs[q], want, f"receive buffer {q}")
                received.append(want)
        else:
            send = []
            for r in range(world):
                a, buf = arena(sizes[r], 3 + r)
                debug_pass(ex, d_keys[r], sizes[r], xshift, hist=_dev(lays[r]["pass_hist"]), out=buf)
                send.append((a, 3 + r))
            torch.cuda.synchronize()
            sent = []
            for r in range(world):
                want = np.concatenate(parts[r][:bins] + [np.empty(0, np.uint32)])  # stable bin-major partition
                check_arena(send[r][0], send[r][1], want, f"send buffer {r}")
                sent.append(want)
            received = []
            for q in range(world):  # ncclSend / ncclRecv with the staged offsets
                rf = lays[q]["recv_from_off"].astype(np.int64)
                got = np.full(int(recv_count[q]), SENTINEL)
                for src in range(world):
                    so = lays[src]["send_off"].astype(np.int64)
                    piece = sent[src][so[q]:so[q + 1]]
                    assert piece.size == rf[src + 1] - rf[src], f"{src} -> {q}: sent {piece.size}, expected"
                    got[rf[src]:rf[src + 1]] = piece
                # source-major: every source's bins of q in bin order
                want = np.concatenate([parts[src][b] for src in range(world) for b in owned[q]] + [np.empty(0, np.uint32)])
                assert np.array_equal(got, want), f"received by {q}: {int(np.count_nonzero(got != want))} words differ"
                received.append(got)
        for r in range(world):
            assert np.array_equal(_host(d_keys[r]), keys[r]), f"input of rank {r} was modified"

        # 5. the local sorts: concatenated, the global ascending order
        with g.OneSweepSorter(cap) as loc:
            out = []
            for q in range(world):
                t = _dev(received[q])
                loc.sort_keys(t)
                out.append(_host(t))
        assert np.array_equal(np.concatenate(out), np.sort(np.concatenate(keys)))
        return lay0
    finally:
        ex.close()


COARSE = [2, 4, 8, 32, 64]  # digit widths 1, 2, 3, 5 (few-bins scatter) and 6 (plain scatter)


@pytest.mark.parametrize("mode", ["fused", "staged"])
@pytest.mark.parametrize("force_fine", [False, True])
@pytest.mark.parametrize("world", COARSE)
def test_power_of_two_worlds(oracle, world, force_fine, mode):
    run_exchange(oracle, world, mode=mode, force_fine=force_fine, expect="fine" if force_fine else "coarse")


@pytest.mark.parametrize("mode", ["fused", "staged"])
@pytest.mark.parametrize("world", [1, 3, 5, 7])
def test_other_worlds_take_the_fine_plan(oracle, world, mode):
    run_exchange(oracle, world, mode=mode, expect="fine")


@pytest.mark.parametrize("mode", ["fused", "staged"])
@pytest.mark.parametrize("world,force_fine", [(4, False), (4, True), (3, False), (8, False)])
def test_skewed_rank0_holds_small_keys(oracle, world, force_fine, mode):
    run_exchange(oracle, world, "skewed", mode=mode, force_fine=force_fine)


@pytest.mark.parametrize("mode", ["fused", "staged"])
def test_one_full_coarse_bin_falls_back_to_fine(oracle, mode):
    """Every key below 2^30 but spread over its 64 top bytes: the equal-width split would hand rank 0 all of them, beyond
    50 % slack, so the layout takes the 256-bucket plan."""
    T = tile_keys()
    lay = run_exchange(oracle, 4, "quarter", mode=mode, sizes=[3 * T + 17, 2 * T + 1, 5 * T + 4097, 4 * T], expect="fine")
    assert lay["recv_count"].min() > 0


@pytest.mark.parametrize("world", [3, 4])
def test_one_top_byte_is_size_for_every_rank(oracle, world):
    T = tile_keys()
    sizes = [3 * T + 17, 2 * T + 1, 5 * T + 4097, 4 * T][:world]
    assert run_exchange(oracle, world, "one_byte", sizes=sizes, expect="size") == "size"


@pytest.mark.parametrize("mode", ["fused", "staged"])
@pytest.mark.parametrize("preset", [3, 4, 5])
def test_entropy_presets(oracle, preset, mode):
    T = tile_keys()
    run_exchange(oracle, 2, f"entropy{preset}", mode=mode, slack=100, sizes=[3 * T + 17, 5 * T + 4097])


@pytest.mark.parametrize("mode", ["fused", "staged"])
@pytest.mark.parametrize("force_fine", [False, True])
def test_all_keys_equal_go_to_one_rank(oracle, force_fine, mode):
    T = tile_keys()
    lay = run_exchange(oracle, 2, "equal", mode=mode, force_fine=force_fine, slack=100, sizes=[3 * T + 17, 5 * T + 4097],
                       expect="fine" if force_fine else "coarse")
    assert sorted(int(c) for c in lay["recv_count"]) == [0, 8 * T + 4114]


SCHEDULES = {
    "default": (),
    "max_ctas1": (("debug_max_ctas", 1),),
    "max_ctas3": (("debug_max_ctas", 3),),
    "stall2": (("debug_stall_every", 2), ("spin_cap", 16)),
}


@pytest.mark.parametrize("mode", ["fused", "staged"])
@pytest.mark.parametrize("world,force_fine", [(4, False), (64, False), (3, False)])
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("rank_mode", [0, 1])
def test_schedules(oracle, rank_mode, schedule, world, force_fine, mode):
    """Both ranking modes; few persistent CTAs (tiles handed out by the ticket); and stalled tiles, whose successors
    re-reduce them while the pass scatters to virtual bases."""
    T = tile_keys()
    sizes = [(3 + r % 5) * T + 17 * r + 1 for r in range(world)]
    run_exchange(oracle, world, mode=mode, force_fine=force_fine, sizes=sizes, seed=7,
                 options=(("rank_mode", rank_mode),) + SCHEDULES[schedule])


def test_large_fused_coarse(oracle):
    """R = 8 with 2^25 keys per rank (2^28 in all): tiles far outnumber resident CTAs."""
    run_exchange(oracle, 8, mode="fused", sizes=[1 << 25] * 8, expect="coarse", seed=3)


def test_debug_hooks_validate_their_arguments():
    n = 1 << 12
    with g.OneSweepSorter(n) as s, g.OneSweepSorter(n, 8) as s64:
        keys = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
        out = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
        hist = torch.zeros(256, dtype=torch.int64, device="cuda")
        base = torch.zeros(256, dtype=torch.int64, device="cuda")
        k, o, h, b, q = keys.data_ptr(), out.data_ptr(), hist.data_ptr(), base.data_ptr(), _stream()
        H, P = lib.osb200_debug_digit_histogram, lib.osb200_debug_exchange_pass
        assert H(None, k, n, 24, h, q) == -1
        assert H(s64._h, k, n, 24, h, q) == -1  # 64-bit keys
        assert H(s._h, k + 4, n, 24, h, q) == -1  # not 16-byte aligned
        assert H(s._h, k, n, 32, h, q) == -1
        assert H(s._h, k, n + 1, 24, h, q) == -2
        assert H(s._h, k, n, 24, h, q) == 0
        assert P(s._h, k, o, n, 24, h, None, q) == 0
        assert P(s._h, k, o, n, 24, h, b, q) == -1  # fused bases come without an output pointer
        assert P(s._h, k, None, n, 24, h, None, q) == -1
        assert P(s._h, k, o, n, 24, None, None, q) == -1  # staged: the pass needs its histogram
        assert P(s._h, k + 4, o, n, 24, h, None, q) == -1
        assert P(s._h, k, o, n, 32, h, None, q) == -1
        assert P(s._h, k, o, n + 1, 24, h, None, q) == -2
        assert P(s64._h, k, o, n, 24, h, None, q) == -1
        torch.cuda.synchronize()
