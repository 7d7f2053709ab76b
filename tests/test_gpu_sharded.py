"""Sharded sort (NCCL, one process per GPU): fused NVLink scatter and staged NCCL exchange both produce the globally
sorted, complete result.  The exchange tests need >= 2 GPUs and skip on a single-GPU box; the single-rank test runs the
host side of the sharded sort on one GPU.  -m gpu"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, n, fused, fine, q):
    import sys

    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import gpusorting_b200 as g
        from gpusorting_b200 import sharded
        from tests import oraclelib

        orc = oraclelib.load_oracle()
        s = sharded.ShardedSorter(n, slack_percent=50)
        s.set_fused(fused)
        s.force_fine(fine)
        ok = True
        for trial, nl in enumerate([n, n - 12345, 1000 + rank, n]):
            keys = orc.init_random_u32(nl, 0, 10 + rank + 100 * trial)
            if trial == 3 and rank == 0:
                keys &= np.uint32(0x3FFFFFFF)  # skewed: rank 0 only holds small keys
            t = torch.from_numpy(keys.view(np.int32).copy()).cuda()
            res = s.sort_keys(t)
            torch.cuda.synchronize()
            mine = res.cpu().numpy().view(np.uint32).copy()
            allk = [None] * world
            dist.all_gather_object(allk, keys)
            sizes = [None] * world
            dist.all_gather_object(sizes, int(mine.size))
            want = np.sort(np.concatenate(allk))
            lo = int(sum(sizes[:rank]))
            ok = ok and sum(sizes) == want.size and np.array_equal(mine, want[lo:lo + mine.size])
            ok = ok and bool(np.array_equal(t.cpu().numpy().view(np.uint32), keys))  # input untouched
        tm = s.last_timing()
        ok = ok and tm["total_ms"] > 0
        s.close()
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("fine", [False, True])
@pytest.mark.parametrize("fused", [True, False])
def test_sharded_sort_matches_global_sort(fused, fine):
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + (os.getpid() % 1000) + (1 if fused else 0) + (2 if fine else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, 1 << 20, fused, fine, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    res = sorted(q.get(timeout=5) for _ in range(world))
    assert all(ok for _, ok in res)


def test_sharded_single_rank():
    """World size 1: create and destroy, the MSD histogram and its all-gather, the copy to the host and the busy-polled
    wait for it, the plan and the local sort, with every result compared element by element to np.sort."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29800 + (os.getpid() % 1000)
    p = ctx.Process(target=_worker, args=(0, 1, port, (1 << 20) + 12345, True, False, q))
    p.start()
    p.join(300)
    assert p.exitcode == 0
    assert q.get(timeout=5) == (0, True)


def _overflow_worker(rank, world, port, n, q):
    import sys

    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import gpusorting_b200 as g
        from gpusorting_b200 import sharded
        from tests import oraclelib

        orc = oraclelib.load_oracle()
        s = sharded.ShardedSorter(n, slack_percent=10)
        # every rank holds only keys of ONE top byte: the whole input lands on a single rank, far beyond the 10 % slack
        keys = (orc.init_random_u32(n, 0, 3 + rank) & np.uint32(0x00FFFFFF)) | np.uint32(0x42000000)
        t = torch.from_numpy(keys.view(np.int32).copy()).cuda()
        status = None
        try:
            s.sort_keys(t)
        except g.OneSweepError as e:
            status = e.status
        torch.cuda.synchronize()
        # the sorter is still usable afterwards: nobody is stuck in a collective
        keys2 = orc.init_random_u32(n, 0, 50 + rank)
        res = s.sort_keys(torch.from_numpy(keys2.view(np.int32).copy()).cuda())
        torch.cuda.synchronize()
        ok = status == -2 and res.numel() > 0 and bool((res[1:].to(torch.int64) & 0xFFFFFFFF >= res[:-1].to(torch.int64) & 0xFFFFFFFF).all())
        s.close()
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_slack_overflow_is_reported_by_every_rank_together():
    """ADVICE r1: the capacity check must make ALL ranks return OSB200_ERR_SIZE (status -2) before any collective of
    the exchange, not only the overloaded rank (which would leave the others spinning in a barrier)."""
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 1000)
    procs = [ctx.Process(target=_overflow_worker, args=(r, world, port, 1 << 18, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    res = sorted(q.get(timeout=5) for _ in range(world))
    assert all(ok for _, ok in res)
