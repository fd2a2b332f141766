"""Host-side pieces of tile sharding: the unit plan and per-rank tile counts, and the variable-count all-gather under
gloo (world 3, one rank empty)."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from resshift_b200.parallel import gather_counts
from resshift_b200.sampler import ResShiftSampler, plan_tiles


def _host_sampler(chop_size, chop_stride, chop_bs):
    s = ResShiftSampler.__new__(ResShiftSampler)          # the planning methods need no device
    s.chop_size, s.chop_stride, s.chop_bs = chop_size, chop_stride, chop_bs
    return s


def test_units_follow_one_gpu_call_order():
    s = _host_sampler(64, 48, 5)
    units = s._plan_units([(200, 148), (60, 50), (64, 64)])
    starts = plan_tiles(200, 148, 64, 48, 5)[4]
    assert [len(st) for st in starts] == [5, 5, 2]
    assert units == [(0, st, 64, 64) for st in starts] + [(1, [(0, 0)], 60, 50), (2, [(0, 0)], 64, 64)]
    for world in (1, 2, 5, 13):
        counts = s._share_counts([(200, 148), (60, 50), (64, 64)], world)
        assert [sum(c) for c in counts] == [12, 1, 1]
    assert s._share_counts([(200, 148), (60, 50), (64, 64)], 2) == [[12, 0], [0, 1], [0, 1]]       # units 0-2 | 3-4
    assert s._share_counts([(200, 148), (60, 50), (64, 64)], 4) == [[10, 2, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]]
    assert s._share_counts([(200, 148)], 13) == [[5, 5, 2] + [0] * 10]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        counts = [3, 0, 2]
        first = sum(counts[:rank])
        local = torch.arange(first, first + counts[rank], dtype=torch.float32)[:, None, None].repeat(1, 2, 3)
        full = gather_counts(local, counts)
        q.put((rank, full.shape == (5, 2, 3) and torch.equal(full[:, 0, 0], torch.arange(5, dtype=torch.float32))))
    finally:
        dist.destroy_process_group()


def test_gather_counts_world3_with_an_empty_rank():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 7) % 2000
    procs = [ctx.Process(target=_worker, args=(r, 3, port, q)) for r in range(3)]
    try:
        for p in procs:
            p.start()
        res = sorted(q.get(timeout=120) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join()
    assert res == [(0, True), (1, True), (2, True)]
