"""Host-side pieces of tile sharding: the unit plan, the unit schedule and per-rank tile counts, and the variable-count
all-gather under gloo (world 3, one rank empty)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from resshift_b200.parallel import gather_counts, unit_schedule
from resshift_b200.sampler import ResShiftSampler, plan_tiles, tile_counts


def _host_sampler(chop_size, chop_stride, chop_bs):
    s = ResShiftSampler.__new__(ResShiftSampler)          # the planning methods need no device
    s.chop_size, s.chop_stride, s.chop_bs = chop_size, chop_stride, chop_bs
    return s


def _counts(s, shapes, world, teams=False):
    units = s._plan_units(shapes)
    return tile_counts(units, unit_schedule(len(units), world, teams), world)


def test_units_follow_one_gpu_call_order_and_schedule_counts():
    s = _host_sampler(64, 48, 5)
    units = s._plan_units([(200, 148), (60, 50), (64, 64)])
    starts = plan_tiles(200, 148, 64, 48, 5)[4]
    assert [len(st) for st in starts] == [5, 5, 2]
    assert units == [(0, st, 64, 64) for st in starts] + [(1, [(0, 0)], 60, 50), (2, [(0, 0)], 64, 64)]
    for world in (1, 2, 5, 13):
        counts = _counts(s, [(200, 148), (60, 50), (64, 64)], world)
        assert [sum(c) for c in counts] == [12, 1, 1]
    assert _counts(s, [(200, 148), (60, 50), (64, 64)], 2) == [[12, 0], [0, 1], [0, 1]]       # units 0-2 | 3-4
    assert _counts(s, [(200, 148), (60, 50), (64, 64)], 4) == [[10, 2, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]]
    assert _counts(s, [(200, 148)], 13) == [[5, 5, 2] + [0] * 10]


@pytest.mark.parametrize("chop_bs", [1, 5])
@pytest.mark.parametrize("teams", [False, True])
def test_schedule_runs_every_unit_and_keeps_it_once(chop_bs, teams):
    """Every unit is run by at least one rank and kept by exactly one, and the tiles each rank keeps (a rank runs the
    units whose executors [a, e) contain it and keeps those with rank == a) are its gather counts, with and without
    attention teams."""
    s = _host_sampler(64, 48, chop_bs)
    shapes = [(200, 148), (60, 50), (64, 64)]
    units = s._plan_units(shapes)
    for world in (1, 2, 3, 5, 8, 13):
        schedule = unit_schedule(len(units), world, teams)
        counts = tile_counts(units, schedule, world)
        assert len(schedule) == len(units)
        runs, keeps = [0] * len(units), [0] * len(units)
        for rank in range(world):
            kept = [0] * len(shapes)
            for u, ((g, starts, _, _), (a, e)) in enumerate(zip(units, schedule)):
                if a <= rank < e:
                    runs[u] += 1
                    if rank == a:
                        keeps[u] += 1
                        kept[g] += len(starts)
            assert kept == [c[rank] for c in counts], (world, rank)
        assert min(runs) >= 1 and keeps == [1] * len(units), (world, runs, keeps)
        assert [sum(c) for c in counts] == [12, 1, 1]
        if teams and len(units) < world:
            assert sum(runs) == world                      # every rank works on a unit
        else:
            assert runs == [1] * len(units)


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
