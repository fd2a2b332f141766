"""Host-side pieces of attention teams (a chunk with fewer work units than ranks: each unit runs on a team of ranks that
splits the VQ-GAN bottleneck attention's query rows): the team partition, the row partition, the gather counts, and the
row exchange under gloo (world 4: a team of three and a team of one)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from resshift_b200.parallel import attention_row_ranges, attention_teams, row_exchange, team_group, unit_schedule
from resshift_b200.sampler import ResShiftSampler, tile_counts


def _host_sampler(chop_size, chop_stride, chop_bs):
    s = ResShiftSampler.__new__(ResShiftSampler)          # the planning methods need no device
    s.chop_size, s.chop_stride, s.chop_bs = chop_size, chop_stride, chop_bs
    return s


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 7, 8, 13, 16])
def test_teams_partition_the_ranks(world):
    for units in range(1, 20):
        teams = attention_teams(units, world)
        if units >= world:
            assert teams is None
            continue
        assert len(teams) == units
        assert teams[0][0] == 0 and teams[-1][1] == world
        for (a, e), (a2, _) in zip(teams, teams[1:]):
            assert e == a2                                # contiguous, disjoint, in rank order
        sizes = [e - a for a, e in teams]
        assert min(sizes) >= 1 and max(sizes) - min(sizes) <= 1, sizes
    assert attention_teams(1, 8) == [(0, 8)]
    assert attention_teams(3, 8) == [(0, 3), (3, 6), (6, 8)]
    assert attention_teams(2, 3) == [(0, 2), (2, 3)]


@pytest.mark.parametrize("T", [8256, 12288, 16384, 24576, 65536, 262144])
def test_row_blocks_are_covered_exactly_once(T):
    for size in range(1, 17):
        ranges = attention_row_ranges(T, size)
        assert len(ranges) == size
        covered = torch.zeros(T // 64, dtype=torch.int32)
        for b, e in ranges:
            assert b % 64 == 0 and e % 64 == 0 and 0 <= b <= e <= T
            covered[b // 64:e // 64] += 1
        assert bool((covered == 1).all()), (T, size)
        if size <= 8:
            assert all(e > b for b, e in ranges)         # every member of a team up to 8 computes rows
    assert attention_row_ranges(16384, 3) == [(0, 5504), (5504, 11008), (11008, 16384)]


def _counts(s, shapes, world, teams):
    units = s._plan_units(shapes)
    return tile_counts(units, unit_schedule(len(units), world, teams), world)


def test_schedule_counts_leader_only_with_fewer_units_than_ranks():
    s = _host_sampler(64, 48, 5)
    shapes = [(200, 148), (60, 50), (64, 64)]              # units: 3 of the pair's tiles (5, 5, 2) + 1 + 1
    units = s._plan_units(shapes)
    assert len(units) == 5
    for world in (1, 2, 3, 4, 5, 6, 7, 8, 13):
        counts = _counts(s, shapes, world, teams=True)
        if len(units) >= world:
            assert counts == _counts(s, shapes, world, teams=False)
            continue
        teams = unit_schedule(len(units), world, True)
        assert teams == attention_teams(len(units), world)
        firsts = {a for a, _ in teams}
        assert [sum(c) for c in counts] == [12, 1, 1]
        for g in range(len(shapes)):
            assert all(counts[g][r] == 0 for r in range(world) if r not in firsts)
    assert _counts(s, shapes, 8, teams=True) == [[5, 0, 5, 0, 2, 0, 0, 0], [0] * 6 + [1, 0], [0] * 7 + [1]]
    assert _counts(s, [(60, 50)], 3, teams=True) == [[1, 0, 0]]


def _exchange_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        groups = {}
        for a, e in [(0, 3), (3, 4)]:                      # every rank creates the multi-rank team's group
            if e - a > 1:
                team_group(tuple(range(a, e)), groups)
        N, T, Cc = 2, 640, 8                               # 10 row blocks over 3 members: 4, 4, 2
        full = torch.arange(N * T * Cc, dtype=torch.float32).reshape(N, T, Cc).half()
        ok = True
        if rank < 3:
            member = rank
            view = torch.full((N, T, Cc), -7.0, dtype=torch.float16)
            rb, re = attention_row_ranges(T, 3)[member]
            view[:, rb:re] = full[:, rb:re]
            row_exchange(team_group((0, 1, 2), groups), 3, member)(view, rb, re)
            ok = torch.equal(view, full)
        q.put((rank, ok, len(groups)))
    finally:
        dist.destroy_process_group()


def test_row_exchange_gloo_world4_team_of_three():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 11) % 2000
    procs = [ctx.Process(target=_exchange_worker, args=(r, 4, port, q)) for r in range(4)]
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
    assert res == [(0, True, 1), (1, True, 1), (2, True, 1), (3, True, 1)]
