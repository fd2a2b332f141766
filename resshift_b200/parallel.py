"""Multi-GPU plumbing of the hot path: independent image shards, one weight broadcast, one final gather.

The path shards trivially (SURVEY.md §8e): every LR image is an independent sample and nothing inside
the T-step loop communicates.  Partitioning is the reference's (contiguous slices of size
ceil(bs / world) per rank, reference sampler.py:273-277).  Collectives go through ``torch.distributed``
(NCCL over NVLink on the GPU box, gloo in the CPU tests) — a broadcast of the flattened weights from
rank 0 at start-up and an all-gather of the result shards at the end.  Tile sharding
(``ResShiftSampler(shard_tiles=True)``) deals the tiles of a chunk instead, by ``unit_schedule``, and gathers them with
``gather_counts``; when a chunk has fewer units than ranks, the schedule gives each unit a team of ranks that splits the
VQ-GAN bottleneck attention's query rows and exchanges them (``row_exchange``).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(batch: int, world: int, rank: int) -> Tuple[int, int]:
    """[start, end) of rank's slice of a global batch (may be empty for trailing ranks)."""
    micro = math.ceil(batch / world)
    start = min(rank * micro, batch)
    return start, min(start + micro, batch)


def broadcast_state_dict(sd: Dict[str, torch.Tensor], src: int = 0) -> None:
    """In-place broadcast of all floating tensors of ``sd`` as ONE flat buffer (a single collective)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    keys = [k for k in sorted(sd) if sd[k].is_floating_point()]
    flat = torch.cat([sd[k].reshape(-1).float() for k in keys])
    dist.broadcast(flat, src=src)
    off = 0
    for k in keys:
        n = sd[k].numel()
        sd[k].copy_(flat[off:off + n].view_as(sd[k]))
        off += n


def gather_shards(local: torch.Tensor, batch: int) -> torch.Tensor:
    """All-gather variable-length shards (padded to ceil(batch/world)) and return the global batch."""
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    return gather_counts(local, [e - s for s, e in (shard_range(batch, world, r) for r in range(world))])


def gather_counts(local: torch.Tensor, counts: List[int]) -> torch.Tensor:
    """All-gather shards of known, unequal lengths: rank r holds ``counts[r]`` rows (possibly none), every rank passes
    the same ``counts``, and every rank gets all rows in rank order.  Shards are padded to ``max(counts)`` for one
    ``all_gather``; under gloo the exchange is staged through host memory."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world, rank = dist.get_world_size(), dist.get_rank()
    assert len(counts) == world and local.shape[0] == counts[rank], (counts, rank, tuple(local.shape))
    stage = torch.device("cpu") if dist.get_backend() == "gloo" else local.device
    pad = torch.zeros((max(counts),) + tuple(local.shape[1:]), dtype=local.dtype, device=stage)
    pad[:local.shape[0]] = local
    outs: List[torch.Tensor] = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(outs, pad)
    return torch.cat([o[:n] for o, n in zip(outs, counts)], dim=0).to(local.device)


def attention_teams(n_units: int, world: int) -> Optional[List[Tuple[int, int]]]:
    """Ranks [start, end) of the team that runs unit u, for a chunk of ``n_units`` work units on ``world`` ranks with
    fewer units than ranks: contiguous teams, in rank order, whose sizes differ by at most one (the larger ones first).
    None when every rank has a unit of its own to run (``n_units >= world``)."""
    if n_units < 1 or n_units >= world:
        return None
    base, extra = divmod(world, n_units)
    teams, start = [], 0
    for u in range(n_units):
        size = base + (1 if u < extra else 0)
        teams.append((start, start + size))
        start += size
    return teams


def unit_schedule(n_units: int, world: int, teams: bool) -> List[Tuple[int, int]]:
    """The executors (ranks, or a device pool's replicas) [a, e) that run each of a chunk's ``n_units`` work units;
    executor a keeps the unit's tiles.  With ``teams`` and fewer units than executors, the attention_teams partition;
    otherwise the units dealt as contiguous shard_range ranges, one executor each."""
    if teams and 0 < n_units < world:
        return attention_teams(n_units, world)
    return [(r, r + 1) for r in range(world) for _ in range(*shard_range(n_units, world, r))]


def attention_row_ranges(n_rows: int, size: int) -> List[Tuple[int, int]]:
    """[row_begin, row_end) of each of ``size`` team members for an attention over ``n_rows`` query rows (a multiple of
    64): the 64-row blocks dealt as shard_range does."""
    return [(64 * a, 64 * e) for a, e in (shard_range(n_rows // 64, size, m) for m in range(size))]


def team_group(ranks: Tuple[int, ...], cache: Dict[Tuple[int, ...], object]):
    """The process group of ``ranks``, created once.  dist.new_group must be entered by every rank of the default group,
    in the same order: callers ask for every team of a chunk in team order on every rank."""
    if ranks not in cache:
        cache[ranks] = dist.new_group(list(ranks))
    return cache[ranks]


def row_exchange(group, size: int, member: int):
    """``exchange(view, row_begin, row_end)`` for VQModelTorch.attention_team: all-gathers every member's rows of the
    [N, T, C] attention output ``view`` inside ``group`` (this member's are [row_begin, row_end)) and writes the other
    members' rows into ``view``.  Shares are padded to the largest for one ``all_gather``; under gloo the exchange is
    staged through host memory, as gather_counts does."""
    def exchange(view: torch.Tensor, row_begin: int, row_end: int) -> None:
        n, t, c = view.shape
        ranges = attention_row_ranges(t, size)
        assert ranges[member] == (row_begin, row_end), (ranges, member, row_begin, row_end)
        stage = torch.device("cpu") if dist.get_backend(group) == "gloo" else view.device
        pad = torch.zeros((n, max(e - b for b, e in ranges), c), dtype=view.dtype, device=stage)
        pad[:, :row_end - row_begin] = view[:, row_begin:row_end]
        outs: List[torch.Tensor] = [torch.empty_like(pad) for _ in range(size)]
        dist.all_gather(outs, pad, group=group)
        for m, (b, e) in enumerate(ranges):
            if m != member and e > b:
                view[:, b:e] = outs[m][:, :e - b].to(view.device)
    return exchange
