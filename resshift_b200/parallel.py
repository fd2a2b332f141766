"""Multi-GPU plumbing of the hot path: independent image shards, one weight broadcast, one final gather.

The path shards trivially (SURVEY.md §8e): every LR image is an independent sample and nothing inside
the T-step loop communicates.  Partitioning is the reference's (contiguous slices of size
ceil(bs / world) per rank, reference sampler.py:273-277).  Collectives go through ``torch.distributed``
(NCCL over NVLink on the GPU box, gloo in the CPU tests) — a broadcast of the flattened weights from
rank 0 at start-up and an all-gather of the result shards at the end.  Tile sharding
(``ResShiftSampler(shard_tiles=True)``) deals the tiles of a chunk instead and gathers them with ``gather_counts``.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

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
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world, rank = dist.get_world_size(), dist.get_rank()
    micro = math.ceil(batch / world)
    pad = torch.zeros((micro,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    outs: List[torch.Tensor] = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(outs, pad)
    parts = []
    for r in range(world):
        s, e = shard_range(batch, world, r)
        parts.append(outs[r][:e - s])
    return torch.cat(parts, dim=0)


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
