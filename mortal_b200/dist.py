"""Multi-GPU plumbing: tables shard embarrassingly (no data-path collective); the only exchange is one
all-gather of end-of-hanchan returns (scores i32[4] + rank u8[4] = 20 B/table) so that every rank holds all
returns for reward computation (SURVEY.md §8e; the reference itself has nothing distributed)."""
from __future__ import annotations

import numpy as np


def shard_seeds(seed_start, seed_count_per_rank: int, rank: int, games_per_seed: int = 4):
    """Contiguous block of seeds per rank; the `games_per_seed` seat rotations of a seed stay on one GPU."""
    start = int(seed_start[0]) + seed_count_per_rank * rank
    nonces = np.repeat(np.arange(start, start + seed_count_per_rank, dtype=np.uint64), games_per_seed)
    keys = np.full(nonces.shape[0], int(seed_start[1]), dtype=np.uint64)
    return nonces, keys


def seed_block(seed_count: int, rank: int, world: int):
    """(first seed offset, seed count) of the rank's contiguous block of `seed_count` seeds split over `world` ranks: the first
    seed_count % world ranks take one seed more, so the blocks cover every seed once, in rank order"""
    base, extra = divmod(seed_count, world)
    return rank * base + min(rank, extra), base + (rank < extra)


def gather_returns(scores, ranks, device=None):
    """all_gather of {scores i32[n,4], ranks u8[n,4]} -> (scores [world*n,4], ranks [world*n,4]) on every rank.
    Works with any initialised torch.distributed backend (nccl on GPUs, gloo in the CPU tests)."""
    import torch
    import torch.distributed as dist

    s = torch.as_tensor(np.ascontiguousarray(scores, dtype=np.int32))
    r = torch.as_tensor(np.ascontiguousarray(ranks, dtype=np.uint8)).to(torch.int32)
    packed = torch.cat([s, (r[:, 0] | (r[:, 1] << 8) | (r[:, 2] << 16) | (r[:, 3] << 24)).unsqueeze(1)], dim=1)
    if device is not None:
        packed = packed.to(device)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        out = packed
    else:
        out = torch.empty((dist.get_world_size() * packed.shape[0], 5), dtype=torch.int32, device=packed.device)
        dist.all_gather_into_tensor(out, packed.contiguous())
    out = out.cpu()
    pr = out[:, 4]
    ranks_all = torch.stack([(pr >> (8 * i)) & 0xFF for i in range(4)], dim=1).to(torch.uint8)
    return out[:, :4].numpy().copy(), ranks_all.numpy().copy()
