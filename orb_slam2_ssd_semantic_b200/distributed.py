"""Multi-GPU plumbing (SURVEY §8(e)): one process per GPU, frames / keyframes sharded in contiguous ranges with no
data-path collective; the only exchange is the occupancy-map merge, ocm_merge_nccl (PointCloudMapping.merge()), which
replays the per-voxel clamp-add summaries of every rank in shard (= keyframe) order."""
from __future__ import annotations

from typing import Tuple


def shard_range(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous [begin, end) of `n` items for `rank`; the first n % world ranks get one extra item."""
    base, rem = divmod(n, world)
    b = rank * base + min(rank, rem)
    return b, b + base + (1 if rank < rem else 0)


def shard_frames_with_halo(n: int, world: int, rank: int) -> Tuple[int, int, int]:
    """Frame range of a rank for the stream pipeline plus its halo: SearchByProjection(t, t-1) needs the features of
    frame begin-1, which the rank re-extracts itself (cheaper than any transfer) -> (halo_begin, begin, end)."""
    b, e = shard_range(n, world, rank)
    return (max(b - 1, 0), b, e)
