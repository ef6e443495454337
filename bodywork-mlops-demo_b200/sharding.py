"""Row sharding of the accumulated dataset over the GPUs of one box (one process per GPU).

The statistic S = [X 1 y]^T [X 1 y] is a sum over rows, so any row partition works: rank r accumulates
rows [lo, hi) and the only exchange is one all-reduce of (D+2)^2 doubles (b2_gram_allreduce).  Scoring shards
the same way and combines ten numbers (eight sums, two maxima: b2_score_allreduce).
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np

TILE_ROWS = 64  # rows per TMA tile of the tensor-core kernel: shard boundaries are tile aligned


def shard_bounds(n_rows: int, world: int, rank: int, align: int = TILE_ROWS) -> Tuple[int, int]:
    """Contiguous block [lo, hi) of rank `rank`; boundaries are multiples of `align`, blocks differ by at
    most one tile, the union is [0, n_rows) and blocks are disjoint."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError(f"bad rank {rank} for world size {world}")
    tiles = (n_rows + align - 1) // align
    lo_t = rank * tiles // world
    hi_t = (rank + 1) * tiles // world
    return min(lo_t * align, n_rows), min(hi_t * align, n_rows)


def all_shards(n_rows: int, world: int, align: int = TILE_ROWS) -> List[Tuple[int, int]]:
    return [shard_bounds(n_rows, world, r, align) for r in range(world)]


def combine_score_stats(parts: np.ndarray) -> np.ndarray:
    """Combine per-rank score reductions (10 per rank) the way b2_score_allreduce does: sums, maxima at 4 and 9."""
    parts = np.asarray(parts, dtype=np.float64).reshape(-1, 10)
    out = parts.sum(axis=0)
    out[4] = parts[:, 4].max()
    out[9] = parts[:, 9].max()
    return out
