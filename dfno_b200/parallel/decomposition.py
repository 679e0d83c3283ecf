"""Balanced block decomposition of an N-D index space over a Cartesian worker grid.

This is the arithmetic every other layer (Repartition plans, spectral-weight shards,
checkpoint layout, the per-rank dataset slabs) is built on.  The rule is the one the
reference inherits from DistDL (contract described in SURVEY.md §2.2 E9 and used at
reference ``dfno/utils.py:58-70`` and ``training/two_phase/sleipner_dataset.py:51-52``):
a length ``n`` axis split over ``p`` workers gives the first ``n mod p`` workers
``ceil(n/p)`` entries and the rest ``floor(n/p)``.

Everything here is plain integer math (numpy), usable without torch.distributed.
"""
from __future__ import annotations

import itertools
from typing import Iterable, List, Sequence, Tuple

import numpy as np

__all__ = [
    "balanced_extent", "balanced_bounds", "axis_table",
    "compute_subtensor_shapes_balanced", "compute_subtensor_start_indices",
    "compute_subtensor_stop_indices", "assemble_slices", "compute_start_index",
    "compute_stop_index", "shard_bounds", "shard_shape", "overlap", "grid_indices",
    "rank_of_index", "index_of_rank",
]


def balanced_extent(n: int, p: int, i: int) -> int:
    """Number of entries worker ``i`` of ``p`` owns along an axis of length ``n``."""
    q, r = divmod(int(n), int(p))
    return q + (1 if i < r else 0)


def balanced_bounds(n: int, p: int, i: int) -> Tuple[int, int]:
    """Half-open ``[start, stop)`` owned by worker ``i`` of ``p`` along an axis of length ``n``."""
    q, r = divmod(int(n), int(p))
    start = i * q + min(i, r)
    return start, start + q + (1 if i < r else 0)


def axis_table(n: int, p: int) -> np.ndarray:
    """``(p, 2)`` table of ``[start, stop)`` for all workers on one axis."""
    return np.array([balanced_bounds(n, p, i) for i in range(p)], dtype=np.int64).reshape(p, 2)


def grid_indices(grid: Sequence[int]) -> Iterable[Tuple[int, ...]]:
    """Row-major walk over the worker grid (matches MPI Cartesian rank order)."""
    return itertools.product(*[range(int(g)) for g in grid])


def rank_of_index(grid: Sequence[int], index: Sequence[int]) -> int:
    return int(np.ravel_multi_index(tuple(int(i) for i in index), tuple(int(g) for g in grid)))


def index_of_rank(grid: Sequence[int], rank: int) -> Tuple[int, ...]:
    return tuple(int(i) for i in np.unravel_index(int(rank), tuple(int(g) for g in grid)))


def shard_bounds(shape: Sequence[int], grid: Sequence[int], index: Sequence[int]):
    """Per-axis ``[start, stop)`` of the shard owned by grid coordinate ``index``."""
    assert len(shape) == len(grid) == len(index), (shape, grid, index)
    b = [balanced_bounds(n, p, i) for n, p, i in zip(shape, grid, index)]
    return [s for s, _ in b], [e for _, e in b]


def shard_shape(shape: Sequence[int], grid: Sequence[int], index: Sequence[int]) -> List[int]:
    return [balanced_extent(n, p, i) for n, p, i in zip(shape, grid, index)]


def overlap(start_a, stop_a, start_b, stop_b):
    """Intersection of two boxes; returns ``(start, stop)`` lists or ``None`` when empty."""
    lo = [max(a, b) for a, b in zip(start_a, start_b)]
    hi = [min(a, b) for a, b in zip(stop_a, stop_b)]
    if any(h <= l for l, h in zip(lo, hi)):
        return None
    return lo, hi


# ---- array-valued helpers with the names/shapes the reference call sites expect -------------

def _as_shape(tensor_or_shape) -> Tuple[int, ...]:
    shp = getattr(tensor_or_shape, "shape", tensor_or_shape)
    return tuple(int(s) for s in shp)


def compute_subtensor_shapes_balanced(tensor_or_shape, grid) -> np.ndarray:
    """Array of shape ``(*grid, ndim)`` holding every worker's shard shape."""
    shape = _as_shape(tensor_or_shape)
    grid = tuple(int(g) for g in grid)
    out = np.zeros(grid + (len(shape),), dtype=np.int64)
    for idx in grid_indices(grid):
        out[idx] = shard_shape(shape, grid, idx)
    return out


def compute_subtensor_start_indices(shapes: np.ndarray) -> np.ndarray:
    """Exclusive prefix sums of ``shapes`` along each grid axis."""
    shapes = np.asarray(shapes)
    starts = np.zeros_like(shapes)
    nd = shapes.shape[-1]
    for ax in range(nd):
        c = np.cumsum(shapes[..., ax], axis=ax)
        starts[..., ax] = c - shapes[..., ax]
    return starts


def compute_subtensor_stop_indices(shapes: np.ndarray) -> np.ndarray:
    shapes = np.asarray(shapes)
    return compute_subtensor_start_indices(shapes) + shapes


def assemble_slices(start, stop) -> Tuple[slice, ...]:
    return tuple(slice(int(a), int(b), 1) for a, b in zip(start, stop))


def compute_start_index(grid, index, shape) -> np.ndarray:
    return np.array(shard_bounds(shape, grid, index)[0], dtype=np.int64)


def compute_stop_index(grid, index, shape) -> np.ndarray:
    return np.array(shard_bounds(shape, grid, index)[1], dtype=np.int64)
