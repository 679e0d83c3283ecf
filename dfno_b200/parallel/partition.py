"""Cartesian process partitions on top of ``torch.distributed``.

A :class:`Partition` is an ordered set of world ranks arranged on an N-D worker grid
(row-major).  It is the object every distributed layer takes as ``P_x`` and the public
workflow starts from :func:`create_standard_partitions`.  It plays the role DistDL's MPI
``Partition`` plays for the reference (contract: SURVEY.md §2.2 E1; call sites
reference ``dfno/utils.py:72-83``, reference ``dfno/dfno.py:83-97``) but is
built for one-process-per-GPU on a single NVSwitch box:

* rendezvous/control plane is ``torch.distributed`` (NCCL on GPU, gloo on CPU);
* process groups are created once per distinct rank set and cached (an NCCL communicator
  is expensive; the reference creates a fresh ``MPI_Cart_create`` per FNO block);
* with no process group initialised the world is a single rank, so every layer also runs
  unmodified in one process (unit tests, single-GPU runs).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from .decomposition import index_of_rank, rank_of_index

__all__ = ["Partition", "world_rank", "world_size", "create_standard_partitions",
           "create_root_partition"]

_GROUP_CACHE: Dict[Tuple[int, ...], object] = {}


def _dist_on() -> bool:
    return dist.is_available() and dist.is_initialized()


def world_rank() -> int:
    return dist.get_rank() if _dist_on() else 0


def world_size() -> int:
    return dist.get_world_size() if _dist_on() else 1


def _group_for(ranks: Sequence[int]):
    """Process group for a set of world ranks (collective over the WORLD on first use)."""
    key = tuple(sorted(int(r) for r in ranks))
    if not _dist_on() or len(key) <= 1:
        return None
    if key == tuple(range(world_size())):
        return dist.group.WORLD
    if key not in _GROUP_CACHE:
        _GROUP_CACHE[key] = dist.new_group(list(key))
    return _GROUP_CACHE[key]


def reset_group_cache() -> None:
    _GROUP_CACHE.clear()


class _CommShim:
    """Minimal stand-in for the raw communicator scripts reach through ``P._comm``
    (``Barrier`` at reference ``dfno/dfno.py:384``; ``allreduce`` MIN/MAX at
    ``training/two_phase/sleipner_dataset.py:93,96``)."""

    def __init__(self, part: "Partition"):
        self._p = part

    def Barrier(self) -> None:
        self._p.barrier()

    def Get_rank(self) -> int:
        return self._p.rank

    def Get_size(self) -> int:
        return self._p.size

    def allreduce(self, value, op="sum"):
        return self._p.allreduce_scalar(value, op)


class Partition:
    """Ordered set of world ranks on a Cartesian grid.

    Attributes mirror what the model/scripts use: ``active``, ``rank`` (rank *inside* the
    partition, ``-1`` when inactive), ``size``, ``shape`` (``np.ndarray``), ``dim``,
    ``index`` (grid coordinate tuple, ``None`` when inactive).
    """

    def __init__(self, ranks: Optional[Sequence[int]] = None, shape: Optional[Sequence[int]] = None):
        if ranks is None:
            ranks = range(world_size())
        self.world_ranks: Tuple[int, ...] = tuple(int(r) for r in ranks)
        if len(set(self.world_ranks)) != len(self.world_ranks):
            raise ValueError(f"duplicate ranks in partition: {self.world_ranks}")
        if shape is None:
            shape = [len(self.world_ranks)]
        self.shape = np.asarray([int(s) for s in shape], dtype=np.int64)
        if int(np.prod(self.shape)) != len(self.world_ranks):
            raise ValueError(f"grid {tuple(self.shape)} does not hold {len(self.world_ranks)} ranks")
        self.size = len(self.world_ranks)
        self.dim = len(self.shape)
        me = world_rank()
        self.active = me in self.world_ranks
        self.rank = self.world_ranks.index(me) if self.active else -1
        self.index = index_of_rank(self.shape, self.rank) if self.active else None
        self.group = _group_for(self.world_ranks)
        self._comm = _CommShim(self)

    # ------------------------------------------------------------------ construction
    def create_partition_inclusive(self, ranks: Sequence[int]) -> "Partition":
        """Sub-partition made of the listed ranks *of this partition* (1-D grid)."""
        ranks = [int(r) for r in np.asarray(ranks).reshape(-1)]
        for r in ranks:
            if not 0 <= r < self.size:
                raise ValueError(f"rank {r} outside partition of size {self.size}")
        return Partition([self.world_ranks[r] for r in ranks])

    def create_cartesian_topology_partition(self, shape: Sequence[int]) -> "Partition":
        """Arrange the first ``prod(shape)`` ranks of this partition on a grid.

        Like ``MPI_Cart_create`` the new partition may be smaller than its parent; the
        left-over ranks are simply inactive in it.
        """
        shape = [int(s) for s in np.asarray(shape).reshape(-1)]
        n = int(np.prod(shape))
        if n > self.size:
            raise ValueError(f"grid {shape} needs {n} ranks, partition has {self.size}")
        return Partition(self.world_ranks[:n], shape)

    # ------------------------------------------------------------------ queries
    def world_rank_of(self, index: Sequence[int]) -> int:
        return self.world_ranks[rank_of_index(self.shape, index)]

    def index_of(self, prank: int) -> Tuple[int, ...]:
        return index_of_rank(self.shape, prank)

    def is_root(self) -> bool:
        return self.active and self.rank == 0

    @property
    def root_world_rank(self) -> int:
        return self.world_ranks[0]

    def __eq__(self, other) -> bool:
        return (isinstance(other, Partition) and self.world_ranks == other.world_ranks
                and tuple(self.shape) == tuple(other.shape))

    def __hash__(self) -> int:
        return hash((self.world_ranks, tuple(int(s) for s in self.shape)))

    def __repr__(self) -> str:
        return (f"Partition(shape={tuple(int(s) for s in self.shape)}, ranks={self.world_ranks}, "
                f"rank={self.rank}, active={self.active})")

    def axis_group(self, axes: Sequence[int]):
        """Process group of the ranks that differ from this one only along ``axes``
        (e.g. ``axes=[0]``: the data-parallel replicas of a model shard).  Collective over
        the world on first use: every rank walks all such rank sets in the same order.
        Returns ``(group, world_ranks)``; group is None for singleton sets / inactive ranks."""
        import itertools
        axes = sorted(int(a) % self.dim for a in axes)
        others = [d for d in range(self.dim) if d not in axes]
        mine = (None, ())
        for fixed in itertools.product(*[range(int(self.shape[d])) for d in others]):
            ranks = []
            for var in itertools.product(*[range(int(self.shape[d])) for d in axes]):
                idx = [0] * self.dim
                for d, v in zip(others, fixed):
                    idx[d] = v
                for d, v in zip(axes, var):
                    idx[d] = v
                ranks.append(self.world_rank_of(idx))
            g = _group_for(ranks)
            if self.active and world_rank() in ranks:
                mine = (g, tuple(ranks))
        return mine

    # ------------------------------------------------------------------ small collectives
    def barrier(self) -> None:
        if self.group is not None and self.active:
            dist.barrier(group=self.group)

    def allreduce_scalar(self, value, op: str = "sum"):
        """All-reduce one python/torch scalar over the partition (host-side helper)."""
        was_tensor = torch.is_tensor(value)
        if self.group is None or not self.active:
            return value
        dev = value.device if was_tensor else _default_device()
        t = (value.detach().clone().reshape(1).to(dev) if was_tensor
             else torch.tensor([value], dtype=torch.float64, device=dev))
        opmap = {"sum": dist.ReduceOp.SUM, "min": dist.ReduceOp.MIN, "max": dist.ReduceOp.MAX}
        key = op if isinstance(op, str) else str(op).lower()
        for k, v in opmap.items():
            if k in key.lower():
                dist.all_reduce(t, op=v, group=self.group)
                break
        else:
            raise ValueError(f"unsupported reduction {op!r}")
        return t.reshape(()) if was_tensor else t.item()


def _default_device() -> torch.device:
    if _dist_on() and dist.get_backend() == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def create_root_partition(P: Partition) -> Partition:
    """Rank 0 of ``P`` as a ``[1]*dim`` grid (reference ``dfno/utils.py:72-75``)."""
    return P.create_partition_inclusive([0]).create_cartesian_topology_partition([1] * P.dim)


def create_standard_partitions(shape: Sequence[int]):
    """``(P_world, P_x, P_root)`` for a worker grid ``shape``.

    ``P_x`` spans the first ``prod(shape)`` world ranks (row-major on the grid) and
    ``P_root`` is its rank 0 (reference ``dfno/utils.py:77-83``).  If
    ``torch.distributed`` has not been initialised but the launcher environment
    (``RANK``/``WORLD_SIZE``) is present, the process group is created here: NCCL when CUDA
    is available, gloo otherwise.
    """
    from ..utils.env import ensure_process_group
    ensure_process_group()
    shape = [int(s) for s in shape]
    P_world = Partition()
    n = int(np.prod(shape))
    if n > P_world.size:
        raise ValueError(f"partition {tuple(shape)} needs {n} ranks but the world has {P_world.size}")
    P_x = P_world.create_partition_inclusive(np.arange(n)).create_cartesian_topology_partition(shape)
    return P_world, P_x, create_root_partition(P_x)
