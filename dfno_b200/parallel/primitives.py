"""Differentiable data-movement primitives over :class:`Partition` objects.

``Broadcast`` / ``SumReduce`` are an adjoint pair, ``Repartition`` is its own adjoint
family (adjoint of ``P_a -> P_b`` is ``P_b -> P_a``).  These are the torch.distributed
(gloo / NCCL) implementations: they are the CPU path, the functional fallback for any
partition the fused sm_90a engine does not cover, and -- run over NCCL -- the measured
baseline.  Contracts follow SURVEY.md §2.2 (E2, E3, E4, E7, E8); reference call sites are
reference ``dfno/dfno.py:41-42,57-58,99-102`` and reference ``dfno/loss.py:17-35``.

Conventions
-----------
* A rank that owns nothing passes / receives a *zero-volume* tensor (``shape == (0,)``).
* All collectives run over the union of the two partitions' ranks.
* Metadata (global shape, dtype) is discovered lazily on the first call, like the
  reference, unless given explicitly -- which the models always do, so their hot path has
  no object collectives.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from .decomposition import overlap, shard_bounds
from .partition import Partition, _group_for, world_rank

__all__ = [
    "zero_volume_tensor", "is_zero_volume", "Broadcast", "SumReduce", "AllSumReduce",
    "Repartition", "DistributedTranspose", "ZeroVolumeCorrectorFunction", "RepartitionPlan",
    "build_repartition_plan", "replica_grad_sync",
]


def zero_volume_tensor(device=None, dtype=None, requires_grad: bool = False) -> torch.Tensor:
    """Placeholder for "this rank owns no part of the tensor"."""
    return torch.empty(0, device=device, dtype=dtype, requires_grad=requires_grad)


def is_zero_volume(t: torch.Tensor) -> bool:
    return t.numel() == 0


def _union(*parts: Partition) -> Tuple[int, ...]:
    seen: List[int] = []
    for p in parts:
        for r in p.world_ranks:
            if r not in seen:
                seen.append(r)
    return tuple(seen)


def _comm_view(t: torch.Tensor) -> torch.Tensor:
    """Real, contiguous view suitable for any backend (gloo has no complex collectives)."""
    t = t.contiguous()
    return torch.view_as_real(t) if t.is_complex() else t


# =====================================================================================
# Broadcast  <->  SumReduce
# =====================================================================================

class _RootLink:
    """Shared state of a root<->partition link: group, root rank, lazily agreed meta."""

    def __init__(self, P_root: Partition, P_all: Partition):
        if P_root.size != 1:
            raise NotImplementedError("Broadcast/SumReduce need a single-rank root partition")
        self.P_root, self.P_all = P_root, P_all
        self.ranks = _union(P_root, P_all)
        self.group = _group_for(self.ranks)
        self.root = P_root.world_ranks[0]
        self.member = world_rank() in self.ranks
        self.is_root = world_rank() == self.root
        self.meta = None  # (shape, dtype)

    def agree_meta(self, t: torch.Tensor):
        """Root tells everyone the tensor's shape/dtype (once)."""
        if self.meta is None:
            obj = [(tuple(t.shape), t.dtype) if self.is_root else None]
            if self.group is not None:
                dist.broadcast_object_list(obj, src=self.root, group=self.group)
            self.meta = obj[0]
        return self.meta


class _BroadcastFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, link: _RootLink):
        ctx.link = link
        ctx.in_shape = x.shape
        if link.group is None or not link.member:
            return x.clone() if link.is_root else x
        shape, dtype = link.agree_meta(x)
        out = x.detach().clone() if link.is_root else torch.empty(shape, dtype=dtype, device=x.device)
        buf = _comm_view(out)
        dist.broadcast(buf, src=link.root, group=link.group)
        return out

    @staticmethod
    def backward(ctx, g):
        link = ctx.link
        if link.group is None or not link.member:
            return (g if link.is_root else g.new_zeros(ctx.in_shape)), None
        buf = _comm_view(g).clone()
        dist.reduce(buf, dst=link.root, op=dist.ReduceOp.SUM, group=link.group)
        if link.is_root:
            out = torch.view_as_complex(buf) if g.is_complex() else buf
            return out.reshape(ctx.in_shape), None
        return g.new_zeros(ctx.in_shape), None


class _SumReduceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, link: _RootLink):
        ctx.link = link
        ctx.in_shape, ctx.in_dtype = x.shape, x.dtype
        if link.group is None or not link.member:
            return x.clone()
        buf = _comm_view(x).clone()
        dist.reduce(buf, dst=link.root, op=dist.ReduceOp.SUM, group=link.group)
        if link.is_root:
            return torch.view_as_complex(buf) if x.is_complex() else buf
        return zero_volume_tensor(device=x.device, dtype=x.dtype)

    @staticmethod
    def backward(ctx, g):
        link = ctx.link
        if link.group is None or not link.member:
            return g, None
        out = (g.detach().clone().contiguous() if link.is_root
               else torch.empty(ctx.in_shape, dtype=ctx.in_dtype, device=g.device))
        buf = _comm_view(out)
        dist.broadcast(buf, src=link.root, group=link.group)
        return out, None


class _AllSumReduceFn(torch.autograd.Function):
    """All-reduce(sum); self-adjoint."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        if group is None:
            return x.clone()
        buf = _comm_view(x).clone()
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
        return torch.view_as_complex(buf) if x.is_complex() else buf

    @staticmethod
    def backward(ctx, g):
        if ctx.group is None:
            return g, None
        buf = _comm_view(g).clone()
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=ctx.group)
        return (torch.view_as_complex(buf) if g.is_complex() else buf), None


class _ReplicaGradSyncFn(torch.autograd.Function):
    """Identity in the forward; all-reduce(sum) of the gradient over the replicas that hold
    a copy of the same parameter shard (data parallelism along the batch axis -- absent
    from the reference, SURVEY.md §2.4)."""

    @staticmethod
    def forward(ctx, w, group):
        ctx.group = group
        return w.view_as(w)

    @staticmethod
    def backward(ctx, g):
        buf = _comm_view(g).clone()
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=ctx.group)
        return (torch.view_as_complex(buf) if g.is_complex() else buf), None


def replica_grad_sync(w: torch.Tensor, group) -> torch.Tensor:
    return w if group is None else _ReplicaGradSyncFn.apply(w, group)


class Broadcast(nn.Module):
    """Copy a tensor from the single rank of ``P_src`` to every rank of ``P_dst``.
    Non-source ranks pass a zero-volume tensor.  Adjoint: :class:`SumReduce`."""

    def __init__(self, P_src: Partition, P_dst: Partition):
        super().__init__()
        self.P_src, self.P_dst = P_src, P_dst
        self.link = _RootLink(P_src, P_dst)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _BroadcastFn.apply(x, self.link)


class SumReduce(nn.Module):
    """Sum a same-shaped tensor from every rank of ``P_src`` onto the single rank of
    ``P_dst``; other ranks get a zero-volume tensor.  Adjoint: :class:`Broadcast`."""

    def __init__(self, P_src: Partition, P_dst: Partition):
        super().__init__()
        self.P_src, self.P_dst = P_src, P_dst
        self.link = _RootLink(P_dst, P_src)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _SumReduceFn.apply(x, self.link)


class AllSumReduce(nn.Module):
    """Sum over all ranks of ``P``, result everywhere (self-adjoint)."""

    def __init__(self, P: Partition):
        super().__init__()
        self.P = P

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _AllSumReduceFn.apply(x, self.P.group if self.P.active else None)


class ZeroVolumeCorrectorFunction(torch.autograd.Function):
    """Turn a zero-volume result into a scalar 0 so every rank
    can call ``.backward()``; the backward hands the original empty shape back.
    (contract: SURVEY.md §2.2 E7, used at reference ``dfno/loss.py:35``)."""

    @staticmethod
    def forward(ctx, x):
        ctx.in_shape = x.shape
        # decided from the shape alone: no device->host sync (keeps the step CUDA-graph capturable)
        ctx.was_empty = x.numel() == 0
        if ctx.was_empty:
            return x.new_zeros(())
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        if ctx.was_empty:
            return g.new_zeros(ctx.in_shape)
        return g.reshape(ctx.in_shape)


# =====================================================================================
# Repartition
# =====================================================================================

@dataclass
class RepartitionPlan:
    """Everything one rank needs to move its part of a global tensor from ``P_in``'s
    balanced decomposition to ``P_out``'s: per-peer pack/unpack boxes (local coordinates)
    in the order of the union process group, plus element counts for ``all_to_all_single``.
    """
    global_shape: Tuple[int, ...]
    in_shape: Tuple[int, ...]          # this rank's shard under P_in ((0,) if inactive)
    out_shape: Tuple[int, ...]         # this rank's shard under P_out ((0,) if inactive)
    ranks: Tuple[int, ...]             # union world ranks, group order
    send_boxes: List[Optional[Tuple[slice, ...]]] = field(default_factory=list)
    recv_boxes: List[Optional[Tuple[slice, ...]]] = field(default_factory=list)
    send_counts: List[int] = field(default_factory=list)
    recv_counts: List[int] = field(default_factory=list)
    identity: bool = False

    @property
    def bytes_sent_off_rank(self) -> int:
        me = self.ranks.index(world_rank()) if world_rank() in self.ranks else -1
        return sum(c for i, c in enumerate(self.send_counts) if i != me)


def _local_box(lo, hi, origin) -> Tuple[slice, ...]:
    return tuple(slice(int(a - o), int(b - o)) for a, b, o in zip(lo, hi, origin))


def build_repartition_plan(P_in: Partition, P_out: Partition, global_shape: Sequence[int],
                           me: Optional[int] = None) -> RepartitionPlan:
    """Overlap-based all-to-all-v plan (pure integer math; testable without a process group).

    ``me`` overrides the calling world rank (used by tests and the single-process simulator).
    """
    global_shape = tuple(int(s) for s in global_shape)
    if len(global_shape) != P_in.dim or P_in.dim != P_out.dim:
        raise ValueError(f"rank mismatch: tensor {global_shape}, P_in {tuple(P_in.shape)}, "
                         f"P_out {tuple(P_out.shape)}")
    me = world_rank() if me is None else int(me)
    ranks = tuple(sorted(_union(P_in, P_out)))      # torch groups are ordered by world rank

    def bounds(P: Partition, wr: int):
        if wr not in P.world_ranks:
            return None
        return shard_bounds(global_shape, P.shape, P.index_of(P.world_ranks.index(wr)))

    my_in, my_out = bounds(P_in, me), bounds(P_out, me)
    plan = RepartitionPlan(
        global_shape=global_shape,
        in_shape=tuple(b - a for a, b in zip(*my_in)) if my_in else (0,),
        out_shape=tuple(b - a for a, b in zip(*my_out)) if my_out else (0,),
        ranks=ranks,
        identity=(P_in == P_out),
    )
    for wr in ranks:
        sb = rb = None
        if my_in is not None:
            their_out = bounds(P_out, wr)
            if their_out is not None:
                ov = overlap(my_in[0], my_in[1], their_out[0], their_out[1])
                if ov is not None:
                    sb = _local_box(ov[0], ov[1], my_in[0])
        if my_out is not None:
            their_in = bounds(P_in, wr)
            if their_in is not None:
                ov = overlap(their_in[0], their_in[1], my_out[0], my_out[1])
                if ov is not None:
                    rb = _local_box(ov[0], ov[1], my_out[0])
        plan.send_boxes.append(sb)
        plan.recv_boxes.append(rb)
        plan.send_counts.append(int(np.prod([s.stop - s.start for s in sb])) if sb else 0)
        plan.recv_counts.append(int(np.prod([s.stop - s.start for s in rb])) if rb else 0)
    return plan


_P2P_POOL = {}


def _p2p_engine(group, ranks, needed_bytes: int):
    """Shared peer-memory all-to-all engine for a rank set (grown collectively on demand:
    ``needed_bytes`` is derived from the plans, hence identical on every rank)."""
    import os
    if os.environ.get("DFNO_P2P_REPARTITION", "1") == "0" or group is None or len(ranks) > 8:
        return None
    if dist.get_backend(group) != "nccl":
        return None
    key = tuple(ranks)
    eng = _P2P_POOL.get(key)
    if eng is None or eng.capacity < needed_bytes + 16 * len(ranks):
        try:
            from ..runtime.symm import P2PAllToAll
            cap = 1 << max(20, int(needed_bytes + 16 * len(ranks) - 1).bit_length())
            eng = P2PAllToAll(group, list(ranks).index(world_rank()), len(ranks), cap)
        except Exception as e:                               # noqa: BLE001 - IPC unavailable: NCCL path
            import warnings
            warnings.warn(f"peer-memory Repartition unavailable ({e}); using NCCL all_to_all")
            os.environ["DFNO_P2P_REPARTITION"] = "0"
            return None
        _P2P_POOL[key] = eng
    return eng


def _exchange(x: torch.Tensor, plan: RepartitionPlan, group, device, dtype, matrix=None) -> torch.Tensor:
    """Pack -> all-to-all-v -> unpack for one direction of a plan.  On CUDA the exchange runs
    over NVLink peer memory (``runtime.symm.P2PAllToAll``) when ``matrix`` (the full
    receive-count table) is given; otherwise ``all_to_all_single`` (gloo / NCCL)."""
    is_c = dtype.is_complex
    width = 2 if is_c else 1
    rdtype = (torch.float32 if dtype == torch.complex64 else torch.float64) if is_c else dtype
    send = torch.empty(sum(plan.send_counts) * width, dtype=rdtype, device=device)
    off = 0
    for box, cnt in zip(plan.send_boxes, plan.send_counts):
        if cnt:
            piece = x[box]
            piece = torch.view_as_real(piece.contiguous()) if is_c else piece
            send[off:off + cnt * width].view(piece.shape).copy_(piece)
            off += cnt * width
    recv = torch.empty(sum(plan.recv_counts) * width, dtype=rdtype, device=device)
    eng = None
    if group is not None and matrix is not None and device.type == "cuda":
        need = max(sum(-(-c * width * send.element_size() // 16) * 16 for c in row) for row in matrix)
        eng = _p2p_engine(group, plan.ranks, need)
    if group is None:
        recv.copy_(send)
    elif eng is not None:
        recv = eng.exchange(send, [c * width for c in plan.send_counts],
                            [[c * width for c in row] for row in matrix], copy=False)   # unpacked right below
    else:
        dist.all_to_all_single(recv, send,
                               [c * width for c in plan.recv_counts],
                               [c * width for c in plan.send_counts], group=group)
    if plan.out_shape == (0,):
        return zero_volume_tensor(device=device, dtype=dtype)
    out = torch.empty(plan.out_shape, dtype=dtype, device=device)
    off = 0
    for box, cnt in zip(plan.recv_boxes, plan.recv_counts):
        if cnt:
            shp = [s.stop - s.start for s in box]
            chunk = recv[off:off + cnt * width]
            chunk = torch.view_as_complex(chunk.view(*shp, 2)) if is_c else chunk.view(shp)
            out[box] = chunk
            off += cnt * width
    return out


class _RepartitionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fwd: RepartitionPlan, bwd: RepartitionPlan, group, dtype, mats):
        ctx.bwd, ctx.group, ctx.dtype, ctx.mats = bwd, group, dtype, mats
        ctx.in_shape = x.shape
        return _exchange(x, fwd, group, x.device, dtype, mats[0] if mats else None)

    @staticmethod
    def backward(ctx, g):
        gx = _exchange(g, ctx.bwd, ctx.group, g.device, ctx.dtype, ctx.mats[1] if ctx.mats else None)
        return gx.reshape(ctx.in_shape) if gx.numel() == 0 else gx, None, None, None, None, None


class Repartition(nn.Module):
    """Re-shard one global tensor from ``P_in``'s balanced block decomposition to
    ``P_out``'s.  Covers scatter (root -> grid), gather (grid -> root) and pencil
    transposes.  ``global_shape``/``dtype`` may be given up front; otherwise they are
    agreed on the first call.  Adjoint: ``Repartition(P_out, P_in)``."""

    def __init__(self, P_in: Partition, P_out: Partition, global_shape: Optional[Sequence[int]] = None,
                 dtype: Optional[torch.dtype] = None):
        super().__init__()
        self.P_in, self.P_out = P_in, P_out
        self.ranks = _union(P_in, P_out)
        self.group = _group_for(self.ranks)
        self.member = world_rank() in self.ranks
        self.dtype = dtype
        self.fwd_plan: Optional[RepartitionPlan] = None
        self.bwd_plan: Optional[RepartitionPlan] = None
        if global_shape is not None:
            self._build(global_shape)

    def _build(self, global_shape) -> None:
        self.fwd_plan = build_repartition_plan(self.P_in, self.P_out, global_shape)
        self.bwd_plan = build_repartition_plan(self.P_out, self.P_in, global_shape)
        # full receive-count tables (pure integer math) for the peer-memory data plane
        self.mats = None
        if self.group is not None and len(self.ranks) <= 8 and not self.fwd_plan.identity:
            order = self.fwd_plan.ranks
            f = [build_repartition_plan(self.P_in, self.P_out, global_shape, me=r).recv_counts for r in order]
            b = [build_repartition_plan(self.P_out, self.P_in, global_shape, me=r).recv_counts for r in order]
            self.mats = (f, b)

    def _discover(self, x: torch.Tensor) -> None:
        """Agree on global shape and dtype from the local shards (one object all-gather)."""
        mine = (tuple(x.shape), x.dtype) if self.P_in.active else None
        if self.group is None:
            metas = [mine]
        else:
            metas = [None] * len(self.ranks)
            dist.all_gather_object(metas, (world_rank(), mine), group=self.group)
            metas = [m for _, m in sorted(metas, key=lambda t: t[0])]
        by_rank = dict(zip(sorted(self.ranks), metas))
        P = self.P_in
        gshape = []
        for ax in range(P.dim):
            tot = 0
            for i in range(int(P.shape[ax])):
                idx = [0] * P.dim
                idx[ax] = i
                tot += by_rank[P.world_rank_of(idx)][0][ax]
            gshape.append(tot)
        if self.dtype is None:
            self.dtype = next(m[1] for m in metas if m is not None)
        self._build(gshape)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self.member:
            return x
        if self.fwd_plan is None or self.dtype is None:
            every_member_is_source = set(self.ranks) == set(self.P_in.world_ranks)
            if self.fwd_plan is not None and every_member_is_source:
                self.dtype = x.dtype       # nothing to agree on
            else:
                self._discover(x)          # collective over all members
        if self.P_in.active and tuple(x.shape) != tuple(self.fwd_plan.in_shape):
            raise ValueError(f"Repartition was planned for local shards of shape {self.fwd_plan.in_shape} "
                             f"(global {self.fwd_plan.global_shape}) but got {tuple(x.shape)}; use one "
                             f"Repartition module per tensor shape")
        if self.fwd_plan.identity:
            return x
        return _RepartitionFn.apply(x, self.fwd_plan, self.bwd_plan, self.group, self.dtype, self.mats)


#: DistDL's older name for the same operator (``experiment_navier_stokes.py:92,193``).
DistributedTranspose = Repartition
