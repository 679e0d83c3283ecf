"""Optimizer set-up shared by the training scripts: Adam with an optional StepLR schedule, decoupled (AdamW) weight
decay and global gradient-norm clipping, on either backend.

On the fused engine all three run inside :class:`~dfno_b200.models.fused.FusedAdam` (device-side hyperparameters,
a device-side global norm).  On the portable backend they are ``torch.optim.Adam(decoupled_weight_decay=...)`` and
:func:`clip_grad_norm_global`, which is ``torch.nn.utils.clip_grad_norm_`` over the parameters of every rank."""
from __future__ import annotations

import argparse
import functools
from typing import Callable, Optional, Tuple

import torch
import torch.distributed as dist

__all__ = ["add_optimizer_args", "make_optimizer", "clip_grad_norm_global"]


def add_optimizer_args(ap: argparse.ArgumentParser) -> argparse.ArgumentParser:
    """The schedule / decay / clipping flags.  Their defaults keep plain Adam with L2 decay and a constant lr."""
    g = ap.add_argument_group("optimizer")
    g.add_argument("--lr-step-size", type=int, default=None,
                   help="StepLR: multiply the learning rate by --lr-gamma every this many epochs (default: constant)")
    g.add_argument("--lr-gamma", type=float, default=0.5, help="StepLR factor (with --lr-step-size)")
    g.add_argument("--clip-grad-norm", type=float, default=None,
                   help="clip the global gradient norm (all ranks' parameters) to this value")
    g.add_argument("--decoupled-weight-decay", action="store_true",
                   help="AdamW: decay the weights directly instead of adding weight_decay * w to the gradient")
    return ap


def _replica_copies(net) -> set:
    """ids of the parameters this rank holds as a data-parallel copy: the spectral shards of a batch-partitioned
    portable model, which every replica holds (and whose summed gradient every replica gets).  The first replica of
    each set counts them."""
    me = dist.get_rank() if dist.is_initialized() else 0
    out = set()
    for m in net.modules():
        ranks = getattr(m, "replica_ranks", ())
        if getattr(m, "replica_group", None) is not None and ranks and me != ranks[0]:
            out.update(id(p) for p in getattr(m, "weights", ()))
    return out


def clip_grad_norm_global(net, max_norm: float, group=None) -> torch.Tensor:
    """``clip_grad_norm_`` over the parameters of the whole model, where every rank of ``group`` holds a part of it:
    root-owned pointwise weights, spectral shards, and on a batch-partitioned partition data-parallel copies of those
    shards, counted once.  Collective over ``group`` on every call (a rank without gradients contributes zero).
    Returns the pre-clip norm."""
    params = [p for p in net.parameters() if p.numel() > 0]
    if group is None or not dist.is_initialized() or dist.get_world_size(group) <= 1:
        return torch.nn.utils.clip_grad_norm_(params, max_norm)
    copies = _replica_copies(net)
    if params:
        dev = params[0].device
    elif dist.get_backend(group) == "nccl":
        dev = torch.device("cuda", torch.cuda.current_device())
    else:
        dev = torch.device("cpu")
    sq = torch.zeros((), dtype=torch.float64, device=dev)
    for p in params:
        if p.grad is not None and id(p) not in copies:
            g = torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad
            sq = sq + torch.linalg.vector_norm(g, 2, dtype=torch.float64) ** 2
    dist.all_reduce(sq, group=group)
    total = sq.sqrt().to(torch.float32)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for p in params:
        if p.grad is not None:
            p.grad.mul_(coef.to(p.grad.device, p.grad.dtype))
    return total


def make_optimizer(net, args: argparse.Namespace, fused: bool, lr: float, weight_decay: float = 0.0, group=None
                   ) -> Tuple[Optional[torch.optim.Optimizer], Optional[object], Optional[Callable[[], object]]]:
    """``(optimizer, scheduler, clip)`` for ``args`` from :func:`add_optimizer_args`.  ``clip`` is ``None`` or a
    callable to run between the backward and ``optimizer.step()`` (portable backend; the fused optimizer clips in its
    step).  ``optimizer`` is ``None`` on a rank that holds no parameters."""
    if fused:
        from ..models.fused import FusedAdam
        opt = FusedAdam(net, lr=lr, weight_decay=weight_decay, decoupled_weight_decay=args.decoupled_weight_decay,
                        max_grad_norm=args.clip_grad_norm)
        clip = None
    else:
        params = [p for p in net.parameters() if p.numel() > 0]
        if not params:
            return None, None, None
        opt = torch.optim.Adam(params, lr=lr, weight_decay=weight_decay,
                               decoupled_weight_decay=args.decoupled_weight_decay)
        clip = (functools.partial(clip_grad_norm_global, net, args.clip_grad_norm, group)
                if args.clip_grad_norm is not None else None)
    sched = (torch.optim.lr_scheduler.StepLR(opt, step_size=args.lr_step_size, gamma=args.lr_gamma)
             if args.lr_step_size else None)
    return opt, sched, clip
