"""Losses over a ``P_x``-decomposed prediction.

Both reduce per-rank partial sums onto rank 0 with :class:`SumReduce` (adjoint:
Broadcast), so the scalar is *valid on the root rank* and a differentiable ``0`` elsewhere
-- every rank can call ``loss.backward()``.

* ``DistributedRelativeLpLoss``: batch mean of ``||y^-y||_p / ||y||_p`` with the norms taken
  over the whole (global) sample -- reference ``dfno/loss.py:8-35``.
* ``DistributedMSELoss``: global mean squared error (DistDL module the reference's
  scripts use: ``experiment_navier_stokes.py:118``, ``dfno.py:374``; SURVEY.md §2.2 E6).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ..parallel.partition import Partition, create_root_partition
from ..parallel.primitives import SumReduce, ZeroVolumeCorrectorFunction

__all__ = ["DistributedRelativeLpLoss", "DistributedMSELoss"]


def _acc_dtype(t: torch.Tensor) -> torch.dtype:
    return torch.float32 if t.dtype in (torch.bfloat16, torch.float16) else t.dtype


def _native_ok(y_hat: torch.Tensor, y: torch.Tensor) -> bool:
    """fp32 contiguous CUDA fields: the elementwise passes run as two native kernels (csrc/loss.cu)."""
    return (y_hat.is_cuda and y.is_cuda and y_hat.dtype == torch.float32 and y.dtype == torch.float32
            and y_hat.is_contiguous() and y.is_contiguous() and y_hat.shape == y.shape and y_hat.numel() > 0)


class _EngineReducedLoss(torch.autograd.Function):
    """Relative-L2 / MSE whose cross-rank sums need no NCCL call: ``engine`` is a fused engine (peer-memory
    all-reduce of the 2B partial sums, CUDA-graph capturable, value valid on *every* rank) or ``None`` for a
    partition of one rank.  On fp32 CUDA fields the forward is one pass over ``y_hat`` and ``y`` and the backward
    one pass writing the gradient (``csrc/loss.cu``) -- the autograd graph of the reference formulation
    (reference ``dfno/loss.py:8-35``) launches eight elementwise / reduction kernels and keeps the
    difference field alive between them."""

    @staticmethod
    def forward(ctx, y_hat, y, engine, kind):
        B = y_hat.shape[0]
        native = _native_ok(y_hat, y)
        if native:
            from ..ops import build
            C_ = build.load()
            nb = B if kind == "rel2" else 1
            part = torch.zeros(2 * nb, device=y_hat.device, dtype=torch.float32)
            C_.sq_partials(y_hat, y, part, nb)
            if kind != "rel2":
                part[1] = float(y_hat.numel())
            d = None
        else:
            d = y_hat.float() - y.float()
            if kind == "rel2":
                part = torch.cat([(d * d).reshape(B, -1).sum(1), (y.float() * y.float()).reshape(B, -1).sum(1)])
            else:
                part = torch.stack([(d * d).sum(), d.new_tensor(float(d.numel()))])
        tot = engine.allreduce_small_(part.contiguous()) if engine is not None else part
        if kind == "rel2":
            num, den = tot[:B].sqrt(), tot[B:].sqrt()
            out = (num / den).mean()
            ctx.save_for_backward(*((y_hat, y) if native else (d,)), num, den)
        else:
            out = tot[0] / tot[1]
            ctx.save_for_backward(*((y_hat, y) if native else (d,)), tot)
        ctx.kind, ctx.in_dtype, ctx.native = kind, y_hat.dtype, native
        return out

    @staticmethod
    def backward(ctx, g):
        saved = ctx.saved_tensors
        if ctx.kind == "rel2":
            num, den = saved[-2], saved[-1]
            B = num.shape[0]
            scale = ((g / B) / (num * den).clamp_min(1e-30)).to(torch.float32).contiguous()
        else:
            B, scale = 1, (2.0 * g / saved[-1][1]).reshape(1).to(torch.float32).contiguous()
        if ctx.native:
            from ..ops import build
            y_hat, y = saved[0], saved[1]
            grad = torch.empty_like(y_hat)
            build.load().scaled_diff(y_hat, y, scale, grad, B)
            return grad, None, None, None
        d = saved[0]
        grad = d * (scale.view(B, *([1] * (d.dim() - 1))) if ctx.kind == "rel2" else scale)
        return grad.to(ctx.in_dtype), None, None, None


class DistributedRelativeLpLoss(nn.Module):
    """``engine=<FusedDistributedFNO>`` (p = 2 only) routes the two scalar reductions through the
    engine's NVLink peer-memory all-reduce instead of NCCL; the loss is then valid on all ranks."""

    def __init__(self, P_x: Partition, p: float = 2, engine=None):
        super().__init__()
        self.P_x, self.p = P_x, p
        self.engine = engine if (engine is not None and getattr(engine, "world", 1) > 1 and p == 2
                                 and getattr(engine, "use_p2p", False)) else None
        self.local = P_x.active and P_x.size == 1 and p == 2        # one rank: nothing to reduce across
        self.P_0 = create_root_partition(P_x)
        self.sr0 = SumReduce(P_x, self.P_0)
        self.sr1 = SumReduce(P_x, self.P_0)

    def forward(self, y_hat: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        if self.engine is not None or (self.local and _native_ok(y_hat, y)):
            return _EngineReducedLoss.apply(y_hat, y, self.engine, "rel2")
        B = y_hat.shape[0]
        acc = _acc_dtype(y_hat)
        d = (y_hat.to(acc) - y.to(acc)).reshape(B, -1)
        r = y.to(acc).reshape(B, -1)
        if self.p == 2:
            num, den = (d * d).sum(dim=1), (r * r).sum(dim=1)
        else:
            num, den = d.abs().pow(self.p).sum(dim=1), r.abs().pow(self.p).sum(dim=1)
        num, den = self.sr0(num), self.sr1(den)
        if self.P_0.active:
            out = (num.pow(1.0 / self.p) / den.pow(1.0 / self.p)).mean()
        else:
            out = num            # zero-volume; corrected below
        return ZeroVolumeCorrectorFunction.apply(out)


class DistributedMSELoss(nn.Module):
    def __init__(self, P_x: Partition, engine=None):
        super().__init__()
        self.P_x = P_x
        self.engine = engine if (engine is not None and getattr(engine, "world", 1) > 1
                                 and getattr(engine, "use_p2p", False)) else None
        self.local = P_x.active and P_x.size == 1
        self.P_0 = create_root_partition(P_x)
        self.sr = SumReduce(P_x, self.P_0)

    def forward(self, y_hat: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        if self.engine is not None or (self.local and _native_ok(y_hat, y)):
            return _EngineReducedLoss.apply(y_hat, y, self.engine, "mse")
        acc = _acc_dtype(y_hat)
        d = y_hat.to(acc) - y.to(acc)
        part = torch.stack([(d * d).sum(), d.new_tensor(float(d.numel()))])
        tot = self.sr(part)
        out = tot[0] / tot[1] if self.P_0.active else tot
        return ZeroVolumeCorrectorFunction.apply(out)
