"""Batch normalisation over a domain-decomposed field.

The reference constructs two ``DistributedBatchNorm(P_x, width)`` modules and leaves them
out of the forward (reference ``dfno/dfno.py:325-326,340,346``); they matter only for
``state_dict()`` parity.  This is a complete implementation nonetheless (per-channel
statistics all-reduced over ``P_x`` so every shard normalises with the global mean and
variance), usable by models that want it.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ..parallel.partition import Partition
from ..parallel.primitives import _AllSumReduceFn

__all__ = ["DistributedBatchNorm"]


class DistributedBatchNorm(nn.Module):
    def __init__(self, P_x: Partition, num_features: int, eps: float = 1e-5, momentum: float = 0.1,
                 affine: bool = True, track_running_stats: bool = True,
                 device=torch.device("cpu"), dtype=torch.float32):
        super().__init__()
        self.P_x = P_x
        self.num_features, self.eps, self.momentum = int(num_features), eps, momentum
        self.affine, self.track_running_stats = affine, track_running_stats
        shape = [1] * P_x.dim
        shape[1] = self.num_features
        stat_dtype = torch.float32 if dtype in (torch.bfloat16, torch.float16) else dtype
        if affine:
            self.gamma = nn.Parameter(torch.ones(shape, device=device, dtype=stat_dtype))
            self.beta = nn.Parameter(torch.zeros(shape, device=device, dtype=stat_dtype))
        else:
            self.register_parameter("gamma", None)
            self.register_parameter("beta", None)
        if track_running_stats:
            self.register_buffer("running_mean", torch.zeros(shape, device=device, dtype=stat_dtype))
            self.register_buffer("running_var", torch.ones(shape, device=device, dtype=stat_dtype))
            self.register_buffer("num_batches_tracked", torch.zeros((), dtype=torch.long, device=device))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        dims = [d for d in range(x.dim()) if d != 1]
        xf = x.float() if x.dtype in (torch.bfloat16, torch.float16) else x
        if self.training or not self.track_running_stats:
            group = self.P_x.group if self.P_x.active else None
            stats = torch.stack([
                xf.sum(dim=dims, keepdim=True),
                (xf * xf).sum(dim=dims, keepdim=True),
                torch.full_like(xf.sum(dim=dims, keepdim=True), float(xf.numel() // xf.shape[1])),
            ])
            stats = _AllSumReduceFn.apply(stats, group)
            count = stats[2]
            mean = stats[0] / count
            var = (stats[1] / count - mean * mean).clamp_min(0)
            if self.track_running_stats and self.training:
                with torch.no_grad():
                    unbiased = var * count / (count - 1).clamp_min(1)
                    self.running_mean.lerp_(mean.to(self.running_mean.dtype), self.momentum)
                    self.running_var.lerp_(unbiased.to(self.running_var.dtype), self.momentum)
                    self.num_batches_tracked += 1
        else:
            mean, var = self.running_mean, self.running_var
        y = (xf - mean) * torch.rsqrt(var + self.eps)
        if self.affine:
            y = y * self.gamma + self.beta
        return y.to(x.dtype)
