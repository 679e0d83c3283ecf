"""Root-owned pointwise linear layer.

``BroadcastedLinear`` applies ``y[.., o, ..] = sum_i W[o, i] x[.., i, ..] (+ b)`` along one
axis of an N-D field shard.  The parameters live **only on rank 0 of ``P_x``**; other ranks
hold zero-volume parameters (so optimizers and checkpoints see the same key set
everywhere).  Forward broadcasts ``W``/``b``; the autograd adjoint sum-reduces their
gradients back onto the root.  Spec: reference ``dfno/dfno.py:17-65``.

Differences by design: the bias parameter is only materialised when ``bias=True`` is
requested *or* ``ref_state_dict=True`` (checkpoint parity with the reference, which always
creates it, SURVEY.md §7.5); communication time is measured with the module-wide
:class:`~dfno_b200.utils.timers.CommTimer` rather than bare ``time.time()``.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ..parallel.partition import Partition, create_root_partition
from ..parallel.primitives import Broadcast, zero_volume_tensor
from ..utils.timers import CommTimer

__all__ = ["BroadcastedLinear", "BroadcastedAffineOperator"]


class BroadcastedLinear(nn.Module):
    def __init__(self, P_x: Partition, in_features: int, out_features: int, dim: int = -1,
                 bias: bool = True, device=torch.device("cpu"), dtype=torch.float32):
        super().__init__()
        self.P_x = P_x
        self.in_features, self.out_features = int(in_features), int(out_features)
        self.dim = dim if dim >= 0 else P_x.dim + dim
        self.bias = bool(bias)
        self.b_shape = [1] * P_x.dim
        self.b_shape[self.dim] = self.out_features
        self.P_root = create_root_partition(P_x)

        if self.P_root.active:
            W = torch.empty(self.out_features, self.in_features, device=device, dtype=dtype)
            nn.init.kaiming_uniform_(W, a=math.sqrt(5))
            self.W = nn.Parameter(W)
            self.b = nn.Parameter(torch.zeros(*self.b_shape, device=device, dtype=dtype))
        else:
            self.W = nn.Parameter(zero_volume_tensor(device=device, dtype=dtype))
            self.b = nn.Parameter(zero_volume_tensor(device=device, dtype=dtype))
        if not self.bias:
            self.b.requires_grad_(False)      # key kept for checkpoint parity, never trained

        self.W_bcast = Broadcast(self.P_root, P_x)
        self.b_bcast = Broadcast(self.P_root, P_x)
        self.W_bcast.link.meta = ((self.out_features, self.in_features), dtype)
        self.b_bcast.link.meta = (tuple(self.b_shape), dtype)
        # the contraction in einsum notation ("oi,ab..i..->ab..o.."), kept as an attribute for API
        # parity (reference dfno/dfno.py:44-49); the forward uses movedim + matmul instead
        letters = "abcdefghjklmnpqrstuvwxyz"[:P_x.dim]
        lhs = letters[:self.dim] + "i" + letters[self.dim + 1:]
        self.eqn = f"oi,{lhs}->{lhs.replace('i', 'o')}"
        self.timer = CommTimer()
        self.dt_comm = 0.0

    def extra_repr(self) -> str:
        return f"{self.in_features}->{self.out_features} along dim {self.dim}, bias={self.bias}"

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        self.timer.reset()
        with self.timer:
            W = self.W_bcast(self.W)
            b = self.b_bcast(self.b) if self.bias else None
        self.dt_comm = self.timer.seconds
        last = x.dim() - 1
        if self.dim != last:
            x = x.movedim(self.dim, last)
        y = torch.matmul(x, W.to(x.dtype).t())
        if self.dim != last:
            y = y.movedim(last, self.dim)
        if b is not None:
            y = y + b.to(y.dtype)
        return y


#: stale name imported by reference ``tests/gradient_test_distdl.py:7``
BroadcastedAffineOperator = BroadcastedLinear
