import torch
import torch.distributed as dist

from ..backend.backend import _on, my_world_rank
from ._wire import unwire, wire


class _Reduce(torch.autograd.Function):
    """forward: sum over workers, result on the root, zero-volume elsewhere; backward: root's gradient to all."""

    @staticmethod
    def forward(ctx, x, layer):
        ctx.layer, ctx.given, ctx.dtype = layer, tuple(x.shape), x.dtype
        if layer.local:
            return x.clone()
        buf = wire(x).clone()
        dist.reduce(buf, dst=layer.root, op=dist.ReduceOp.SUM)
        if layer.i_am_root:
            return unwire(buf, x.is_complex())
        return torch.empty(0, dtype=x.dtype, device=x.device)

    @staticmethod
    def backward(ctx, g):
        layer = ctx.layer
        if layer.local:
            return g, None
        out = g.detach().clone().contiguous() if layer.i_am_root else torch.empty(ctx.given, dtype=ctx.dtype, device=g.device)
        dist.broadcast(wire(out), src=layer.root)
        return out.reshape(ctx.given), None


class SumReduce(torch.nn.Module):
    """``SumReduce(P_x, P_root)`` (reference ``dfno/loss.py:17-18``).  Adjoint = :class:`Broadcast`."""

    def __init__(self, P_x, P_y, **_unused):
        super().__init__()
        assert P_y.size == 1, "the target of a SumReduce must be a single-worker partition"
        self.P_x, self.P_y = P_x, P_y
        self.root = P_y._members[0]
        self.i_am_root = my_world_rank() == self.root
        self.local = (not _on()) or dist.get_world_size() == 1 or P_x.size == 1 and P_x._members == P_y._members
        self.meta = None

    def forward(self, x):
        return _Reduce.apply(x, self)
