import torch
import torch.distributed as dist

from ..backend.backend import _on, my_world_rank
from ._wire import tell_everyone, unwire, wire


class _Bcast(torch.autograd.Function):
    """forward: root's tensor to every worker; backward: sum of the workers' gradients onto the root."""

    @staticmethod
    def forward(ctx, x, layer):
        ctx.layer, ctx.given = layer, tuple(x.shape)
        if layer.local:
            return x.clone()
        if layer.meta is None:                  # first call: root announces shape / dtype
            layer.meta = tell_everyone((tuple(x.shape), x.dtype) if layer.i_am_root else None, layer.root)
        shape, dtype = layer.meta
        out = x.detach().clone() if layer.i_am_root else torch.empty(shape, dtype=dtype, device=x.device)
        dist.broadcast(wire(out), src=layer.root)
        return out

    @staticmethod
    def backward(ctx, g):
        layer = ctx.layer
        if layer.local:
            return g, None
        buf = wire(g).clone()
        dist.reduce(buf, dst=layer.root, op=dist.ReduceOp.SUM)
        if layer.i_am_root:
            return unwire(buf, g.is_complex()).reshape(ctx.given), None
        return torch.empty(ctx.given, dtype=g.dtype, device=g.device), None


class Broadcast(torch.nn.Module):
    """``Broadcast(P_root, P_x)``: differentiable copy from a one-worker partition to all workers
    (reference ``dfno/dfno.py:41-42``).  Adjoint = :class:`SumReduce`."""

    def __init__(self, P_x, P_y, **_unused):
        super().__init__()
        assert P_x.size == 1, "the source of a Broadcast must be a single-worker partition"
        self.P_x, self.P_y = P_x, P_y
        self.root = P_x._members[0]
        self.i_am_root = my_world_rank() == self.root
        self.local = (not _on()) or dist.get_world_size() == 1 or P_y.size == 1 and P_y._members == P_x._members
        self.meta = None

    def forward(self, x):
        return _Bcast.apply(x, self)
