"""``Repartition(P_a, P_b)``: move one global tensor from the balanced block decomposition over ``P_a`` to
the one over ``P_b`` (reference ``dfno/dfno.py:99-102``).  Every pair of workers whose blocks
overlap exchanges exactly that overlap; here all pairs go out in ONE ``all_to_all_single`` over the
world group (DistDL posts an Isend/Irecv per pair)."""
import numpy as np
import torch
import torch.distributed as dist

from ..backend.backend import _on, my_world_rank, n_world
from ..utilities.slicing import _cuts
from ._wire import collect_from_everyone


def _block(partition, world_rank, gshape):
    """[lo, hi) corner pair of ``world_rank``'s block of a ``gshape`` tensor, or None if it owns nothing."""
    pos = partition.grid_index_of(world_rank)
    if pos is None:
        return None
    lo = [int(_cuts(n, p)[i]) for n, p, i in zip(gshape, partition.shape, pos)]
    hi = [int(_cuts(n, p)[i + 1]) for n, p, i in zip(gshape, partition.shape, pos)]
    return lo, hi


def _meet(a, b, origin):
    """Intersection of two blocks as a slice tuple relative to ``origin`` (None if empty)."""
    if a is None or b is None:
        return None
    lo = [max(x, y) for x, y in zip(a[0], b[0])]
    hi = [min(x, y) for x, y in zip(a[1], b[1])]
    if any(h <= l for l, h in zip(lo, hi)):
        return None
    return tuple(slice(l - o, h - o) for l, h, o in zip(lo, hi, origin))


class _Route:
    """One direction of the exchange for this worker: what to cut out for whom, where arrivals go."""

    def __init__(self, P_from, P_to, gshape):
        me = my_world_rank()
        mine_from, mine_to = _block(P_from, me, gshape), _block(P_to, me, gshape)
        self.out_shape = tuple(h - l for l, h in zip(*mine_to)) if mine_to else (0,)
        self.cut, self.paste = [], []
        for w in range(n_world()):
            self.cut.append(_meet(mine_from, _block(P_to, w, gshape), mine_from[0]) if mine_from else None)
            self.paste.append(_meet(_block(P_from, w, gshape), mine_to, mine_to[0]) if mine_to else None)
        count = lambda box: int(np.prod([s.stop - s.start for s in box])) if box else 0   # noqa: E731
        self.n_out = [count(b) for b in self.cut]
        self.n_in = [count(b) for b in self.paste]

    def run(self, x, dtype):
        two = 2 if dtype.is_complex else 1
        real = {torch.complex64: torch.float32, torch.complex128: torch.float64}.get(dtype, dtype)
        pieces = []
        for box in self.cut:
            if box is not None:
                p = x[box].contiguous()
                pieces.append((torch.view_as_real(p) if two == 2 else p).reshape(-1))
        outbox = torch.cat(pieces) if pieces else torch.empty(0, dtype=real, device=x.device)
        inbox = torch.empty(sum(self.n_in) * two, dtype=real, device=x.device)
        if _on():
            dist.all_to_all_single(inbox, outbox, [n * two for n in self.n_in], [n * two for n in self.n_out])
        else:
            inbox.copy_(outbox)
        if self.out_shape == (0,):
            return torch.empty(0, dtype=dtype, device=x.device)
        out = torch.empty(self.out_shape, dtype=dtype, device=x.device)
        at = 0
        for box, n in zip(self.paste, self.n_in):
            if box is None:
                continue
            ext = [s.stop - s.start for s in box]
            chunk = inbox[at:at + n * two]
            out[box] = torch.view_as_complex(chunk.view(*ext, 2)) if two == 2 else chunk.view(ext)
            at += n * two
        return out


class _Move(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, layer):
        ctx.layer, ctx.given = layer, tuple(x.shape)
        return layer.there.run(x, layer.dtype)

    @staticmethod
    def backward(ctx, g):
        back = ctx.layer.back.run(g, ctx.layer.dtype)
        return back.reshape(ctx.given) if back.numel() == 0 else back, None


class Repartition(torch.nn.Module):
    def __init__(self, P_x, P_y, **_unused):
        super().__init__()
        self.P_x, self.P_y = P_x, P_y
        self.identity = P_x == P_y
        self.there = self.back = self.dtype = None

    def _setup(self, x):
        """First call (like DistDL): learn the global shape from the local blocks of ``P_x``."""
        known = collect_from_everyone((tuple(x.shape), x.dtype) if self.P_x.active else None)
        gshape = []
        for ax in range(self.P_x.dim):
            total = 0
            for i in range(int(self.P_x.shape[ax])):
                pos = [0] * self.P_x.dim
                pos[ax] = i
                total += known[self.P_x.member(pos)][0][ax] if _on() else known[0][0][ax]
            gshape.append(total)
        self.dtype = next(k[1] for k in known if k is not None)
        self.there = _Route(self.P_x, self.P_y, gshape)
        self.back = _Route(self.P_y, self.P_x, gshape)

    def forward(self, x):
        if self.identity:
            return x.clone()
        if self.there is None:
            self._setup(x)
        return _Move.apply(x, self)


DistributedTranspose = Repartition
