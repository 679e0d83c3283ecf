"""Model-parallel Fourier Neural Operator -- portable (torch.fft / torch.distributed) backend.

This backend defines the *semantics* of the framework: any device, fp32/fp64 (bf16 is
up-cast inside the transforms), any Cartesian partition, gloo or NCCL.  On H100 the fused
sm_90a engine (:mod:`dfno_b200.models.fused`) computes the same function; run over NCCL,
this backend is also the measured baseline (``bench.py --impl baseline``).

Mathematical specification of one block (SURVEY.md §3.1; reference
reference ``dfno/dfno.py:241-291``)::

    y0  = W_lin ._c x                                          (no bias)
    X^  = Trunc( FFT_{axes 1..n-1}( RFFT_{axis n}(x) ) )       keep [0,m) u [N-m,N), rfft axis [0,m)
    Y^[b,o,k] = sum_i X^[b,i,k] R[i,o,k]
    y   = IRFFT_n( IFFT_{1..n-1}( ZeroPad(Y^) ) )
    out = gelu_erf(y0 + y)

with the field block-decomposed over ``P_x`` and the transform done in two local stages
(``P_m`` then ``P_y``, see :mod:`dfno_b200.parallel.planner`) joined by four Repartitions.
Spectral weights are sharded by Fourier mode over ``P_y`` and stored as one parameter per
non-empty low/high "corner" -- the reference's checkpoint layout.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from ..parallel.decomposition import shard_bounds
from ..parallel.partition import Partition
from ..parallel.planner import (corner_boxes, make_pencil_plan, spectrum_shape, validate_modes)
from ..parallel.primitives import Repartition, replica_grad_sync
from ..utils.misc import alphabet
from ..utils.timers import CommTimer
from .linear import BroadcastedLinear
from .norm import DistributedBatchNorm

__all__ = ["DistributedFNOBlock", "DistributedFNO", "DistributedFNONd", "infer_global_shape"]


def _complex_of(dtype: torch.dtype) -> torch.dtype:
    return torch.complex128 if dtype == torch.float64 else torch.complex64


def _keep_modes(x: torch.Tensor, dim: int, m: int, two_sided: bool) -> torch.Tensor:
    """Truncate a spectrum axis to its retained modes."""
    if not two_sided:
        return x.narrow(dim, 0, m)
    n = x.shape[dim]
    return torch.cat((x.narrow(dim, 0, m), x.narrow(dim, n - m, m)), dim=dim)


def _pad_modes(y: torch.Tensor, dim: int, m: int, n_full: int, two_sided: bool) -> torch.Tensor:
    """Inverse of :func:`_keep_modes`: scatter retained modes into a zero spectrum."""
    if y.shape[dim] == n_full:
        return y
    shape = list(y.shape)
    shape[dim] = n_full
    out = y.new_zeros(shape)
    out.narrow(dim, 0, m).copy_(y.narrow(dim, 0, m))
    if two_sided:
        out.narrow(dim, n_full - m, m).copy_(y.narrow(dim, m, m))
    return out


def _fft(x: torch.Tensor, dim: int, kind: str, n: Optional[int] = None) -> torch.Tensor:
    """torch.fft wrapper that tolerates zero-volume shards (a rank can own no modes when an
    axis has fewer retained modes than workers; MKL/cuFFT reject empty batches)."""
    if x.numel() == 0:
        # stay attached to the autograd graph: the backward of an empty shard must still
        # run the matching collectives on this rank
        shape = list(x.shape)
        tie = x.sum() * 0
        if kind == "rfft":
            shape[dim] = shape[dim] // 2 + 1
            return x.new_zeros(shape, dtype=_complex_of(x.dtype)) + tie
        if kind == "irfft":
            shape[dim] = n
            return x.new_zeros(shape, dtype=x.real.dtype) + tie.real
        return x
    if kind == "rfft":
        return torch.fft.rfft(x, dim=dim)
    if kind == "irfft":
        return torch.fft.irfft(x, n=n, dim=dim)
    return torch.fft.fft(x, dim=dim) if kind == "fft" else torch.fft.ifft(x, dim=dim)


class DistributedFNOBlock(nn.Module):
    """One Fourier layer on a ``P_x``-decomposed field.

    ``in_shape`` is the **global** ``[B, width, *spatial, T]``; ``modes`` has one entry per
    transformed axis (last = time / rfft axis).
    """

    def __init__(self, P_x: Partition, in_shape: Sequence[int], modes: Sequence[int],
                 device=torch.device("cpu"), dtype=torch.float32, plan: str = "reference",
                 fft_impl: str = "torch"):
        super().__init__()
        if fft_impl not in ("torch", "native"):
            raise ValueError("fft_impl is 'torch' (cuFFT / MKL) or 'native' (csrc/fft_radix.cu on CUDA tensors)")
        self.fft_impl = fft_impl
        self.P_x = P_x
        self.in_shape = [int(s) for s in in_shape]
        self.modes = [int(m) for m in modes]
        self.width = self.in_shape[1]
        self.n = P_x.dim - 2
        self.device, self.dtype = device, dtype
        self.compute_dtype = torch.float32 if dtype in (torch.bfloat16, torch.float16) else dtype
        self.dtype_complex = _complex_of(self.compute_dtype)
        validate_modes(self.in_shape, self.modes)

        # ---- pencil plan and the four re-shards
        self.fft_shape = spectrum_shape(self.in_shape, self.modes)
        self.plan = make_pencil_plan(P_x.shape, kind=plan, spectrum=self.fft_shape)
        self.dim_m = np.asarray(self.plan.dim_m)
        self.dim_y = np.asarray(self.plan.dim_y)
        self.P_m = P_x.create_cartesian_topology_partition(self.plan.grid_m)
        self.P_y = P_x.create_cartesian_topology_partition(self.plan.grid_y)

        # global shapes at the two re-shard points: full field, and spectrum after stage m
        shape_after_m = list(self.in_shape)
        for d in self.plan.dim_m:
            shape_after_m[d] = self.fft_shape[d]
        cdt = self.dtype_complex
        self.R1 = Repartition(P_x, self.P_m, self.in_shape, dtype=self.compute_dtype)
        self.R2 = Repartition(self.P_m, self.P_y, shape_after_m, dtype=cdt)
        self.R3 = Repartition(self.P_y, self.P_m, shape_after_m, dtype=cdt)
        self.R4 = Repartition(self.P_m, P_x, self.in_shape, dtype=self.compute_dtype)

        # ---- mode-restriction tables (API parity: dim -> retained count)
        rfft_dim = self.plan.rfft_dim
        self.restrict_prefixes = {int(d): self.modes[d - 2] for d in (*self.plan.dim_m, *self.plan.dim_y)}
        self.restrict_suffixes = {int(d): self.modes[d - 2] for d in (*self.plan.dim_m, *self.plan.dim_y)
                                  if d != rfft_dim}

        # ---- spectral weights: one parameter per non-empty corner of the local P_y slab
        self.scale = 1.0 / (self.width * self.width)
        self.weights = nn.ParameterList()
        self.slices: List[tuple] = []
        if self.P_y.active:
            start, stop = shard_bounds(self.fft_shape, self.P_y.shape, self.P_y.index)
            for box in corner_boxes(self.fft_shape, self.modes, start, stop):
                ext = [b - a for a, b in box]
                w = self.scale * torch.rand(self.width, self.width, *ext, device=device, dtype=cdt)
                self.weights.append(nn.Parameter(w))
                self.slices.append((slice(None), slice(None)) + tuple(slice(a, b) for a, b in box))

        # data-parallel replicas (batch axis of P_y partitioned) share each weight shard:
        # their gradients are summed in the backward ...
        self.replica_group, self.replica_ranks = self.P_y.axis_group([0])
        # ... so they must also START from the same values: every replica drew its shard from its own RNG
        # stream, the first rank of the replica set wins (without this the replicas train different models
        # forever while applying identical gradients)
        if self.replica_group is not None:
            import torch.distributed as dist
            with torch.no_grad():
                for w in self.weights:
                    buf = torch.view_as_real(w.data) if w.is_complex() else w.data
                    buf = buf.contiguous()
                    dist.broadcast(buf, src=self.replica_ranks[0], group=self.replica_group)
                    (torch.view_as_real(w.data) if w.is_complex() else w.data).copy_(buf)

        letters = alphabet(P_x.dim, as_array=True)
        xs, ws, ys = list(letters), list(letters), list(letters)
        xs[1], ws[0], ws[1], ys[1] = "i", "i", "o", "o"
        self.eqn = f"{''.join(xs)},{''.join(ws)}->{''.join(ys)}"

        self.linear = BroadcastedLinear(P_x, self.width, self.width, dim=1, bias=False,
                                        device=device, dtype=dtype)
        self.timer = CommTimer()
        self.dt_comm = 0.0

    # ------------------------------------------------------------------ API-parity helpers
    def restrict(self, x: torch.Tensor, dim: int) -> torch.Tensor:
        """Discard the unused high-frequency entries along ``dim``."""
        if dim not in self.restrict_prefixes:
            return x
        return _keep_modes(x, dim, self.restrict_prefixes[dim], dim in self.restrict_suffixes)

    def zeropad(self, y: torch.Tensor, dim: int, target_shape: Sequence[int]) -> torch.Tensor:
        """Re-insert zeros for the discarded entries along ``dim``."""
        if dim not in self.restrict_prefixes:
            return y
        return _pad_modes(y, dim, self.restrict_prefixes[dim], int(target_shape[dim]),
                          dim in self.restrict_suffixes)

    # ------------------------------------------------------------------ spectral path
    # transform + truncate / pad + inverse transform along one axis: torch.fft (cuFFT / MKL) or, with
    # ``fft_impl="native"`` on a GPU, the hand-written Stockham kernel with the truncation fused in (ops/fft.py)
    def _fwd(self, x: torch.Tensor, d: int, real_input: bool) -> torch.Tensor:
        m = self.modes[d - 2]
        if self.fft_impl == "native" and x.numel() and x.is_cuda and x.dtype in (torch.float32, torch.complex64):
            from ..ops.fft import fwd_transform
            return fwd_transform(x, d, m, real_input)
        return _keep_modes(_fft(x, d, 'rfft' if real_input else 'fft'), d, m, not real_input)

    def _inv(self, y: torch.Tensor, d: int, n_full: int, real_output: bool) -> torch.Tensor:
        m = self.modes[d - 2]
        if self.fft_impl == "native" and y.numel() and y.is_cuda and y.dtype == torch.complex64:
            from ..ops.fft import inv_transform
            return inv_transform(y, d, n_full, real_output)
        if real_output:
            return _fft(_pad_modes(y, d, m, n_full // 2 + 1, False), d, 'irfft', n=n_full)
        return _fft(_pad_modes(y, d, m, n_full, True), d, 'ifft')

    def spectral_forward(self, x: torch.Tensor) -> torch.Tensor:
        """``x`` (P_x shard, real) -> spectral branch output (P_x shard, real)."""
        t = self.timer
        rdim = self.plan.rfft_dim
        full = {}
        with t:
            x = self.R1(x)
        if self.P_m.active:
            full[rdim] = x.shape[rdim]
            x = self._fwd(x, rdim, True)
            for d in reversed(self.plan.dim_m[:-1]):
                full[d] = x.shape[d]
                x = self._fwd(x, d, False)
        with t:
            x = self.R2(x)
        if self.P_y.active:
            for d in reversed(self.plan.dim_y):
                full[d] = x.shape[d]
                x = self._fwd(x, d, False)
            # the corners tile the whole local slab, so every entry is written exactly once;
            # a rank that owns no modes keeps a (differentiable) empty tensor
            y = torch.empty_like(x) if len(self.weights) else x * 0
            for w, sl in zip(self.weights, self.slices):
                y[sl] = torch.einsum(self.eqn, x[sl], replica_grad_sync(w, self.replica_group))
            for d in self.plan.dim_y:
                y = self._inv(y, d, full[d], False)
        else:
            y = x
        with t:
            y = self.R3(y)
        if self.P_m.active:
            for d in self.plan.dim_m[:-1]:
                y = self._inv(y, d, full[d], False)
            y = self._inv(y, rdim, full[rdim], True)
        with t:
            y = self.R4(y)
        return y

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        self.timer.reset()
        y0 = self.linear(x)
        y = self.spectral_forward(x.to(self.compute_dtype))
        self.dt_comm = self.timer.seconds + self.linear.dt_comm
        return F.gelu(y0 + y.to(y0.dtype))


class DistributedFNO(nn.Module):
    """Lift (time axis ``T_in->T_out``, channels ``C_in->width``), ``num_blocks`` Fourier
    layers, projection ``width->128->out_channels``.  ``in_shape`` is the **global**
    ``[B, C_in, *spatial, T_in]``; the forward takes/returns this rank's ``P_x`` shard
    (reference ``dfno/dfno.py:293-353``).

    ``backend="auto"`` hands construction to the fused sm_90a engine when the device,
    dtype and partition are ones it covers (see :func:`dfno_b200.models.fused.supports`);
    ``backend="torch"`` forces this portable implementation.  ``input_grad=True`` asks for dL/dx on either backend
    (the fused engine refuses an input that requires grad without it).  ``out_channels`` (default 1) predicts that
    many fields from one trunk: the output is ``[B, out_channels, *spatial, T_out]``.

    ``padding`` (one non-negative int per transformed axis, in the order of ``modes``) makes the Fourier layers see a
    non-periodic field: the lifted field gets ``padding[a]`` zeros appended at the end of axis ``a``, the blocks run on
    the larger grid (``modes`` refer to it) and the result is cropped back before the projection head (Li et al.,
    FNO-3D).  ``None`` or all zeros is the periodic network.  The parameters do not depend on ``padding``, so a state
    dict loads across paddings -- but the function it computes changes.  Only axes the work partition ``P_work``
    does not split can be padded.
    """

    def __new__(cls, *args, backend: str = "auto", **kwargs):
        if cls is DistributedFNO and backend != "torch":
            from . import fused
            if fused.wants(args, kwargs, backend):
                return fused.FusedDistributedFNO(*args, **kwargs)
        return super().__new__(cls)

    def __init__(self, P_x: Partition, in_shape: Sequence[int], out_timesteps: int, width: int,
                 modes: Sequence[int], num_blocks: int = 4, device=torch.device("cpu"),
                 dtype=torch.float32, plan: str = "reference", backend: str = "auto",
                 init_seed: Optional[int] = None, fft_impl: str = "torch", input_grad: bool = False,
                 out_channels: int = 1, padding: Optional[Sequence[int]] = None):
        # input_grad: accepted for constructor parity with the fused engine (which returns dL/dx only when asked);
        # this backend always differentiates its input
        super().__init__()
        self.out_channels = check_out_channels(out_channels)
        self.padding = check_padding(padding, len(in_shape) - 2)
        if init_seed is not None:       # reproducible draw (per rank; the fused engine's is partition independent)
            torch.manual_seed(int(init_seed) + 7919 * max(int(P_x.rank), 0))
        self.P_x = P_x
        self.in_shape = [int(s) for s in in_shape]
        self.out_timesteps, self.width = int(out_timesteps), int(width)
        self.modes = [int(m) for m in modes]
        self.num_blocks = int(num_blocks)
        self.device, self.dtype = device, dtype
        if len(self.in_shape) != P_x.dim:
            raise ValueError(f"in_shape {self.in_shape} does not match partition rank {P_x.dim}")
        # The lift / projection contract the time and channel axes locally.  The reference is
        # silently wrong when those axes are partitioned (SURVEY.md 5.7 item 4); here such a P_x
        # is *defined*: the field is re-sharded once onto a work partition whose time/channel
        # workers are folded onto the roomiest spatial axis, the network runs there, and the
        # output is re-sharded back (BASELINE.json config 4: 8-way time-axis partition).
        self.P_outer = P_x
        self.R_in = self.R_out = None
        if int(P_x.shape[-1]) != 1 or int(P_x.shape[1]) != 1:
            work = [int(v) for v in P_x.shape]
            extra = work[1] * work[-1]
            work[1] = work[-1] = 1
            sp = list(range(2, P_x.dim - 1))
            tgt = max(sp, key=lambda d: self.in_shape[d] / work[d])
            work[tgt] *= extra
            if work[tgt] > self.in_shape[tgt]:
                raise ValueError(f"cannot fold {extra} time/channel workers onto a spatial axis of {self.in_shape}")
            out_shape = [self.in_shape[0], self.out_channels, *self.in_shape[2:-1], self.out_timesteps]
            P_work = P_x.create_cartesian_topology_partition(work)
            self.R_in = Repartition(P_x, P_work, self.in_shape, dtype=dtype)
            self.R_out = Repartition(P_work, P_x, out_shape, dtype=dtype)
            P_x = P_work
        self.P_work = P_x
        if self.padding is not None:
            split = [a for a, p in enumerate(self.padding) if p and int(P_x.shape[2 + a]) > 1]
            if split:
                raise ValueError(f"padding {list(self.padding)} pads transformed axes {split}, which the work "
                                 f"partition {tuple(int(s) for s in P_x.shape)} splits; only unsplit axes can be padded")

        self.block_in_shape = [self.in_shape[0], self.width, *self.in_shape[2:-1], self.out_timesteps]
        if self.padding is not None:            # the blocks run on the padded grid
            self.block_in_shape[2:] = [n + p for n, p in zip(self.block_in_shape[2:], self.padding)]
        kw = dict(device=device, dtype=dtype)
        self.linear1 = BroadcastedLinear(P_x, self.in_shape[-1], self.out_timesteps, dim=-1, **kw)
        self.linear2 = BroadcastedLinear(P_x, self.in_shape[1], self.width, dim=1, **kw)
        self.linear3 = BroadcastedLinear(P_x, self.width, 128, dim=1, **kw)
        self.linear4 = BroadcastedLinear(P_x, 128, self.out_channels, dim=1, **kw)
        self.blocks = nn.ModuleList(
            DistributedFNOBlock(P_x, self.block_in_shape, self.modes, plan=plan, fft_impl=fft_impl, **kw)
            for _ in range(self.num_blocks))
        # constructed for state-dict parity, not part of the forward (reference :325-346)
        self.bn1 = DistributedBatchNorm(P_x, self.width, **kw)
        self.bn2 = DistributedBatchNorm(P_x, self.width, **kw)
        self.dt_comm = 0.0

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        dt = 0.0
        if self.R_in is not None:
            x = self.R_in(x)
        x = F.gelu(self.linear1(x)); dt += self.linear1.dt_comm
        x = F.gelu(self.linear2(x)); dt += self.linear2.dt_comm
        if self.padding is not None:            # trailing zeros on every padded axis (last axis first for F.pad)
            x = F.pad(x, [v for p in reversed(self.padding) for v in (0, p)])
        for blk in self.blocks:
            x = blk(x); dt += blk.dt_comm
        if self.padding is not None:
            for a, p in enumerate(self.padding):
                if p:
                    x = x.narrow(2 + a, 0, x.shape[2 + a] - p)
        x = F.gelu(self.linear3(x)); dt += self.linear3.dt_comm
        x = self.linear4(x); dt += self.linear4.dt_comm
        if self.R_out is not None:
            x = self.R_out(x)
        self.dt_comm = dt
        return x


def check_out_channels(out_channels) -> int:
    """``out_channels`` as an int >= 1 (``ValueError`` otherwise)."""
    if isinstance(out_channels, bool) or not isinstance(out_channels, (int, np.integer)) or int(out_channels) < 1:
        raise ValueError(f"out_channels must be an integer >= 1, got {out_channels!r}")
    return int(out_channels)


def check_padding(padding, n_axes: int) -> Optional[tuple]:
    """``padding`` as a tuple of ``n_axes`` non-negative ints, or ``None`` when it pads nothing (``None`` or all
    zeros); ``ValueError`` otherwise."""
    if padding is None:
        return None
    if isinstance(padding, (str, bytes)) or not hasattr(padding, "__len__"):
        raise ValueError(f"padding must be None or a sequence of {n_axes} non-negative ints, got {padding!r}")
    if len(padding) != n_axes:
        raise ValueError(f"padding needs one entry per transformed axis ({n_axes}), got {len(padding)}: {padding!r}")
    for p in padding:
        if isinstance(p, bool) or not isinstance(p, (int, np.integer)) or int(p) < 0:
            raise ValueError(f"padding entries must be non-negative ints, got {padding!r}")
    out = tuple(int(p) for p in padding)
    return out if any(out) else None


def infer_global_shape(P: Partition, local_shape: Sequence[int]) -> List[int]:
    """Global tensor shape from every rank's balanced shard shape (one all-gather)."""
    import torch.distributed as dist
    local = [int(s) for s in local_shape]
    if P.group is None or not P.active:
        return local
    gathered = [None] * P.size
    dist.all_gather_object(gathered, (P.rank, local), group=P.group)
    by_rank = dict(gathered)
    out = []
    for ax in range(P.dim):
        tot = 0
        for i in range(int(P.shape[ax])):
            idx = [0] * P.dim
            idx[ax] = i
            tot += by_rank[int(np.ravel_multi_index(idx, tuple(int(s) for s in P.shape)))][ax]
        out.append(tot)
    return out


class DistributedFNONd(nn.Module):
    """Keyword-style, lazily-shaped front end kept for scripts written against the older
    API (reference ``tests/gradient_test_dfno.py:11-26``): no ``in_shape`` -- it is
    inferred from the first input shard.  ``decomposition_order`` and ``P_y`` are accepted
    and ignored (the pencil plan is derived from ``P_x``)."""

    def __init__(self, P_x: Partition = None, width: int = 20, modes: Sequence[int] = None,
                 out_timesteps: int = 1, decomposition_order: int = 1, num_blocks: int = 4,
                 device=torch.device("cpu"), dtype=torch.float32, P_y: Optional[Partition] = None,
                 in_shape: Optional[Sequence[int]] = None, **extra):
        super().__init__()
        self.P_x = P_x
        self._cfg = dict(out_timesteps=out_timesteps, width=width, modes=modes,
                         num_blocks=num_blocks, device=device, dtype=dtype, **extra)
        self.decomposition_order = decomposition_order
        self.net: Optional[DistributedFNO] = None
        if in_shape is not None:
            self._materialise(in_shape)

    def _materialise(self, in_shape) -> None:
        self.net = DistributedFNO(self.P_x, list(in_shape), **self._cfg)

    @property
    def dt_comm(self) -> float:
        return 0.0 if self.net is None else self.net.dt_comm

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.net is None:
            self._materialise(infer_global_shape(self.P_x, x.shape))
        return self.net(x)
