"""Fused sm_90a engine for the model-parallel FNO (``backend="fused"``).

Same function as :class:`dfno_b200.models.fno.DistributedFNO` (spec: SURVEY.md §3.1), but
organised around H100 hardware instead of around ``torch.fft`` + MPI:

* **Layout.**  Activations live as ``h[b*C + c, x, y_local, t, z]`` in bf16 with ``z``
  contiguous.  The public tensors keep the reference layout ``[B, C, X, Y, Z, T]``; the lift
  and the projection head are the only places the layouts meet, so no transpose pass exists.
* **Transforms are GEMMs.**  Each truncated (inverse) DFT stage is ``lines x K`` times a tiny
  resident operator on wgmma (``csrc/dft_gemm_sm90.cu``), written by its epilogue directly
  in the layout -- and onto the GPU -- the next stage wants.  Complex data is interleaved
  (re, im) so a complex DFT is one real GEMM (``ops/operators.py``).
* **Pencil transposes are fused.**  With the field split along ``y`` over ``P`` GPUs, stage m
  (axes z, t) is local; its last GEMM scatters every (kz, kt) mode slab straight into the
  owning GPU's symmetric buffer over NVLink (Repartition R2), stage y (axes y, x), the
  per-mode channel mixing and the inverse stage y run on the mode-sharded data, and the
  inverse y-GEMM scatters back (R3).  R1/R4 are identities for a y-pencil.  Ordering is a
  device-side flag barrier (``csrc/p2p.cu``); there is no NCCL call on the hot path.
* **Weights.**  All parameters sit in ONE flat fp32 buffer ``theta``: the pointwise weights
  (replicated on every rank, kept identical by all-reducing their tiny gradient once per
  step -- the reference broadcasts each of them every forward) followed by this rank's
  spectral shard (modes ``kz in [rank*kzl, (rank+1)*kzl)``, all ``kt, ky, kx``).  One fused
  Adam launch updates the model.
* **Backward is the same chain.**  The adjoint of every stage has the shape of its mirror
  stage, so the backward runs the identical kernel sequence with transposed operators.

Reference call stack being replaced: ``dfno/dfno.py:241-291`` of the reference package (block),
``:330-353`` (model).
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from ..ops import operators as OPS
from ..ops.gemm import DFT_GEMM_SMEM, ScatterSpec, dft_gemm_fits, dft_gemm_min_smem, pad_operator
from ..parallel.partition import Partition

__all__ = ["FusedDistributedFNO", "FusedAdam", "supports", "wants", "EnginePlan", "fold_onto_pencil",
           "SUPPORTED_WIDTHS", "WIDE_WIDTHS"]

SUPPORTED_WIDTHS = (4, 8, 12, 16, 20, 24, 32)
# widths served by the round-2 route only (EnginePlan.fused_pw) with a single output channel: the wide-width spectral
# mix, lift backward and channel-major head kernels exist for them, the round-1 kernels do not
WIDE_WIDTHS = (48, 64)
MAX_OUT = 4                  # output channels of the multi-output head kernels (csrc/head_multi_sm90.cu)
MAX_IN = 16                  # input channels of the lift kernels (Cin > 4: lift_*_many_kernel, csrc/pointwise.cu)
MAX_N = 256                  # n_pad limit of dft_gemm (accumulator columns of one 64-row warpgroup tile)
HBM_BUDGET = 72 * 2 ** 30    # of an H100's 80 GB: leave room for the CUDA context, NCCL and the allocator
HEAD_HIDDEN = 128
LIFT_MAX_W = 4096            # floats of shared memory for the lift weights (kLiftMaxW, csrc/pointwise.cu)
H100_COPY_GBS = 3027.0       # device-to-device copy bandwidth (GB/s, read + write) measured on an H100 80GB HBM3 at 700 W


# =====================================================================================
# eligibility
# =====================================================================================

def _as_6d(grid: Sequence[int], in_shape: Sequence[int], modes: Sequence[int]):
    """The engine computes on 6-D ``[B, C, X, Y, Z, T]`` tensors.  A 2-D + time problem ``[B, C, X', Y', T]`` (the
    reference's Navier-Stokes trainer, ``experiment_navier_stokes.py:22,30``) is the same thing with a singleton
    leading spatial axis -- ``[B, C, 1, X', Y', T]`` is a free view -- whose (identity) x-transform the plan skips.
    Returns ``(grid6, in_shape6, modes6, five_d)``; lengths other than 5 / 6 give ``None``."""
    g, sh, m = [int(v) for v in grid], [int(v) for v in in_shape], [int(v) for v in modes]
    if len(g) == 6 and len(sh) == 6 and len(m) == 4:
        return g, sh, m, False
    if len(g) == 5 and len(sh) == 5 and len(m) == 3:
        return [g[0], g[1], 1, g[2], g[3], g[4]], [sh[0], sh[1], 1, sh[2], sh[3], sh[4]], [0, m[0], m[1], m[2]], True
    return None


def _pencil_axis(grid: Sequence[int]) -> Optional[int]:
    """Return the partitioned axis if ``grid`` (5-D or 6-D) is a supported 1 x P pencil, else None."""
    g = [int(v) for v in grid]
    if len(g) not in (5, 6):
        return None
    pa = len(g) - 3                       # the engine's y axis: public Y (6-D) / public X (5-D)
    parted = [i for i, v in enumerate(g) if v > 1]
    if not parted or parted == [pa]:
        return pa
    return None


def fold_onto_pencil(P_x: Partition, in_shape: Sequence[int], out_timesteps: int, out_channels: int = 1):
    """``(P_work, R_in, R_out)``: the y-pencil over ``P_x``'s ranks and the two re-shards that move
    the network input onto it and the ``out_channels``-channel output back (``None`` when ``P_x`` already is that
    pencil)."""
    if _pencil_axis(P_x.shape) is not None:
        return P_x, None, None
    from ..parallel.primitives import Repartition
    nd = int(P_x.dim)
    work = [1] * nd
    work[nd - 3] = int(np.prod(P_x.shape))
    P_work = P_x.create_cartesian_topology_partition(work)
    out_shape = [int(in_shape[0]), int(out_channels), *[int(v) for v in in_shape[2:-1]], int(out_timesteps)]
    return P_work, Repartition(P_x, P_work, [int(v) for v in in_shape]), Repartition(P_work, P_x, out_shape)


def supports(P_x: Partition, in_shape: Sequence[int], out_timesteps: int, width: int,
             modes: Sequence[int], out_channels: int = 1) -> Tuple[bool, str]:
    """Can the fused engine run this configuration?  Returns ``(ok, reason)``.

    The engine computes on a ``(1,1,1,P,1,1)`` y-pencil.  Any other 6-D ``P_x`` without a batch
    split (e.g. BASELINE config 3's ``(1,1,2,2,2,1)`` or config 4's 8-way time partition) is served
    by re-sharding the (small) network input onto that pencil once, running the engine there and
    re-sharding the output back -- instead of the reference's two full-resolution
    re-shards R1/R4 per Fourier layer (``dfno/dfno.py:247,288`` of the reference).  5-D (2-D + time)
    problems run as 6-D ones with a singleton x axis (:func:`_as_6d`).  ``out_channels`` > 1 (at most
    :data:`MAX_OUT`) runs the multi-output head kernels, which exist on the round-2 route only.  An
    ``out_channels`` that is not an integer >= 1 raises ``ValueError``."""
    from .fno import check_out_channels
    O = check_out_channels(out_channels)
    six = _as_6d(P_x.shape, in_shape, modes)
    if six is None:
        return False, "fused engine covers 2-D + time and 3-D + time fields (5-D / 6-D tensors)"
    grid, shape6, modes6, _ = six
    if grid[0] != 1:
        return False, "batch-partitioned P_x (data parallel) runs on the portable backend"
    P = int(np.prod(grid))
    B, Cin, X, Y, Z, Tin = shape6
    T = int(out_timesteps)
    mx, my, mz, mt = modes6
    if width not in SUPPORTED_WIDTHS + WIDE_WIDTHS:
        return False, f"width {width} not in {SUPPORTED_WIDTHS} (nor in {WIDE_WIDTHS}, the round-2 widths)"
    if O > MAX_OUT:
        return False, f"out_channels = {O}: the fused projection head covers 1 <= out_channels <= {MAX_OUT}"
    if O > 1 and 2 * (2 * mz) > 128:
        return False, (f"out_channels = {O} needs the round-2 route (2 * 2 * modes_z <= 128, here {4 * mz}); the "
                       f"round-1 head is single-output")
    if O > 1 and width > 31:
        return False, (f"out_channels = {O} at width {width}: the multi-output head backward covers width <= 31 "
                       f"(its consumer registers run out at 32)")
    if width in WIDE_WIDTHS and 2 * (2 * mz) > 128:
        return False, (f"width {width} needs the round-2 route (2 * 2 * modes_z <= 128, here {4 * mz}); the round-1 "
                       f"kernels cover widths {SUPPORTED_WIDTHS}")
    if P > 8:
        return False, "at most 8 peers (one NVSwitch box)"
    if Y % P or (2 * mz) % P:
        return False, "Y and 2*modes_z must divide evenly over the pencil"
    if Cin > MAX_IN or Tin > 64:
        return False, f"lift kernels cover Cin <= {MAX_IN} and Tin <= 64"
    lift_w = T * Tin + T + 2 * (width * Cin + width)
    if lift_w > LIFT_MAX_W:
        return False, (f"lift weights need {lift_w} floats of shared memory, more than the lift kernel's "
                       f"{LIFT_MAX_W} (kLiftMaxW)")
    # T % 4 != 0 (e.g. the reference's two-phase run and in-module demo, T = 30) uses a padded t pitch in Z1
    # (EnginePlan.Tp); covered by tests/test_fused_gpu.py
    if Z % 8 or T % 2 or Y % 4 or (X % 4 and X != 1) or (mx % 2 and X != 1) or my % 2 or mz % 2:
        return False, "extents must satisfy Z%8 = T%2 = X%4 = Y%4 = 0 and even modes (TMA pitch alignment)"
    if (X != 1 and 2 * mx > X) or 2 * my > Y or 2 * mz > Z or mt > T // 2 + 1:
        return False, "mode counts exceed the axes"
    if max(Z, 2 * T) > 256 or max(2 * X, 2 * Y) > 512:
        return False, "transformed axes: Z <= 256, T <= 128, X, Y <= 256 samples"
    if B * width * X * (Y // P) * Z * T >= 2 ** 31:
        return False, "per-rank activation must stay below 2^31 elements"
    pl = EnginePlan(B, Cin, Tin, width, T, X, Y, Z, modes6, world=P, rank=0, out_channels=O)
    pl.finish(4)
    need = pl.memory_bytes(train=True)["total"]
    if need > HBM_BUDGET:
        return False, (f"needs {need / 2 ** 30:.0f} GiB per GPU for training with 4 blocks "
                       f"(budget {HBM_BUDGET / 2 ** 30:.0f} GiB): use more GPUs or a smaller batch")
    # every GEMM stage keeps its operator (or, for the inverse stages of axes longer than 128 samples, each column
    # part of it) resident in shared memory; the adjoint chain's operators have the same shapes
    for staged in {False, P >= 8}:
        for st in pl.chain(staged=staged):
            if "N" not in st:
                continue
            try:
                parts = pl.parts(st)
            except ValueError as e:
                return False, str(e)
            for _, n, _, _, _ in parts:
                rows = 2 * n
                if not dft_gemm_fits(rows, st["K"]):
                    return False, (f"stage {st['name']}: a resident {rows} x {st['K']} operator needs "
                                   f"{dft_gemm_min_smem(rows, st['K']) // 1024} KiB of shared memory, more than "
                                   f"dft_gemm's {DFT_GEMM_SMEM // 1024} KiB")
    return True, ""


def wants(args, kwargs, backend: str) -> bool:
    """Should ``DistributedFNO(...)`` be served by the fused engine?"""
    if backend not in ("auto", "fused"):
        return False
    names = ["P_x", "in_shape", "out_timesteps", "width", "modes", "num_blocks", "device", "dtype"]
    cfg = dict(zip(names, args))
    cfg.update(kwargs)
    if "P_x" not in cfg or "in_shape" not in cfg:
        return False
    device = torch.device(cfg.get("device", "cpu"))
    dtype = cfg.get("dtype", torch.float32)
    try:
        ok, why = supports(cfg["P_x"], cfg["in_shape"], cfg["out_timesteps"], cfg["width"], cfg["modes"],
                           out_channels=cfg.get("out_channels", 1))
    except Exception as e:           # noqa: BLE001 - malformed arguments: let the portable constructor report them
        ok, why = False, f"{type(e).__name__}: {e}"
    if backend == "fused":
        if not ok:
            raise ValueError(f"backend='fused' requested but unsupported: {why}")
        if device.type != "cuda":
            raise ValueError("backend='fused' needs a CUDA device")
        return True
    return ok and device.type == "cuda" and dtype == torch.bfloat16 and cfg.get("plan", None) in (None, "balanced")


# =====================================================================================
# static plan: shapes, buffers, stage descriptors
# =====================================================================================

class EnginePlan:
    """All integer bookkeeping of one rank; no tensors, no CUDA -- unit-testable on CPU."""

    def __init__(self, B, Cin, Tin, C, T, X, Y, Z, modes, world=1, rank=0, hidden=HEAD_HIDDEN, out_channels=1):
        self.B, self.Cin, self.Tin, self.C, self.T = B, Cin, Tin, C, T
        self.O = int(out_channels)                         # output channels (fields) of the head
        self.X, self.Y, self.Z = X, Y, Z
        self.mx, self.my, self.mz, self.mt = [int(m) for m in modes]
        self.world, self.rank, self.H = world, rank, hidden
        self.max_n = MAX_N                                 # widest operator one GEMM launch keeps resident
        self.Yl = Y // world
        self.y_off = rank * self.Yl
        self.has_x = X > 1                                 # X == 1: 2-D + time problem, no x transform (see _as_6d)
        self.KX, self.KY, self.KZ = (2 * self.mx if self.has_x else 1), 2 * self.my, 2 * self.mz
        self.kzl = self.KZ // world
        self.kz_off = rank * self.kzl
        self.mtp = (self.mt + 3) // 4 * 4
        self.Tp = (T + 3) // 4 * 4                         # t pitch of Z1: G1b reads rows of 2*Tp bf16 (16-byte TMA pitch)
        self.BC = B * C
        self.S = X * self.Yl * T * Z                       # positions per (b, c) slab
        self.npos = B * self.S
        self.Q = self.kzl * self.mt * self.KY * self.KX    # local modes
        self.CP = (C + 7) // 8 * 8                         # channels-last pitch (16-byte rows)
        # Routes, decided by the shape: the module runs them, memory_bytes / cost_model size them.  fused_pw: the round-2
        # pointwise dataflow (the chain's last GEMM also applies bypass conv + GELU, csrc/spectral_out_sm90.cu), whose
        # inverse z-DFT takes K = 2*KZ <= 128; else round 1's separate bypass and channels-last head.  tc_bypass (round
        # 1 only): whole 128-position tiles for the tensor-core bypass, else CUDA cores + kreduce_gemm.  staged: chain()'s
        # staged peer layout pays once the direct NVLink runs get short (many ranks) and costs a permutation with few.
        self.fused_pw = 2 * self.KZ <= 128
        self.tc_bypass = self.S % 128 == 0
        self.staged = world >= 8
        # element counts (bf16 unless noted)
        BC, Yl, kzl, mt, mtp = self.BC, self.Yl, self.kzl, self.mt, self.mtp
        self.n_act = BC * self.S
        self.n_Z1 = BC * X * self.KZ * Yl * self.Tp * 2
        self.n_S1 = BC * kzl * mt * X * Y * 2
        self.n_S2 = BC * kzl * mt * self.KY * X * 2
        self.n_S3 = BC * self.Q * 2
        self.n_T2 = BC * X * kzl * mt * self.KY * 2
        self.n_T1 = BC * X * Yl * self.KZ * mtp * 2
        self.n_U = BC * X * Yl * T * self.KZ * 2
        # flat parameter layout (fp32 elements)
        self.segments: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
        off = 0

        def seg(name, *shape):
            nonlocal off
            self.segments[name] = (off, tuple(shape))
            off += int(np.prod(shape))

        seg("linear1.W", T, Tin); seg("linear1.b", T)
        seg("linear2.W", C, Cin); seg("linear2.b", C)
        self.num_blocks = None

    def finish(self, num_blocks: int) -> None:
        off = sum(int(np.prod(s)) for _, s in self.segments.values())
        C, H = self.C, self.H

        def seg(name, *shape):
            nonlocal off
            self.segments[name] = (off, tuple(shape))
            off += int(np.prod(shape))

        for k in range(num_blocks):
            seg(f"blocks.{k}.linear.W", C, C)
        seg("linear3.W", H, C); seg("linear3.b", H)
        seg("linear4.W", self.O, H); seg("linear4.b", self.O)          # adjacent: FusedDistributedFNO._w4b4
        self.n_small = (off + 63) // 64 * 64               # replicated segment (all-reduced)
        off = self.n_small
        for k in range(num_blocks):
            seg(f"blocks.{k}.spectral", C, C, self.Q, 2)
        self.n_theta = off
        self.num_blocks = num_blocks

    # ---------------------------------------------------------------- stage descriptors
    def chain(self, staged: bool = False) -> List[dict]:
        """The GEMM stages of one spectral convolution (forward *or* adjoint: only the operator
        matrices and the end buffers differ).  Strides in bf16 elements.

        ``staged`` (multi-GPU) changes how both pencil transposes cross NVLink: instead of
        interleaving directly into the consumer layout (64- / 40-byte runs per destination row)
        every source rank deposits its contribution as long contiguous runs into a per-source
        block of a staging buffer (``S1s`` / ``T1s``, >= 512-byte runs), and a tiny local
        permutation (``permS1`` / ``permT1``) produces the K-major layout of the next stage."""
        BC, X, Y, Z, T = self.BC, self.X, self.Y, self.Z, self.T
        Yl, KX, KY, KZ, kzl, mt, mtp = self.Yl, self.KX, self.KY, self.KZ, self.kzl, self.mt, self.mtp
        P, r = self.world, self.rank
        m_loc = kzl * mt
        Tp = self.Tp
        st = []
        if not staged:
            st.append(dict(name="G1a", src="src", dst="Z1", M=BC * X * Yl * T, K=Z, lda=Z, N=2 * KZ, op="G1a",
                           scatter=ScatterSpec(rows=[(T, 2), (Yl, 2 * Tp), (BC * X, KZ * Yl * Tp * 2)],
                                               cols=(KZ, Yl * Tp * 2, 0))))
            st.append(dict(name="G1b", src="Z1", dst="S1", M=BC * X * KZ * Yl, K=2 * T, lda=2 * Tp, N=2 * mt, op="G1b",
                           scatter=ScatterSpec(rows=[(Yl, 2), (KZ, mt * X * Y * 2), (X, Y * 2), (BC, m_loc * X * Y * 2)],
                                               cols=(mt, X * Y * 2, 0), peer=("row", 1, kzl), base_off=self.y_off * 2),
                           peer_dst=True, barrier_after=True))
        else:
            st.append(dict(name="G1a", src="src", dst="Z1", M=BC * X * Yl * T, K=Z, lda=Z, N=2 * KZ, op="G1a",
                           scatter=ScatterSpec(rows=[(T, 2), (Yl, 2 * Tp), (X, Yl * 2 * Tp), (BC, KZ * X * Yl * 2 * Tp)],
                                               cols=(KZ, X * Yl * 2 * Tp, 0))))
            st.append(dict(name="G1b", src="Z1", dst="S1s", M=BC * KZ * X * Yl, K=2 * T, lda=2 * Tp, N=2 * mt, op="G1b",
                           scatter=ScatterSpec(rows=[(Yl, 2), (X, Yl * 2), (KZ, mt * P * X * Yl * 2),
                                                     (BC, m_loc * P * X * Yl * 2)],
                                               cols=(mt, P * X * Yl * 2, 0), peer=("row", 2, kzl),
                                               base_off=r * X * Yl * 2),
                           peer_dst=True, barrier_after=True))
            # S1s[a=(bc,kzl,kt), r_src, x, y_loc] -> S1[a, x, (r_src, y_loc)]   (32-bit words = complex pairs)
            st.append(dict(name="permS1", src="S1s", dst="S1", size=[Yl, P, X, BC * m_loc],
                           sstr=[1, X * Yl, Yl, P * X * Yl], dstr=[1, Yl, Y, X * Y]))
        # X == 1: S2[bc, kz, kt, ky, x=1, ri] already is the row-major S3 layout and T2 the S4 layout, so the x stages vanish
        st.append(dict(name="G2", src="S1", dst="S2" if self.has_x else "S3", M=BC * m_loc * X, K=2 * Y, lda=2 * Y,
                       N=2 * KY, op="G2",
                       scatter=ScatterSpec(rows=[(X, 2), (BC * m_loc, KY * X * 2)], cols=(KY, X * 2, 0))))
        if self.has_x:
            st.append(dict(name="G3", src="S2", dst="S3", M=BC * m_loc * KY, K=2 * X, lda=2 * X, N=2 * KX, op="G3",
                           ldc=2 * KX))
        st.append(dict(name="mix"))
        if self.has_x:
            st.append(dict(name="iG3", src="S4", dst="T2", M=BC * m_loc * KY, K=2 * KX, lda=2 * KX, N=2 * X, op="iG3",
                           scatter=ScatterSpec(rows=[(KY, 2), (m_loc, KY * 2), (BC, X * m_loc * KY * 2)],
                                               cols=(X, m_loc * KY * 2, 0))))
        if not staged:
            st.append(dict(name="iG2", src="T2" if self.has_x else "S4", dst="T1", M=BC * X * m_loc, K=2 * KY,
                           lda=2 * KY, N=2 * Y, op="iG2",
                           scatter=ScatterSpec(rows=[(mt, 2), (kzl, mtp * 2), (X, Yl * KZ * mtp * 2),
                                                     (BC, X * Yl * KZ * mtp * 2)],
                                               cols=(Yl, KZ * mtp * 2, 0), peer=("col", Yl),
                                               base_off=self.kz_off * mtp * 2),
                           peer_dst=True, barrier_after=True))
        else:
            st.append(dict(name="iG2", src="T2" if self.has_x else "S4", dst="T1s", M=BC * X * m_loc, K=2 * KY,
                           lda=2 * KY, N=2 * Y, op="iG2",
                           scatter=ScatterSpec(rows=[(mt, 2), (kzl, mt * 2), (X, m_loc * 2),
                                                     (BC, P * Yl * X * m_loc * 2)],
                                               cols=(Yl, X * m_loc * 2, 0), peer=("col", Yl),
                                               base_off=r * Yl * X * m_loc * 2),
                           peer_dst=True, barrier_after=True))
            # T1s[bc, r_src, y_loc, x, kzl, kt] -> T1[bc, x, y_loc, (r_src, kzl), kt (pitch mtp)]
            st.append(dict(name="permT1", src="T1s", dst="T1", size=[mt, kzl, P, Yl, X, BC],
                           sstr=[1, mt, Yl * X * m_loc, X * m_loc, m_loc, P * Yl * X * m_loc],
                           dstr=[1, mtp, kzl * mtp, KZ * mtp, Yl * KZ * mtp, X * Yl * KZ * mtp]))
        st.append(dict(name="iG1b", src="T1", dst="U", M=BC * X * Yl * KZ, K=2 * mt, lda=2 * mtp, N=2 * T, op="iG1b",
                       scatter=ScatterSpec(rows=[(KZ, 2), (BC * X * Yl, T * KZ * 2)], cols=(T, KZ * 2, 0))))
        st.append(dict(name="iG1a", src="U", dst="dst", M=BC * X * Yl * T, K=2 * KZ, lda=2 * KZ, N=Z, op="iG1a",
                       ldc=Z))
        return st

    def parts(self, st: dict) -> List[Tuple[int, int, Optional[ScatterSpec], int, Optional[int]]]:
        """Column parts of one GEMM stage: ``[(j0, n_pairs, spec, first_peer, n_peers)]``.  A stage
        whose N fits one resident operator (``max_n``) is a single part; the inverse x / y stages of
        axes longer than 128 samples (N = 2X, 2Y up to 512) are issued as 2 or 4 launches, each with
        the operator rows ``[2*j0, 2*(j0+n))`` and the matching slice of the scatter."""
        npairs = st["N"] // 2
        if st["N"] <= self.max_n:
            return [(0, npairs, st.get("scatter"), 0, None)]
        if "scatter" not in st:
            raise ValueError(f"stage {st['name']}: row-major output wider than {self.max_n} is not supported")
        spec: ScatterSpec = st["scatter"]
        for k in range(2, npairs + 1):
            if npairs % k or 2 * (npairs // k) > self.max_n:
                continue
            n = npairs // k
            try:
                return [(j0, n) + spec.column_part(j0, n) for j0 in range(0, npairs, n)]
            except ValueError:
                continue
        raise ValueError(f"stage {st['name']}: no column split of {npairs} pairs fits {self.max_n}")

    def memory_bytes(self, train: bool = True) -> Dict[str, int]:
        """Per-rank device memory of the engine for this plan and its routes, by category (bytes).  Mirrors the
        allocations of :class:`FusedDistributedFNO` (``__init__``, ``_ensure_train_buffers``,
        ``_ensure_eval_buffers``) and :class:`FusedAdam`; used to size shards for the 80 GB of an H100
        before anything is allocated."""
        if self.num_blocks is None:
            raise RuntimeError("call finish(num_blocks) first")
        nb, bf, f32 = self.num_blocks, 2, 4
        legacy = not self.fused_pw
        cl = self.npos * self.CP                                   # channels-last slab
        out = {
            "parameters": self.n_theta * f32,
            "workspaces": (max(self.n_Z1, self.n_U) + self.n_S1 + self.n_T1 + self.n_S2 + 2 * self.n_S3 + self.n_T2) * bf,
            "staging": (((self.n_S1 + self.n_T1) * bf if self.staged else 0) + self.n_small * f32
                        if self.world > 1 else 0),
            "input_output": self.B * self.S // self.T * self.Cin * self.Tin * f32 + self.O * self.B * self.S * f32,
        }
        if train and legacy:            # round-1 dataflow: channels-last head, separate bypass
            out["saved_activations"] = (2 * nb * self.n_act + nb * self.n_S3 + cl) * bf
            out["backward_workspaces"] = (2 * self.n_act + cl) * bf
        elif train:                     # block inputs + last output, pre-activations, spectra entering the mix
            out["saved_activations"] = ((2 * nb + 1) * self.n_act + nb * self.n_S3) * bf
            out["backward_workspaces"] = self.n_act * bf
        if train:
            out["gradients"] = self.n_theta * f32
            out["adam_moments"] = 2 * self.n_theta * f32
        else:
            out["eval_activations"] = ((3 * self.n_act + cl) if legacy else 2 * self.n_act) * bf
        out["total"] = sum(out.values())
        return out

    def cost_model(self, hbm_gbs: float = H100_COPY_GBS, nvlink_gbs: Optional[float] = None,
                   front: bool = False) -> Dict[str, object]:
        """Bytes every kernel of one training step must move (per rank) on this plan's routes and the resulting
        floors.  ``front``: G1a + G1b run as the single ``spectral_in`` kernel (Z1 stays on the SM).

        Pure bookkeeping of the dataflow in :class:`FusedDistributedFNO` -- each stage reads its input
        buffer and writes its output buffer once; nothing is assumed to stay in L2 (the working set of a
        stage is far above the 50 MB L2 for the configurations this is meant for).  ``hbm_gbs`` defaults to
        the device-to-device copy bandwidth measured on an H100 (:data:`H100_COPY_GBS`); without
        ``nvlink_gbs`` the NVLink time is not estimated (``nvlink_ms`` is None).  Returns ``{"stages": [(name, calls_per_step, hbm_bytes, nvlink_bytes)], "hbm_bytes",
        "nvlink_bytes", "hbm_floor_ms", "nvlink_ms"}``; the NVLink time is overlappable (the transfers are
        issued from GEMM epilogues), so the step floor is ``max`` of the two per chain, not their sum."""
        if self.num_blocks is None:
            raise RuntimeError("call finish(num_blocks) first")
        nb, bf, f32 = self.num_blocks, 2, 4
        legacy = not self.fused_pw
        P = self.world
        act, cl = self.n_act * bf, self.npos * self.CP * bf
        x_in = self.B * self.S // self.T * self.Cin * self.Tin * f32    # the network input (fp32, as memory_bytes)
        Z1, S1, S2, S3, T2, U = (self.n_Z1 * bf, self.n_S1 * bf, self.n_S2 * bf, self.n_S3 * bf, self.n_T2 * bf,
                                 self.n_U * bf)
        T1 = self.n_T1 // self.mtp * self.mt * bf                      # valid (kt < mt) part
        W = self.C * self.C * self.Q * 2 * f32                         # one block's spectral shard
        off = (P - 1) / P if P > 1 else 0.0
        chain = [("G1a", act + Z1, 0), ("G1b", Z1 + S1, S1 * off), ("G2", S1 + S2, 0), ("G3", S2 + S3, 0),
                 ("iG3", S3 + T2, 0), ("iG2", T2 + T1, T1 * off), ("iG1b", T1 + U, 0)]
        if front and not legacy:
            chain = [("spectral_in", act + S1, S1 * off)] + chain[2:]
        if not self.has_x:
            chain = [c for c in chain if c[0] not in ("G3", "iG3")]
        if legacy:
            chain.append(("iG1a", U + act, 0))
        if P > 1 and self.staged:
            chain += [("permS1", 2 * S1, 0), ("permT1", 2 * T1, 0)]
        st = [(n, 2 * nb, b, l) for n, b, l in chain]                  # forward + adjoint chain per block
        st += [("spectral_mix fwd", nb, 2 * S3 + W, 0), ("spectral_mix bwd", nb, 3 * S3 + 2 * W, 0),
               ("lift fwd", 1, act + x_in, 0), ("lift bwd", 1, act + x_in, 0), ("adam", 1, 7 * self.n_theta * f32, 0)]
        if legacy:
            st += [("iG1a add (bwd)", nb, act, 0), ("bypass fwd", nb, 4 * act, 0), ("bypass bwd", nb, 5 * act, 0),
                   ("head fwd", 1, cl + self.O * self.npos * f32, 0), ("head bwd", 1, 2 * cl + self.O * self.npos * f32, 0)]
        else:
            # the chain's last GEMM also applies the bypass conv (+ GELU): reads U and the block input, writes the
            # pre-activation and the output (forward) / reads U and dpre, writes the input gradient (adjoint)
            st += [("spectral_out fwd", nb, U + 3 * act, 0), ("spectral_out adj", nb, U + 2 * act, 0),
                   ("dpre_dw", nb, 4 * act, 0),
                   ("head fwd", 1, act + self.O * self.npos * f32, 0),
                   ("head bwd", 1, 2 * act + 2 * self.O * self.npos * f32, 0)]
        hbm = sum(c * b for _, c, b, _ in st)
        link = sum(c * l for _, c, _, l in st)
        return {"stages": st, "hbm_bytes": hbm, "nvlink_bytes": link,
                "hbm_floor_ms": hbm / (hbm_gbs * 1e9) * 1e3,
                "nvlink_ms": (link / (nvlink_gbs * 1e9) * 1e3 if link else 0.0) if nvlink_gbs else None}

    def operators(self) -> Dict[str, torch.Tensor]:
        """Forward-chain operators (float64) and their adjoint-chain counterparts (``*_adj``)."""
        X, Y, Z, T = self.X, self.Y, self.Z, self.T
        f = {
            "G1a": OPS.fwd_real_to_complex(Z, self.mz), "G1b": OPS.fwd_complex(T, self.mt, False),
            "G2": OPS.fwd_complex(Y, self.my), "iG2": OPS.inv_complex(Y, self.my),
            "iG1b": OPS.inv_complex_hermitian(T, self.mt), "iG1a": OPS.inv_complex_to_real(Z, self.mz),
        }
        mirror = {"G1a": "iG1a", "G1b": "iG1b", "G2": "iG2", "iG2": "G2", "iG1b": "G1b", "iG1a": "G1a"}
        if self.has_x:
            f["G3"], f["iG3"] = OPS.fwd_complex(X, self.mx), OPS.inv_complex(X, self.mx)
            mirror.update({"G3": "iG3", "iG3": "G3"})
        out = dict(f)
        for slot, src in mirror.items():       # the adjoint chain's stage in slot X is adj(mirror(X))
            out[slot + "_adj"] = f[src].t().contiguous()
        return out


# =====================================================================================
# the module
# =====================================================================================

class _NoRange:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


_NO_RANGE = _NoRange()


def _nvtx(name: str):
    """NVTX range around an engine phase when ``DFNO_NVTX=1`` (for Nsight timelines); free otherwise."""
    if os.environ.get("DFNO_NVTX", "0") == "0":
        return _NO_RANGE
    from ..utils.timers import nvtx_range
    return nvtx_range(name)


class _LaunchCounter:
    """Proxy around the extension module that counts kernel launches issued by the engine
    (reported by ``bench.py`` as ``gpu_launches``)."""

    _multi = {"spectral_mix_bwd": "B"}

    def __init__(self, mod):
        self._mod = mod
        self.count = 0

    def __getattr__(self, name):
        fn = getattr(self._mod, name)
        if name.startswith(("symm_", "tensor_from_ptr")) or name.endswith("_check"):
            return fn

        def call(*a, **k):
            self.count += 1
            return fn(*a, **k)
        return call


class _FusedFn(torch.autograd.Function):
    """Autograd edge of the engine.  The saved activations live in ONE engine-owned buffer set, so a backward is
    only valid for the most recent saving forward: every such forward gets a generation number and a stale
    backward raises instead of silently using another forward's activations (micro-batch accumulation must run
    forward -> backward per micro-batch, with ``accumulate_grads``).

    With ``input_grad=True`` the backward also returns dL/dx, and a frozen ``theta`` (``requires_grad=False``)
    gets a backward that computes dL/dx alone and leaves ``theta.grad`` untouched.  There is no double backward."""

    @staticmethod
    def forward(ctx, x, theta, eng, save):
        if ctx.needs_input_grad[0] and not eng.input_grad:
            raise RuntimeError("the fused engine does not produce input gradients (dL/dx) unless it is built with "
                               "input_grad=True; use that, backend='torch', or detach the input")
        ctx.eng = eng
        if save:
            eng._generation += 1
        ctx.generation = eng._generation if save else -1
        y = eng._forward(x, save=save)
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        eng = ctx.eng
        if torch.is_grad_enabled():
            raise RuntimeError("the fused engine has no double backward (create_graph=True); use backend='torch'")
        if ctx.generation != eng._generation:
            raise RuntimeError("backward through a fused-engine forward whose saved activations were overwritten by a "
                               "later forward (the engine keeps one set); run forward/backward pairs back to back")
        want_dx, want_dtheta = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        # the engine writes straight into theta.grad's storage (no 2 GB autograd copy)
        dx = eng._backward(x, dy, input_grad=want_dx, theta_grad=want_dtheta)
        if dx is not None:
            dx = dx.view(x.shape).to(x.dtype)
        return dx, None, None, None


class FusedDistributedFNO(nn.Module):
    """Drop-in ``DistributedFNO`` on the fused sm_90a engine.  Same constructor; the forward
    takes this rank's ``[B, C_in, X, Y_local, Z, T_in]`` shard (fp32 or bf16, CUDA) and returns
    ``[B, out_channels, X, Y_local, Z, T_out]`` in fp32.

    ``input_grad=True``: an input that requires grad gets dL/dx (in its own dtype and shape) from the backward, for
    surrogate inversion and sensitivity studies.  With ``theta.requires_grad_(False)`` that backward computes dL/dx
    only and leaves ``theta.grad`` as it was.  Without it (the default) such an input is refused."""

    def __init__(self, P_x: Partition, in_shape: Sequence[int], out_timesteps: int, width: int,
                 modes: Sequence[int], num_blocks: int = 4, device=torch.device("cuda"),
                 dtype=torch.bfloat16, plan: Optional[str] = None, backend: str = "fused",
                 use_p2p: Optional[bool] = None, init_seed: Optional[int] = None, input_grad: bool = False,
                 out_channels: int = 1):
        super().__init__()
        self.input_grad = bool(input_grad)
        ok, why = supports(P_x, in_shape, out_timesteps, width, modes, out_channels=out_channels)
        if not ok:
            raise ValueError(f"fused engine cannot run this configuration: {why}")
        from ..ops import build
        self._C = _LaunchCounter(build.load())   # fails loudly if the extension is missing
        self.P_x = P_x
        self.in_shape = [int(s) for s in in_shape]
        self.out_timesteps, self.width = int(out_timesteps), int(width)
        self.modes = [int(m) for m in modes]
        self.num_blocks = int(num_blocks)
        self.out_channels = int(out_channels)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("the fused engine needs a CUDA device")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.dtype = torch.bfloat16
        self.block_in_shape = [self.in_shape[0], self.width, *self.in_shape[2:-1], self.out_timesteps]
        # 2-D + time problems run as 3-D + time with a singleton x axis (free views at entry / exit)
        _, shape6, modes6, self.five_d = _as_6d(P_x.shape, self.in_shape, self.modes)
        B, Cin, X, Y, Z, Tin = shape6
        # work partition: the y-pencil the engine computes on.  A differently shaped P_x is folded
        # onto it once at the network's entry / exit (see supports()).
        self.P_outer = P_x
        self.P_work, self.R_in, self.R_out = fold_onto_pencil(P_x, self.in_shape, self.out_timesteps, self.out_channels)
        P_x = self.P_work
        pa = P_x.dim - 3                             # the pencil axis of the work partition
        self.world = int(P_x.shape[pa]) if P_x.active else 1
        self.rank = int(P_x.index[pa]) if P_x.active else 0
        self.plan = EnginePlan(B, Cin, Tin, self.width, self.out_timesteps, X, Y, Z, modes6,
                               self.world, self.rank, out_channels=self.out_channels)
        self.plan.finish(self.num_blocks)
        pl = self.plan
        self.dt_comm = 0.0

        # ---- parameters: one flat fp32 buffer
        theta = torch.zeros(pl.n_theta, device=self.device, dtype=torch.float32)
        self.theta = nn.Parameter(theta)
        self._init_parameters(init_seed)

        # ---- operators (bf16, padded) for the forward and the adjoint chain
        self._ops_f64 = pl.operators()
        self.ops = {k: pad_operator(v, device=self.device) for k, v in self._ops_f64.items() if v.shape[0] <= pl.max_n}

        # ---- symmetric buffers + barrier
        from ..runtime.symm import PeerBarrier, SymmetricBuffer
        self.use_p2p = self.world > 1 if use_p2p is None else (use_p2p and self.world > 1)
        grp = P_x.group
        if self.world > 1:
            self.sym_S1 = SymmetricBuffer(pl.n_S1 * 2, grp, self.rank, self.world, self.device.index)
            self.sym_T1 = SymmetricBuffer(pl.n_T1 * 2, grp, self.rank, self.world, self.device.index)
            self.sym_small = SymmetricBuffer(pl.n_small * 4, grp, self.rank, self.world, self.device.index)
        else:
            self.sym_S1 = self.sym_T1 = self.sym_small = None
        self.barrier = PeerBarrier(grp, self.rank, self.world)

        # ---- workspaces
        bf = dict(device=self.device, dtype=torch.bfloat16)
        self.ws = {
            "Z1U": torch.empty(max(pl.n_Z1, pl.n_U), **bf),
            "S1": self.sym_S1.view([pl.n_S1], torch.bfloat16) if self.world > 1 else torch.empty(pl.n_S1, **bf),
            "T1": self.sym_T1.view([pl.n_T1], torch.bfloat16) if self.world > 1 else torch.empty(pl.n_T1, **bf),
            "S2": torch.empty(pl.n_S2, **bf), "S3w": torch.empty(pl.n_S3, **bf),
            "S4": torch.empty(pl.n_S3, **bf), "T2": torch.empty(pl.n_T2, **bf),
        }
        self._saved: Dict[str, torch.Tensor] = {}
        self._train_bufs_ready = False
        self._generation = 0                     # number of saving forwards so far (see _FusedFn)
        # DFNO_STAGED_SCATTER=0|1 overrides the plan's peer layout (A/B runs, the 8-rank layout on fewer GPUs); it is
        # written into the plan so that its memory and cost figures describe the layout that runs
        st = os.environ.get("DFNO_STAGED_SCATTER")
        if st is not None:
            if st not in ("0", "1"):
                raise ValueError(f"DFNO_STAGED_SCATTER must be 0 or 1, got {st!r}")
            pl.staged = st == "1" and self.world > 1
        self.chain_desc = pl.chain(staged=pl.staged)
        # peers write the staging blocks; the consumer-side S1 / T1 become local buffers
        if pl.staged:
            self.ws["S1s"] = self.ws["S1"]
            self.ws["S1"] = torch.empty(pl.n_S1, **bf)
            self.ws["T1s"] = self.ws["T1"]
            self.ws["T1"] = torch.zeros(pl.n_T1, **bf)
        # the first two GEMMs of every chain (z-DFT, t-DFT) + the transpose R2 as ONE kernel that keeps Z1 on the SM
        # (csrc/spectral_in_sm90.cu); None where spectral_in_check refuses the shape (e.g. T > 64), and then G1a + G1b
        # run as two dft_gemm launches
        self.front = self._front_plan()

    @property
    def fused_pw(self) -> bool:
        """The round-2 pointwise dataflow runs (else the round-1 kernels); decided by the plan from the shape."""
        return self.plan.fused_pw

    @property
    def use_tc_bypass(self) -> bool:
        """The round-1 route runs its bypass on the tensor core; decided by the plan from the shape."""
        return self.plan.tc_bypass

    def _front_plan(self) -> Optional[dict]:
        """Destination view of ``spectral_in`` for this plan's S1 layout (direct or staged), or None when the kernel
        does not support the shape (then G1a + G1b run as separate GEMMs)."""
        pl = self.plan
        P, r = max(self.world, 1), self.rank
        X, Y, Yl, mt, kzl = pl.X, pl.Y, pl.Yl, pl.mt, pl.kzl
        if pl.staged:        # S1s[bc, kz', kt, r_src, x, y_loc, ri] on the rank owning kz
            dstr = [Yl * 2, P * X * Yl * 2, mt * P * X * Yl * 2, kzl * mt * P * X * Yl * 2]
            off = r * X * Yl * 2
        else:                # S1[bc, kz', kt, x, y, ri]
            dstr = [Y * 2, X * Y * 2, mt * X * Y * 2, kzl * mt * X * Y * 2]
            off = pl.y_off * 2
        if "G1a" not in self.ops or "G1b" not in self.ops:
            return None
        o1, o2 = self.ops["G1a"], self.ops["G1b"]
        why = self._C.spectral_in_check(o1.shape[0], o1.shape[1], o2.shape[0], o2.shape[1], P, off, dstr,
                                        pl.BC, X, Yl, pl.T, pl.Z, pl.KZ, mt)
        if why:
            return None
        return dict(dstr=dstr, off=off, dst="S1s" if pl.staged else "S1")

    def _front(self, src: torch.Tensor, adj: bool) -> None:
        pl, fr = self.plan, self.front
        if self.world > 1:
            ptrs = self.sym_S1.peer_ptrs()
        else:
            ptrs = [self.ws[fr["dst"]].data_ptr()]
        sfx = "_adj" if adj else ""
        self._C.spectral_in(src, self.ops["G1a" + sfx], self.ops["G1b" + sfx], ptrs, fr["off"], fr["dstr"],
                            pl.BC, pl.X, pl.Yl, pl.T, pl.Z, pl.KZ, pl.mt)

    # ------------------------------------------------------------------ parameters
    def _seg(self, name: str, base: Optional[torch.Tensor] = None) -> torch.Tensor:
        off, shape = self.plan.segments[name]
        base = self.theta.data if base is None else base
        return base[off:off + int(np.prod(shape))].view(shape)

    def _init_parameters(self, seed: Optional[int] = None) -> None:
        """Reference initialisation (reference ``dfno/dfno.py:35-36,114-117,160``): Kaiming-uniform pointwise
        weights, zero biases, ``U[0,1)/C^2`` spectral weights.  With ``seed`` the draw is *partition independent*:
        pointwise weights come from one generator seeded identically on every rank and every retained ``kz`` slab
        of every block from its own generator seeded by its GLOBAL index, so 1, 2, 4 and 8 ranks build the same
        model (``bench.py`` uses this to check an N-rank run against a 1-rank run)."""
        pl = self.plan
        with torch.no_grad():
            gen = None
            if seed is not None:
                gen = torch.Generator(device=self.device)
                gen.manual_seed(int(seed))
            for name, (off, shape) in pl.segments.items():
                t = self._seg(name)
                if name.endswith(".spectral"):
                    if seed is None:
                        t.copy_(torch.rand(shape, device=self.device) / (self.width * self.width))
                    else:
                        k = int(name.split(".")[1])
                        slab = t.view(pl.C, pl.C, pl.kzl, pl.mt * pl.KY * pl.KX, 2)
                        g2 = torch.Generator(device=self.device)
                        for j in range(pl.kzl):
                            g2.manual_seed(int(seed) * 1000003 + k * 4099 + pl.kz_off + j + 1)
                            slab[:, :, j] = torch.rand(pl.C, pl.C, slab.shape[3], 2, device=self.device,
                                                       generator=g2) / (self.width * self.width)
                elif name.endswith(".W"):
                    if seed is None:
                        nn.init.kaiming_uniform_(t, a=math.sqrt(5))
                    else:                                   # kaiming_uniform_(a=sqrt(5)): U(-1/sqrt(fan_in), +)
                        bound = 1.0 / math.sqrt(shape[1])
                        t.copy_((torch.rand(shape, device=self.device, generator=gen) * 2 - 1) * bound)
                else:
                    t.zero_()
            if self.world > 1 and seed is None:   # replicated pointwise weights: everyone takes rank 0's draw
                small = self.theta.data[:pl.n_small]
                dist.broadcast(small, src=self.P_work.world_ranks[0], group=self.P_work.group)

    def named_views(self) -> Dict[str, torch.Tensor]:
        return {name: self._seg(name) for name in self.plan.segments}

    # ------------------------------------------------------------------ buffers
    def _ensure_train_buffers(self) -> None:
        if self._train_bufs_ready:
            return
        pl = self.plan
        bf = dict(device=self.device, dtype=torch.bfloat16)
        nb = self.num_blocks
        # block inputs (+ the last block's output, which the head reads, in the fused pointwise dataflow)
        self._saved["h"] = [torch.empty(pl.n_act, **bf) for _ in range(nb + (1 if pl.fused_pw else 0))]
        self._saved["pre"] = [torch.empty(pl.n_act, **bf) for _ in range(nb)]     # pre-activations
        self._saved["S3"] = [torch.empty(pl.n_S3, **bf) for _ in range(nb)]       # spectra entering the mix
        self.ws["g"] = torch.empty(pl.n_act, **bf)
        if pl.fused_pw:
            self.ws["amax"] = torch.zeros(1, device=self.device, dtype=torch.int32)
        else:
            self._saved["hcl"] = torch.zeros(pl.npos, pl.CP, **bf)                # last block out, channels-last
            self.ws["dhb"] = torch.empty(pl.n_act, **bf)
            self.ws["gcl"] = torch.empty(pl.npos, pl.CP, **bf)
        # theta.grad's storage: allocated by the first backward that produces weight gradients (a frozen network
        # used for inversion never needs it)
        self.grad_flat = None
        self.accumulate_grads = False          # True: keep adding into theta.grad across backward calls
        self._train_bufs_ready = True

    def _ensure_eval_buffers(self) -> None:
        if "eval_h" in self.ws:
            return
        pl = self.plan
        bf = dict(device=self.device, dtype=torch.bfloat16)
        self.ws["eval_h"] = [torch.empty(pl.n_act, **bf) for _ in range(2)]
        if not pl.fused_pw:
            self.ws["eval_pre"] = torch.empty(pl.n_act, **bf)
            if "hcl" not in self._saved:
                self._saved["hcl"] = torch.zeros(pl.npos, pl.CP, **bf)

    # ------------------------------------------------------------------ kernels
    def _operator(self, name: str, j0: int, n: int) -> torch.Tensor:
        """Padded bf16 operator rows ``[2*j0, 2*(j0+n))`` (the whole operator for single-part stages)."""
        full = self._ops_f64[name]
        if j0 == 0 and 2 * n == full.shape[0]:
            return self.ops[name]
        key = (name, j0, n)
        if key not in self.ops:
            self.ops[key] = pad_operator(full[2 * j0:2 * (j0 + n)], device=self.device)
        return self.ops[key]

    def _gemm(self, st: dict, bufs: Dict[str, torch.Tensor], adj: bool, add: Optional[torch.Tensor] = None) -> None:
        name = st["op"] + ("_adj" if adj else "")
        A, dst = bufs[st["src"]], bufs[st["dst"]]
        if "scatter" in st:
            if st.get("peer_dst") and self.world > 1:
                sym = self.sym_S1 if st["dst"] in ("S1", "S1s") else self.sym_T1
                ptrs = sym.peer_ptrs()
            else:
                ptrs = [dst.data_ptr()] * max(self.world, 1)
            for j0, n, spec, p0, pn in self.plan.parts(st):
                self._C.dft_gemm(A, st["M"], st["K"], st["lda"], self._operator(name, j0, n), 2 * n, spec.epi(),
                                 ptrs if pn is None else ptrs[p0:p0 + pn], None, 0, 0)
        else:
            epi = [0, 0, st["ldc"], 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1, 0]
            self._C.dft_gemm(A, st["M"], st["K"], st["lda"], self.ops[name], st["N"], epi, [dst.data_ptr()], add,
                             st["ldc"] if add is not None else 0, 0)
        if st.get("barrier_after"):
            self.barrier()

    def _spectral_chain(self, src, dst, block: int, adj: bool, add=None, fuse: Optional[dict] = None,
                        grad: Optional[torch.Tensor] = None) -> None:
        """src (engine layout) -> truncated spectrum -> channel mix -> dst (engine layout).

        ``fuse`` (round-2 dataflow): the last stage becomes ``spectral_out`` -- inverse z-DFT + bypass conv of
        ``fuse["h"]`` with ``fuse["W"]`` (transposed in the adjoint chain) (+ GELU, pre-activation kept in
        ``fuse["pre"]``) -- instead of a plain row-major GEMM.  ``grad`` (adjoint chain): the flat gradient buffer
        whose spectral segment the mix backward writes; ``None`` runs the dx-only mix backward (frozen weights)."""
        pl = self.plan
        ws = self.ws
        s3 = self._saved["S3"][block] if (self._train_bufs_ready and not self._eval_mode) else ws["S3w"]
        bufs = {"src": src, "Z1": ws["Z1U"], "S1": ws["S1"], "S2": ws["S2"],
                "S3": ws["S3w"] if adj else s3, "S4": ws["S4"], "T2": ws["T2"], "T1": ws["T1"],
                "U": ws["Z1U"], "dst": dst, "S1s": ws.get("S1s"), "T1s": ws.get("T1s")}
        R = self._seg(f"blocks.{block}.spectral")
        for st in self.chain_desc:
            if self.front is not None and st["name"] in ("G1a", "G1b"):
                if st["name"] == "G1a":
                    self._front(bufs["src"], adj)
                elif st.get("barrier_after"):
                    self.barrier()
            elif st["name"].startswith("perm"):
                self._C.permute_u32(bufs[st["src"]], bufs[st["dst"]], st["size"], st["sstr"], st["dstr"])
            elif st["name"] == "mix":
                if adj:
                    gR = None if grad is None else self._seg(f"blocks.{block}.spectral", grad)
                    self._C.spectral_mix_bwd(s3, R, bufs["S3"], bufs["S4"], gR, getattr(self, "_acc", False), pl.B, pl.C, pl.Q)
                else:
                    self._C.spectral_mix_fwd(bufs["S3"], R, bufs["S4"], pl.B, pl.C, pl.Q)
            elif fuse is not None and st["name"] == "iG1a":
                self._C.spectral_out(bufs[st["src"]], fuse["h"], self.ops[st["op"] + ("_adj" if adj else "")],
                                     fuse["W"], adj, fuse.get("pre"), dst, pl.B, pl.C, pl.X * pl.Yl * pl.T, pl.Z,
                                     st["K"], not adj, fuse.get("pre") is not None)
            else:
                self._gemm(st, bufs, adj, add if st["name"] == "iG1a" else None)

    # ------------------------------------------------------------------ projection head
    def _head_operators(self):
        pl = self.plan
        W3 = self._seg("linear3.W")                                   # [H, C] fp32
        w3 = torch.zeros(pl.H, 64, device=self.device, dtype=torch.bfloat16)
        w3[:, :pl.C] = W3.to(torch.bfloat16)
        w3t = torch.zeros(32, pl.H, device=self.device, dtype=torch.bfloat16)
        w3t[:pl.C] = W3.t().to(torch.bfloat16)
        return w3, w3t

    def _head_operators_cm(self):
        """Operands of the channel-major head kernels: ``W3aug`` bf16 [H, 64] ([H, 128] at width 64) with column
        C = b3 (the hidden bias rides through the MMA against the tile's row of ones) and ``W3^T`` as fp16
        [ceil16(C+1), H]."""
        pl = self.plan
        W3, b3 = self._seg("linear3.W"), self._seg("linear3.b")
        # b3 in column C: one 64-column swizzle block up to width 63, two at width 64
        w3a = torch.zeros(pl.H, 64 if pl.C + 1 <= 64 else 128, device=self.device, dtype=torch.bfloat16)
        w3a[:, :pl.C] = W3.to(torch.bfloat16)
        w3a[:, pl.C] = b3.to(torch.bfloat16)
        w3t = torch.zeros((pl.C + 1 + 15) // 16 * 16, pl.H, device=self.device, dtype=torch.float16)
        w3t[:pl.C] = W3.t().to(torch.bfloat16).to(torch.float16)
        return w3a, w3t

    def _wpad(self, W: torch.Tensor) -> torch.Tensor:
        """[C, C] fp32 -> zero-padded bf16 [32, 64] wgmma operand (rows = output index)."""
        out = torch.zeros(32, 64, device=self.device, dtype=torch.bfloat16)
        out[:W.shape[0], :W.shape[1]] = W.to(torch.bfloat16)
        return out

    def _w4b4(self) -> torch.Tensor:
        """``[W4 (O x H), b4 (O)]`` -- adjacent in the flat parameter buffer by construction."""
        pl = self.plan
        off, _ = pl.segments["linear4.W"]
        assert pl.segments["linear4.b"][0] == off + pl.O * pl.H
        return self.theta.data[off:off + pl.O * (pl.H + 1)]

    def _head_row_digits(self):
        """Row (b, x, y, t, z) of the engine layout -> element offset in the public
        ``[B, O, X, Y, Z, T]`` output: digits innermost first.  With several output channels the batch index is its
        own digit (stride O*S) and channel o sits at + o*S (the plane stride)."""
        pl = self.plan
        if pl.O == 1:
            return [pl.Z, pl.T, pl.B * pl.X * pl.Yl], [pl.T, 1, pl.Z * pl.T]
        return [pl.Z, pl.T, pl.X * pl.Yl, pl.B], [pl.T, 1, pl.Z * pl.T, pl.O * pl.S]

    def _head_forward(self, hcl: torch.Tensor) -> torch.Tensor:
        """linear3 -> gelu -> linear4 in the epilogue of one wgmma GEMM (EPI_HEAD)."""
        pl = self.plan
        w3, _ = self._head_operators()
        out = torch.empty(pl.B, 1, pl.X, pl.Yl, pl.Z, pl.T, device=self.device, dtype=torch.float32)
        R, SR = self._head_row_digits()
        epi = [2, 1, 0, 3, *R, 1, *SR, 0, 1, 1, 0, 0, 0, 0, 1, 0]
        self._C.dft_gemm(hcl, pl.npos, pl.C, pl.CP, w3, pl.H, epi, [out.data_ptr()], None, 0, 0,
                         self._seg("linear3.b"), self._w4b4(), 0.0)
        return out

    def _head_backward(self, hcl: torch.Tensor, dy: torch.Tensor, gcl: torch.Tensor, g: torch.Tensor) -> None:
        pl = self.plan
        w3, w3t = self._head_operators()
        R, SR = self._head_row_digits()
        self._C.head_bwd(hcl, pl.npos, pl.C, pl.CP, w3, w3t, self._seg("linear3.b"),
                         self._seg("linear4.W").view(-1), dy, R, SR, gcl,
                         self._seg("linear3.W", g), self._seg("linear3.b", g),
                         self._seg("linear4.W", g).view(-1), self._seg("linear4.b", g))

    # ------------------------------------------------------------------ forward / backward
    _eval_mode = False

    def _lift_dims(self) -> List[int]:
        pl = self.plan
        return [pl.B, pl.Cin, pl.Tin, pl.C, pl.T, pl.X, pl.Yl, pl.Z]

    def _forward(self, x: torch.Tensor, save: bool) -> torch.Tensor:
        pl, C_ = self.plan, self._C
        x = x.contiguous()
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.float()
        expect = (pl.B, pl.Cin, pl.X, pl.Yl, pl.Z, pl.Tin)
        if self.five_d and x.dim() == 5:
            x = x.unsqueeze(2)
        if tuple(x.shape) != expect:
            raise ValueError(f"expected local input {expect[:2] + expect[3:] if self.five_d else expect}, "
                             f"got {tuple(x.shape)}")
        self._eval_mode = not save
        nb = self.num_blocks
        if save:
            self._ensure_train_buffers()
            hs, pres = self._saved["h"], self._saved["pre"]
        else:
            self._ensure_eval_buffers()
            hs = [self.ws["eval_h"][k % 2] for k in range(nb + 1)]
            pres = [self.ws.get("eval_pre")] * nb
        with _nvtx("dfno.lift"):
            C_.lift_fwd(x, self._seg("linear1.W"), self._seg("linear1.b"), self._seg("linear2.W"),
                        self._seg("linear2.b"), hs[0], self._lift_dims())
        if pl.fused_pw:
            for k in range(nb):
                with _nvtx(f"dfno.block{k}"):
                    self._spectral_chain(hs[k], hs[k + 1], k, adj=False,
                                         fuse=dict(h=hs[k], W=self._seg(f"blocks.{k}.linear.W"),
                                                   pre=pres[k] if save else None))
            with _nvtx("dfno.head"):
                w3a, _ = self._head_operators_cm()
                out = torch.empty(pl.B, pl.O, pl.X, pl.Yl, pl.Z, pl.T, device=self.device, dtype=torch.float32)
                R, SR = self._head_row_digits()
                if pl.O == 1:
                    C_.head_fwd(hs[nb], w3a, self._w4b4(), out, pl.B, pl.C, pl.S, R, SR)
                else:
                    C_.head_fwd_multi(hs[nb], w3a, self._w4b4(), out, pl.B, pl.C, pl.S, pl.O, pl.S, R, SR)
                return out.squeeze(2) if self.five_d else out
        hcl = self._saved["hcl"]
        for k in range(nb):
            last = k == nb - 1
            with _nvtx(f"dfno.block{k}.spectral"):
                self._spectral_chain(hs[k], pres[k], k, adj=False)
            Wb = self._seg(f"blocks.{k}.linear.W")
            with _nvtx(f"dfno.block{k}.bypass_gelu"):
                if pl.tc_bypass:
                    C_.bypass_fwd_tc(hs[k], pres[k], self._wpad(Wb), None if last else hs[k + 1],
                                     hcl if last else None, pl.CP, pl.B, pl.C, pl.S, save)
                else:
                    C_.bypass_gelu_fwd(hs[k], pres[k], Wb, None if last else hs[k + 1], hcl if last else None,
                                       pl.CP, pl.B, pl.C, pl.S, save)
        with _nvtx("dfno.head"):
            out = self._head_forward(hcl)
            return out.squeeze(2) if self.five_d else out

    def _backward(self, x: torch.Tensor, dy: torch.Tensor, input_grad: bool = False,
                  theta_grad: bool = True) -> Optional[torch.Tensor]:
        """Backward of the last saving forward.  ``theta_grad``: the weight gradients go to ``grad_flat``, which
        becomes ``theta.grad``.  Otherwise (frozen weights) ``theta.grad`` is left as it was: the spectral-weight
        gradients are not formed and the small segment's kernels accumulate into a scratch buffer.  ``input_grad``:
        returns dL/dx as fp32 in the engine's local 6-D input shape (else ``None``)."""
        pl, C_ = self.plan, self._C
        x = x.contiguous()
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.float()
        if self.five_d and x.dim() == 5:
            x, dy = x.unsqueeze(2), dy.unsqueeze(2)
        self._eval_mode = False
        hs, pres = self._saved["h"], self._saved["pre"]
        g = self.ws["g"]
        if theta_grad:
            if self.grad_flat is None:
                self.grad_flat = torch.zeros(pl.n_theta, device=self.device, dtype=torch.float32)
            if not (self.accumulate_grads and self.theta.grad is self.grad_flat):
                # spectral gradients are overwritten by the mix backward; only the small,
                # atomically accumulated segment needs clearing
                self.grad_flat[:pl.n_small].zero_()
            self._acc = bool(self.accumulate_grads and self.theta.grad is self.grad_flat)
            gf = gR = self.grad_flat
        else:
            if "g_small" not in self.ws:
                self.ws["g_small"] = torch.empty(pl.n_small, device=self.device, dtype=torch.float32)
            gf, gR = self.ws["g_small"], None
            gf.zero_()
        if pl.fused_pw:
            nb = self.num_blocks
            with _nvtx("dfno.head.bwd"):
                w3a, w3t = self._head_operators_cm()
                R, SR = self._head_row_digits()
                head_grads = (self._seg("linear3.W", gf), self._seg("linear3.b", gf),
                              self._seg("linear4.W", gf).view(-1), self._seg("linear4.b", gf))
                if pl.O == 1:
                    C_.head_bwd2(hs[nb], w3a, w3t, self._seg("linear4.W").view(-1), dy.contiguous().float(),
                                 self.ws["amax"], g, *head_grads, pl.B, pl.C, pl.S, R, SR)
                else:
                    C_.head_bwd_multi(hs[nb], w3a, w3t, self._seg("linear4.W").view(-1), dy.contiguous().float(),
                                      self.ws["amax"], g, *head_grads, pl.B, pl.C, pl.S, pl.O, pl.S, R, SR)
            L = pl.X * pl.Yl * pl.T
            for k in reversed(range(nb)):
                with _nvtx(f"dfno.block{k}.bwd"):
                    # dpre over pre (packed fp16 GELU'), bypass weight gradient reduced on the tensor core
                    C_.dpre_dw(g, pres[k], hs[k], self._seg(f"blocks.{k}.linear.W", gf), pl.B, pl.C, L, pl.Z)
                    # adjoint chain; its last GEMM adds W^T dpre (the bypass input gradient) in the same accumulator
                    self._spectral_chain(pres[k], g, k, adj=True,
                                         fuse=dict(h=pres[k], W=self._seg(f"blocks.{k}.linear.W")), grad=gR)
        else:
            hcl, dhb, gcl = self._saved["hcl"], self.ws["dhb"], self.ws["gcl"]
            with _nvtx("dfno.head.bwd"):
                self._head_backward(hcl, dy.contiguous().float(), gcl, gf)
            for k in reversed(range(self.num_blocks)):
                last = k == self.num_blocks - 1
                Wb = self._seg(f"blocks.{k}.linear.W")
                gW = self._seg(f"blocks.{k}.linear.W", gf)
                if pl.tc_bypass:
                    # one wgmma kernel: dpre (over pre), dhb = W^T dpre, dW accumulated in registers
                    C_.bypass_bwd_tc(None if last else g, gcl if last else None, pl.CP, pres[k], hs[k],
                                     self._wpad(Wb.t()), dhb, gW, pl.B, pl.C, pl.S)
                else:
                    # dpre overwrites pre (same thread reads then writes each element)
                    C_.bypass_gelu_bwd(None if last else g, gcl if last else None, pl.CP, pres[k], Wb, pres[k], dhb,
                                       pl.B, pl.C, pl.S)
                    if theta_grad:          # this GEMM only forms the bypass weight gradient
                        for b in range(pl.B):
                            sl = slice(b * pl.C * pl.S, (b + 1) * pl.C * pl.S)
                            C_.kreduce_gemm(pres[k][sl], pl.S, pl.C, hs[k][sl], pl.S, pl.C, pl.S, gW)
                with _nvtx(f"dfno.block{k}.spectral.bwd"):
                    self._spectral_chain(pres[k], g, k, adj=True, add=dhb, grad=gR)
        # lift: fp32 dx in x's (local, 6-D) layout, written whole by the kernel -- no memset
        dx = torch.empty(x.shape, device=self.device, dtype=torch.float32) if input_grad else None
        C_.lift_bwd(x, self._seg("linear1.W"), self._seg("linear1.b"), self._seg("linear2.W"),
                    self._seg("linear2.b"), g, self._seg("linear1.W", gf), self._seg("linear1.b", gf),
                    self._seg("linear2.W", gf), self._seg("linear2.b", gf), self._lift_dims(), dx)
        # the same reduction on every rank either way, so ranks that disagree about theta.requires_grad still pair
        # up their peer barriers
        self._sync_small_grads(gf[:pl.n_small])
        if theta_grad:
            self.theta.grad = self.grad_flat
        return dx

    def _sync_small_grads(self, small: torch.Tensor) -> None:
        """Sum the replicated pointwise-weight gradients over the pencil (the SumReduce side
        of the reference's BroadcastedLinear, once per step instead of per layer)."""
        if self.world <= 1:
            return
        if self.use_p2p:
            self.allreduce_small_(small)
        else:
            dist.all_reduce(small, group=self.P_work.group)

    def allreduce_small_(self, t: torch.Tensor) -> torch.Tensor:
        """In-place sum of a small contiguous fp32 vector over the pencil through peer memory
        (no NCCL; CUDA-graph capturable).  Every rank gets the bitwise identical result."""
        if self.world <= 1:
            return t
        n = t.numel()
        if n > self.plan.n_small or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("allreduce_small_ takes a contiguous fp32 vector no longer than the pointwise segment")
        stage = self.sym_small.view([n], torch.float32)
        self.barrier()                           # previous readers are done with the staging buffer
        stage.copy_(t.view(-1))
        self.barrier()                           # every rank's contribution is visible
        self._C.p2p_allreduce_small(self.sym_small.peer_ptrs(), t.view(-1), n, self.rank)
        return t

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.R_in is not None:
            x = self.R_in(x.contiguous())
        save = bool(torch.is_grad_enabled() and (self.theta.requires_grad or (self.input_grad and x.requires_grad)))
        y = _FusedFn.apply(x, self.theta, self, save)
        if self.R_out is not None:
            y = self.R_out(y)
        return y

    # ------------------------------------------------------------------ canonical state <-> engine
    def engine_meta(self) -> Dict[str, object]:
        """What is needed to interpret this rank's flat ``theta`` outside the module (stored next to per-rank
        checkpoints so that fused checkpoints can be assembled / re-sharded offline)."""
        pl = self.plan
        return {"format": "fused-theta", "segments": dict(pl.segments), "C": pl.C, "kzl": pl.kzl, "kz_off": pl.kz_off,
                "mt": pl.mt, "KX": pl.KX, "KY": pl.KY, "KZ": pl.KZ, "rank": self.rank, "world": self.world,
                "num_blocks": self.num_blocks, "ndim": len(self.in_shape), "out_channels": pl.O}

    @staticmethod
    def theta_to_canonical(theta: torch.Tensor, meta: Dict[str, object], include_pointwise: bool = True):
        """This rank's part of the canonical state from a flat ``theta`` (CPU tensor) and its :meth:`engine_meta`:
        ``{name: tensor}`` for pointwise weights, ``{name: (kz_off, slab)}`` for spectral shards (global layout
        ``[i, o, KX, KY, kzl, mt]``)."""
        out = {}
        C, kzl, mt, KX, KY = (int(meta[k]) for k in ("C", "kzl", "mt", "KX", "KY"))
        for name, (off, shape) in meta["segments"].items():
            t = theta[off:off + int(np.prod(shape))].view(shape).detach().cpu()
            if name.endswith(".spectral"):
                # native [i, o, kzl, mt, KY, KX, 2] -> global slab [i, o, KX, KY, kzl, mt]
                w = torch.view_as_complex(t.reshape(C, C, kzl, mt, KY, KX, 2).contiguous())
                out[name] = (int(meta["kz_off"]), w.permute(0, 1, 5, 4, 2, 3).contiguous())
            elif include_pointwise:
                tt = t
                if name.endswith(".b"):
                    b_shape = [1] * int(meta.get("ndim", 6))
                    b_shape[-1 if name.startswith("linear1") else 1] = t.numel()
                    tt = t.reshape(b_shape)
                out[name] = tt
        return out

    @staticmethod
    def merge_canonical(parts, meta: Dict[str, object]) -> Dict[str, torch.Tensor]:
        """Union of per-rank :meth:`theta_to_canonical` results."""
        C, mt, KX, KY, KZ = (int(meta[k]) for k in ("C", "mt", "KX", "KY", "KZ"))
        out: Dict[str, torch.Tensor] = {}
        for part in parts:
            for k, v in part.items():
                if k.endswith(".spectral"):
                    kz0, w = v
                    if k not in out:
                        out[k] = torch.zeros(C, C, KX, KY, KZ, mt, dtype=torch.complex64)
                    out[k][:, :, :, :, kz0:kz0 + w.shape[4], :] = w
                else:
                    out[k] = v
        nd = int(meta.get("ndim", 6))
        for k in list(out):
            if k.endswith(".spectral") and nd == 5:          # 2-D + time: drop the singleton kx axis
                out[k] = out[k].squeeze(2)
        for k in range(int(meta["num_blocks"])):          # key parity with the portable backend
            out.setdefault(f"blocks.{k}.linear.b", torch.zeros(1, C, *([1] * (nd - 2))))
        return out

    def engine_state_to_global(self, to_all: bool = False):
        """Canonical (partition independent) state on rank 0 / all ranks (CPU tensors)."""
        meta = self.engine_meta()
        mine = self.theta_to_canonical(self.theta.data, meta, include_pointwise=self.rank == 0)
        if self.world > 1:
            gathered = [None] * self.world
            dist.all_gather_object(gathered, mine, group=self.P_work.group)
        else:
            gathered = [mine]
        if not (to_all or self.rank == 0):
            return None
        return self.merge_canonical(gathered, meta)

    def engine_state_from_global(self, state, strict: bool = True) -> None:
        """Load a canonical state.  ``strict``: every engine segment must be present; otherwise missing segments
        keep their values -- but a state that matches NO segment is always an error (it used to load nothing,
        silently)."""
        pl = self.plan
        missing = [n for n in pl.segments if n not in state]
        if missing and (strict or len(missing) == len(pl.segments)):
            raise KeyError(f"canonical state lacks {len(missing)} of {len(pl.segments)} engine segments, e.g. "
                           f"{missing[:3]} (keys present: {sorted(state)[:4]}...)")
        with torch.no_grad():
            for name, (off, shape) in pl.segments.items():
                if name not in state:
                    continue
                src = state[name]
                if name.endswith(".spectral"):
                    if self.five_d and src.dim() == 5:
                        src = src.unsqueeze(2)
                    w = src[:, :, :, :, pl.kz_off:pl.kz_off + pl.kzl, :].to(torch.complex64)
                    w = torch.view_as_real(w.permute(0, 1, 4, 5, 3, 2).contiguous())   # [i,o,kzl,mt,KY,KX,2]
                    self._seg(name).copy_(w.reshape(shape).to(self.device))
                else:
                    if src.numel() != int(np.prod(shape)):
                        raise ValueError(f"canonical state entry {name} has shape {list(src.shape)}, this engine needs "
                                         f"{list(shape)} (out_channels = {pl.O})")
                    self._seg(name).copy_(src.reshape(shape).to(self.device, torch.float32))


# =====================================================================================
# optimizer
# =====================================================================================

class FusedAdam:
    """Adam on the engine's flat parameter buffer with one fused kernel launch per step
    (``csrc/optim.cu``); semantics of ``torch.optim.Adam`` (L2 ``weight_decay``)."""

    def __init__(self, model: FusedDistributedFNO, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0):
        self.model = model
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.m = torch.zeros_like(model.theta.data)
        self.v = torch.zeros_like(model.theta.data)
        self.step_count = 0
        # the step counter also lives on the device so a captured CUDA graph can replay the update
        self.step_dev = torch.zeros(1, device=model.theta.device, dtype=torch.float32)

    def zero_grad(self, set_to_none: bool = True) -> None:
        if set_to_none:
            self.model.theta.grad = None
        elif self.model.theta.grad is not None:
            self.model.theta.grad.zero_()

    def step(self, grad_scale: float = 1.0) -> None:
        g = self.model.theta.grad
        if g is None:
            return
        self.step_count += 1
        self.step_dev += 1.0
        self.model._C.adam_step(self.model.theta.data, g.contiguous(), self.m, self.v, self.lr, self.betas[0],
                                self.betas[1], self.eps, self.weight_decay, self.step_count, grad_scale,
                                self.step_dev)

    def state_dict(self):
        return {"m": self.m, "v": self.v, "step": self.step_count, "lr": self.lr, "betas": self.betas,
                "eps": self.eps, "weight_decay": self.weight_decay}

    def load_state_dict(self, sd) -> None:
        self.m.copy_(sd["m"]); self.v.copy_(sd["v"])
        self.step_count = int(sd["step"])
        self.step_dev.fill_(float(self.step_count))
        self.lr, self.betas, self.eps, self.weight_decay = sd["lr"], tuple(sd["betas"]), sd["eps"], sd["weight_decay"]
