"""Pencil planner for the distributed truncated N-D FFT of one Fourier layer.

Given the activation partition ``P_x`` (grid over ``[batch, channel, *spatial, time]``) the
transform is done in two local stages separated by global re-shards:

    P_x --R1--> P_m : last ``n1`` axes local    -> (r)FFT + truncate those axes
    P_m --R2--> P_y : first ``n0`` axes local   -> FFT + truncate those axes, spectral mix
    P_y --R3--> P_m --R4--> P_x on the way back.

``plan="reference"`` reproduces the worker-grid arithmetic of
reference ``dfno/dfno.py:82-97`` exactly (needed for checkpoint-layout parity; note
its quirk for an odd number of transformed axes, SURVEY.md §5.7 item 5: ranks are left
idle in stage y).  ``plan="balanced"`` is this framework's own choice for stage y: all
workers are spread over the *retained-mode* extents of the stage-m axes so that no rank
idles and the spectral-weight shards are as even as the mode counts allow.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np


__all__ = ["PencilPlan", "make_pencil_plan", "spectrum_shape", "corner_boxes", "validate_modes"]


@dataclass(frozen=True)
class PencilPlan:
    grid_x: Tuple[int, ...]
    grid_m: Tuple[int, ...]
    grid_y: Tuple[int, ...]
    dim_m: Tuple[int, ...]     # tensor axes transformed in stage m (last one is the rfft axis)
    dim_y: Tuple[int, ...]     # tensor axes transformed in stage y
    kind: str = "reference"

    @property
    def rfft_dim(self) -> int:
        return self.dim_m[-1]


def make_pencil_plan(grid_x: Sequence[int], kind: str = "reference",
                     spectrum: Sequence[int] = None) -> PencilPlan:
    g = np.asarray([int(v) for v in grid_x], dtype=np.int64)
    nd = len(g)
    n = nd - 2
    if n < 1:
        raise ValueError("need at least one transformed axis")
    n0, n1 = (n + 1) // 2, n // 2
    gm, gy = g.copy(), g.copy()
    gm[2 + n0:] = 1
    gm[2:2 + n1] *= g[2 + n0:]
    gy[2:2 + n0] = 1
    gy[2 + n0:] *= g[2:2 + n1]
    dim_m = tuple(range(2 + n0, nd))
    dim_y = tuple(range(2, 2 + n0))
    if kind == "balanced":
        # spread *all* workers over the stage-m axes' retained modes, largest extent first
        if spectrum is None:
            raise ValueError("balanced plan needs the truncated spectrum shape")
        workers = int(np.prod(g[2:]))
        gy = np.ones(nd, dtype=np.int64)
        gy[:2] = g[:2]
        if n1 == 0:
            # 1 transformed axis: stage y owns it all; nothing to spread over
            gy = gm.copy()
        else:
            rem = workers
            order = sorted(dim_m, key=lambda d: -int(spectrum[d]))
            for d in order:
                # largest divisor of rem that does not exceed the retained extent
                f = max(k for k in range(1, rem + 1) if rem % k == 0 and k <= int(spectrum[d]))
                gy[d] = f
                rem //= f
            if rem != 1:
                raise ValueError(f"cannot place {workers} workers on spectrum {tuple(spectrum)}")
    elif kind != "reference":
        raise ValueError(f"unknown plan kind {kind!r}")
    return PencilPlan(tuple(int(v) for v in g), tuple(int(v) for v in gm),
                      tuple(int(v) for v in gy), dim_m, dim_y, kind)


def validate_modes(shape: Sequence[int], modes: Sequence[int]) -> None:
    """Reject mode counts for which the truncated spectrum is ill-defined (the reference
    silently mis-shapes: SURVEY.md §2.6 footnote 1)."""
    n = len(shape) - 2
    if len(modes) != n:
        raise ValueError(f"need {n} mode counts, got {len(modes)}")
    for ax in range(n - 1):
        if 2 * modes[ax] > shape[2 + ax]:
            raise ValueError(f"modes[{ax}]={modes[ax]} needs an axis of length >= {2*modes[ax]}, "
                             f"got {shape[2+ax]}")
    if modes[-1] > shape[-1] // 2 + 1:
        raise ValueError(f"modes[-1]={modes[-1]} exceeds rfft bins {shape[-1]//2+1}")
    # T = 1 (a steady problem, or next-step prediction): the single rfft bin is real-valued input, irfft(n=1) takes the
    # real part of it back, so the block is the spatial spectral convolution with the real part taken at the end
    if shape[-1] % 2 and shape[-1] != 1:
        raise ValueError("the last (time) axis must have length 1 or even length (irfft round trip)")


def spectrum_shape(block_shape: Sequence[int], modes: Sequence[int]) -> List[int]:
    """Global truncated spectrum ``[B, C, 2m_1, .., 2m_{n-1}, m_n]``."""
    out = list(int(s) for s in block_shape)
    n = len(out) - 2
    for ax in range(n - 1):
        out[2 + ax] = 2 * int(modes[ax])
    out[-1] = int(modes[-1])
    return out


def corner_boxes(spec_shape: Sequence[int], modes: Sequence[int], start: Sequence[int],
                 stop: Sequence[int]) -> List[List[Tuple[int, int]]]:
    """Low/high-mode "corners" of the truncated spectrum intersected with a local slab.

    Returns, in binary-counter order over the non-rfft transformed axes (the first
    transformed axis is the least significant digit; 0 = low modes ``[0,m)``, 1 = high modes ``[size-m,size)``), the
    non-empty intersections as per-axis ``(a, b)`` *local* bounds for axes ``2..``.  This
    is the enumeration that fixes the ``weights.{j}`` checkpoint keys
    (reference ``dfno/dfno.py:137-161``).
    """
    nd = len(spec_shape)
    n = nd - 2
    out = []
    for rev in itertools.product((0, 1), repeat=n - 1):
        digits = rev[::-1]          # first transformed axis toggles fastest (LSB)
        box = []
        for ax in range(n):
            d = 2 + ax
            m, size = int(modes[ax]), int(spec_shape[d])
            hi = ax < n - 1 and digits[ax] == 1
            lo_g, hi_g = (size - m, size) if hi else (0, m)
            a, b = max(lo_g, int(start[d])), min(hi_g, int(stop[d]))
            box.append((a - int(start[d]), b - int(start[d])))
        if all(b > a for a, b in box):
            out.append(box)
    return out
