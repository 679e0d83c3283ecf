"""Python front end of the resident-operator wgmma GEMM (``csrc/dft_gemm_sm90.cu``)."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from . import build

__all__ = ["pad_operator", "dft_gemm_min_smem", "dft_gemm_fits", "gemm_rowmajor", "gemm_scatter", "ScatterSpec"]

EPI_ROWMAJOR, EPI_PAIR_SCATTER = 0, 1
PEER_NONE, PEER_BY_ROW, PEER_BY_COL = 0, 1, 2


def _ceil(a: int, b: int) -> int:
    return (a + b - 1) // b * b


def pad_operator(B: torch.Tensor, device=None) -> torch.Tensor:
    """``[N, K]`` real operator -> zero-padded bf16 ``[ceil16(N), ceil64(K)]``."""
    N, K = B.shape
    out = torch.zeros(_ceil(N, 16), _ceil(K, 64), dtype=torch.bfloat16, device=device or B.device)
    out[:N, :K] = B.to(device=out.device, dtype=torch.bfloat16)
    return out


# Shared-memory sizing of dft_gemm_launch (csrc/dft_gemm_sm90.cu); keep the two in step.  The padded operator stays
# resident next to 5 KB of barriers, tables and alignment slack and a ring of at least two A stages of one 64-wide
# K block each (64 rows when n_pad > 128, else 128).  The formula also counts 8.5 KB of per-warp row scratch that the
# kernel no longer uses (its epilogues work on the accumulator fragments), so every shape admitted here launches with
# room to spare; the smallest configuration the launcher tries is the one above.
DFT_GEMM_SMEM = 227 * 1024


def dft_gemm_min_smem(rows: int, cols: int) -> int:
    """Fewest bytes of shared memory ``dft_gemm`` needs with a resident ``[rows, cols]`` operator."""
    n_pad, k_pad = _ceil(rows, 16), _ceil(cols, 64)
    tile_m = 64 if n_pad > 128 else 128
    return n_pad * k_pad * 2 + 4096 + 1024 + 4 * 32 * 17 * 4 + 2 * tile_m * 64 * 2


def dft_gemm_fits(rows: int, cols: int) -> bool:
    """Can ``dft_gemm`` keep a ``[rows, cols]`` operator resident (padded to ``[ceil16(rows), ceil64(cols)]``)?"""
    return (_ceil(rows, 16) <= 256 and _ceil(cols, 64) <= 512
            and dft_gemm_min_smem(rows, cols) <= DFT_GEMM_SMEM)


def gemm_rowmajor(A: torch.Tensor, M: int, K: int, lda: int, Bpad: torch.Tensor, N: int,
                  out: torch.Tensor, ldc: int, add: Optional[torch.Tensor] = None, ld_add: int = 0,
                  max_ctas: int = 0) -> torch.Tensor:
    """``out[m, :N] = A[m, :K] @ B[:N, :K]^T (+ add[m, :N])``; ``out`` is bf16 or fp32."""
    epi = [EPI_ROWMAJOR, 1 if out.dtype == torch.float32 else 0, ldc, 0,
           0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, PEER_NONE, 0, 1, 0]
    build.load().dft_gemm(A, M, K, lda, Bpad, N, epi, [out.data_ptr()], add, ld_add, max_ctas)
    return out


class ScatterSpec:
    """Mixed-radix description of where the epilogue puts complex pair ``j`` of row ``r``.

    ``rows``: up to 4 ``(radix, stride)`` digits of the row index, innermost first (the last
    radix is ignored).  ``cols``: ``(J0, SJ0, SJ1)``: pair ``j`` -> ``(j % J0)*SJ0 + (j // J0)*SJ1``.
    ``peer``: ``None`` or ``("row", level, div)`` / ``("col", div)``: that digit selects the
    destination buffer ``peers[digit // div]`` and ``digit % div`` is used for addressing.
    Strides are in bf16 elements.
    """

    def __init__(self, rows: Sequence[Tuple[int, int]], cols: Tuple[int, int, int],
                 peer=None, base_off: int = 0):
        assert 1 <= len(rows) <= 4
        self.rows, self.cols, self.peer, self.base_off = list(rows), cols, peer, base_off

    def epi(self) -> List[int]:
        R = [r for r, _ in self.rows] + [1] * (4 - len(self.rows))
        SR = [s for _, s in self.rows] + [0] * (4 - len(self.rows))
        sel, lvl, div = PEER_NONE, 0, 1
        if self.peer is not None:
            if self.peer[0] == "row":
                sel, lvl, div = PEER_BY_ROW, self.peer[1], self.peer[2]
            else:
                sel, div = PEER_BY_COL, self.peer[1]
        J0, SJ0, SJ1 = self.cols
        return [EPI_PAIR_SCATTER, 0, 0, len(self.rows), *R, *SR, J0, 1, SJ0, SJ1, sel, lvl, div,
                self.base_off]

    def column_part(self, j0: int, n: int) -> Tuple["ScatterSpec", int, Optional[int]]:
        """The same scatter restricted to pairs ``[j0, j0+n)`` as a stand-alone launch (stages whose
        N exceeds one resident operator are issued as several column parts).  Returns
        ``(spec, first_peer, n_peers)``: the part's pair ``j`` lands where pair ``j0+j`` of the full
        spec does, with the peer table sliced to ``peers[first_peer : first_peer+n_peers]``
        (``n_peers=None``: unchanged table)."""
        J0, SJ0, SJ1 = self.cols
        if self.peer is not None and self.peer[0] == "col":
            div = self.peer[1]
            if j0 % div == 0 and n % div == 0:                       # whole peers
                return ScatterSpec(self.rows, self.cols, self.peer, self.base_off), j0 // div, n // div
            if div % n == 0 and j0 % n == 0 and J0 % n == 0:         # inside one peer's columns
                jj = j0 % div
                off = self.base_off + (jj % J0) * SJ0 + (jj // J0) * SJ1
                return ScatterSpec(self.rows, (n, SJ0, 0), None, off), j0 // div, 1
            raise ValueError(f"cannot split {n} pairs at {j0} over peer columns of {div}")
        if J0 % n == 0 and j0 % n == 0:
            off = self.base_off + (j0 % J0) * SJ0 + (j0 // J0) * SJ1
            return ScatterSpec(self.rows, (n, SJ0, 0), self.peer, off), 0, None
        if n % J0 == 0 and j0 % J0 == 0:
            return ScatterSpec(self.rows, self.cols, self.peer, self.base_off + (j0 // J0) * SJ1), 0, None
        raise ValueError(f"cannot split {n} pairs at {j0} with column radix {J0}")

    # pure-python model of the addressing, used by the tests and for planning checks
    def address(self, row: int, j: int) -> Tuple[int, int]:
        off, peer, r = self.base_off, 0, row
        for l, (radix, stride) in enumerate(self.rows):
            d = r if l == len(self.rows) - 1 else r % radix
            r = r // radix if l < len(self.rows) - 1 else 0
            if self.peer is not None and self.peer[0] == "row" and self.peer[1] == l:
                peer, d = d // self.peer[2], d % self.peer[2]
            off += d * stride
        if self.peer is not None and self.peer[0] == "col":
            peer, j = j // self.peer[1], j % self.peer[1]
        J0, SJ0, SJ1 = self.cols
        return peer, off + (j % J0) * SJ0 + (j // J0) * SJ1


def gemm_scatter(A: torch.Tensor, M: int, K: int, lda: int, Bpad: torch.Tensor, N: int,
                 peer_ptrs: Sequence[int], spec: ScatterSpec, max_ctas: int = 0) -> None:
    """Complex-pair scatter epilogue; ``peer_ptrs`` are raw device pointers (bf16 buffers,
    possibly NVLink-mapped memory of other GPUs)."""
    build.load().dft_gemm(A, M, K, lda, Bpad, N, spec.epi(), list(peer_ptrs), None, 0, max_ctas)
