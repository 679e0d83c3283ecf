"""Python front end of the resident-operator wgmma GEMM (``csrc/dft_gemm_sm90.cu``)."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from . import build

__all__ = ["pad_operator", "dft_gemm_min_smem", "dft_gemm_fits", "gemm_rowmajor", "gemm_scatter", "ScatterSpec",
           "BoxSpec"]

EPI_ROWMAJOR, EPI_PAIR_SCATTER, EPI_BOX_STORE = 0, 1, 3
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


class BoxSpec:
    """Box-store epilogue of the inverse y-DFT into ``T1`` (``EPI_BOX_STORE``, ``csrc/dft_gemm_sm90.cu``).

    The rows of A are ``(bcx, kz, kt)``, kt fastest: ``mt`` rows per kz group, ``kzl`` groups per bcx, ``bcx`` = B*C*X
    row blocks.  A tile takes ``G = tile_rows // mt`` whole kz groups of one bcx (rows past them are computed and
    dropped), stages them in shared memory as ``[y][kz][kt (pitch mtp)]`` with zero pad words, and leaves as one TMA
    box per destination buffer.  Pair ``j`` (= y) goes to buffer ``j // ybox`` at ``T1[bcx, y0 + j % ybox, kz, kt]``,
    ``T1`` = that buffer + ``base_off`` bf16 elements with ``[bcx][Yl][KZ][mtp]`` complex pairs; ``ybox = min(n, Yl)``
    for a launch of ``n`` pairs.  Every global run is ``G * mtp`` whole pairs, clipped at ``kzl`` and ``Yl``."""

    def __init__(self, mt: int, mtp: int, kzl: int, KZ: int, Yl: int, bcx: int, base_off: int, y0: int = 0):
        self.mt, self.mtp, self.kzl, self.KZ, self.Yl = mt, mtp, kzl, KZ, Yl
        self.bcx, self.base_off, self.y0 = bcx, base_off, y0

    def epi(self) -> List[int]:
        return [EPI_BOX_STORE] + [0] * 19 + [self.mt, self.mtp, self.kzl, self.KZ, self.Yl, self.y0, self.bcx,
                                             self.base_off]

    def column_part(self, j0: int, n: int) -> Tuple["BoxSpec", int, Optional[int]]:
        """The launch of pairs ``[j0, j0+n)``: ``(spec, first_peer, n_peers)`` as :meth:`ScatterSpec.column_part`
        returns them for the pair scatter of the same stage (whole destinations, or a y range inside one)."""
        Yl = self.Yl
        if j0 % Yl == 0 and n % Yl == 0:
            return BoxSpec(self.mt, self.mtp, self.kzl, self.KZ, Yl, self.bcx, self.base_off), j0 // Yl, n // Yl
        if Yl % n == 0 and j0 % n == 0:
            return (BoxSpec(self.mt, self.mtp, self.kzl, self.KZ, Yl, self.bcx, self.base_off, j0 % Yl), j0 // Yl, 1)
        raise ValueError(f"cannot split {n} pairs at {j0} over destinations of {Yl}")

    @staticmethod
    def tile_rows(n: int) -> int:
        """Rows of one dft_gemm tile for a launch of ``n`` pairs (64 when the operator is wider than 128 rows)."""
        return 64 if _ceil(2 * n, 16) > 128 else 128

    def groups(self, n: int) -> int:
        """kz groups per tile (``G``)."""
        return self.tile_rows(n) // self.mt

    def tiles(self, n: int) -> List[Tuple[int, int]]:
        """``(first row, live rows)`` of every tile, in launch order (the kernel's tile -> row mapping)."""
        G = self.groups(n)
        tpb = -(-self.kzl // G)
        return [((b * self.kzl + c * G) * self.mt, min(G, self.kzl - c * G) * self.mt)
                for b in range(self.bcx) for c in range(tpb)]

    def fits(self, n: int, K: int) -> bool:
        """Can one launch of ``n`` pairs and reduction length ``K`` take the box store?  Mirrors ``box_setup`` and
        the shared-memory sizing of ``dft_gemm_launch``: the resident operator, barriers and tables, and for every
        consumer warpgroup the accumulator allows (2 or 3) a ring of two 64-wide K blocks and one staging tile.  With
        fewer warpgroups a tile's box would have to leave before the next tile's staging starts, so shapes whose
        staging crowds them out (mt = 1 at 128 y: 64 kz groups of 4-word runs per y, 128 KB) keep the pair scatter."""
        G, ybox = self.groups(n), min(n, self.Yl)
        if G < 1 or G * self.mtp > 256 or ybox > 256 or n % ybox or n // ybox > 8 or self.mtp % 4:
            return False
        n_pad, tile = _ceil(2 * n, 16), self.tile_rows(n)
        groups = 3 if (tile // 64) * n_pad // 2 <= 64 else 2
        stg = n // ybox * _ceil(ybox * G * self.mtp * 4, 128)
        return n_pad * _ceil(K, 64) * 2 + 5120 + groups * (stg + 2 * tile * 128) <= DFT_GEMM_SMEM


def gemm_scatter(A: torch.Tensor, M: int, K: int, lda: int, Bpad: torch.Tensor, N: int,
                 peer_ptrs: Sequence[int], spec: ScatterSpec, max_ctas: int = 0) -> None:
    """Complex-pair scatter epilogue; ``peer_ptrs`` are raw device pointers (bf16 buffers,
    possibly NVLink-mapped memory of other GPUs)."""
    build.load().dft_gemm(A, M, K, lda, Bpad, N, spec.epi(), list(peer_ptrs), None, 0, max_ctas)
