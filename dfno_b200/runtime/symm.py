"""Symmetric (peer-mapped) device buffers: the NVLink data plane of the fused engine.

``SymmetricBuffer`` allocates ``nbytes`` on this rank's GPU, exchanges CUDA IPC handles over
the ``torch.distributed`` control plane and maps every peer's allocation, yielding
``ptrs[r]`` = a device pointer *valid on this GPU* to rank ``r``'s buffer.  Kernels store to /
load from those pointers directly (NVSwitch routes the traffic); see ``csrc/symm_mem.cpp``,
``csrc/p2p.cu`` and the peer-scatter epilogue of ``csrc/dft_gemm_sm90.cu``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist

from ..ops import build

__all__ = ["SymmetricBuffer", "PeerBarrier", "P2PAllToAll"]


class SymmetricBuffer:
    def __init__(self, nbytes: int, group=None, rank: int = 0, world: int = 1, device: Optional[int] = None):
        self.nbytes = int((nbytes + 255) // 256 * 256)
        self.group, self.rank, self.world = group, rank, world
        self.device = torch.cuda.current_device() if device is None else device
        C = build.load()
        self._C = C
        self.local_ptr, handle = C.symm_alloc(self.nbytes, self.device)
        self.ptrs: List[int] = [0] * world
        self.ptrs[rank] = self.local_ptr
        self._opened: List[int] = []
        if world > 1:
            handles = [None] * world
            dist.all_gather_object(handles, (rank, bytes(handle)), group=group)
            for r, h in handles:
                if r != rank:
                    p = C.symm_open(h, self.device)
                    self.ptrs[r] = p
                    self._opened.append(p)
            dist.barrier(group=group)

    def view(self, shape: Sequence[int], dtype: torch.dtype, byte_offset: int = 0) -> torch.Tensor:
        """Tensor view of the *local* buffer."""
        return self._C.tensor_from_ptr(self.local_ptr + byte_offset, list(shape), dtype, self.device)

    def peer_ptrs(self, byte_offset: int = 0) -> List[int]:
        return [p + byte_offset for p in self.ptrs]

    def close(self) -> None:
        if getattr(self, "_C", None) is None:
            return
        for p in self._opened:
            self._C.symm_close(p)
        self._opened = []
        if self.local_ptr:
            self._C.symm_free(self.local_ptr)
            self.local_ptr = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PeerBarrier:
    """Device-side flag barrier across the ranks sharing a signal pad (``p2p.cu``)."""

    def __init__(self, group=None, rank: int = 0, world: int = 1, timeout_s: Optional[float] = None):
        import os
        self.rank, self.world = rank, world
        self.epoch = 0
        # bounded spin: a peer that never arrives turns into a CUDA error instead of a hang
        self.timeout_s = float(os.environ.get("DFNO_BARRIER_TIMEOUT_S", "60")) if timeout_s is None else timeout_s
        self.pad = SymmetricBuffer(256, group, rank, world) if world > 1 else None

    def __call__(self) -> None:
        if self.world <= 1:
            return
        self.epoch += 1                       # host-side count (diagnostics); the kernel keeps its own
        self.pad._C.p2p_barrier(self.pad.peer_ptrs(), self.rank, 0, self.timeout_s)

    def late_peers(self):
        """After a barrier timeout: ``{peer: epoch}`` of the slots that never arrived."""
        flags = self.pad.view([64], torch.int32).cpu().tolist()
        return {r: flags[16 + r] for r in range(self.world) if flags[16 + r] != 0}


class P2PAllToAll:
    """All-to-all-v over peer memory (``csrc/p2p.cu: p2p_alltoall``): every rank stores its
    per-peer segments straight into the peers' symmetric receive buffers over NVLink, then a
    flag barrier publishes them.  Drop-in data plane for ``dist.all_to_all_single`` on one
    NVSwitch box -- the NCCL-free Repartition (SURVEY.md §5.8, BASELINE config 5).

    ``capacity_bytes`` is the largest receive total any rank will see; segments are padded to
    16 bytes inside the buffers.
    """

    def __init__(self, group, rank: int, world: int, capacity_bytes: int, ctas_per_peer: int = 16):
        self.group, self.rank, self.world = group, rank, world
        self.capacity = int((capacity_bytes + 16 * world + 255) // 256 * 256)
        self.recv = [SymmetricBuffer(self.capacity, group, rank, world) for _ in range(2)]   # double buffered
        self.barrier = PeerBarrier(group, rank, world)
        self.ctas = ctas_per_peer
        self._flip = 0
        self._cache = {}
        self._C = build.load()

    @staticmethod
    def _pad16(n: int) -> int:
        return (n + 15) // 16 * 16

    def _layout(self, es: int, send_counts, recv_counts_matrix):
        """Byte offsets for one (element size, counts) signature; cached -- the models reuse a
        handful of signatures every step."""
        key = (es, tuple(int(c) for c in send_counts), tuple(tuple(int(c) for c in r) for r in recv_counts_matrix))
        hit = self._cache.get(key)
        if hit is None:
            W = self.world
            dst_off = [sum(self._pad16(recv_counts_matrix[d][s] * es) for s in range(self.rank)) for d in range(W)]
            so = [0]
            for p in range(W):
                so.append(so[-1] + self._pad16(int(send_counts[p]) * es))
            aligned_send = all(int(send_counts[p]) * es % 16 == 0 for p in range(W))
            mine = [int(c) for c in recv_counts_matrix[self.rank]]
            aligned_recv = all(c * es % 16 == 0 for c in mine)
            per_peer = max(so[p + 1] - so[p] for p in range(W))
            ctas = max(1, min(16, per_peer // 65536))
            hit = (dst_off, so, aligned_send, mine, aligned_recv, ctas)
            self._cache[key] = hit
        return hit

    def exchange(self, send: torch.Tensor, send_counts: Sequence[int], recv_counts_matrix,
                 copy: bool = True) -> torch.Tensor:
        """``copy=False`` returns a *view* of the receive window (valid until the exchange after
        the next one) when the segments are 16-byte multiples -- the caller consumes it at once.
        ``send``: flat contiguous tensor whose consecutive pieces of ``send_counts[p]``
        elements go to peer ``p``.  ``recv_counts_matrix[d][s]``: elements rank ``s`` sends to
        rank ``d`` (every rank can compute it from the Repartition plans).  Returns a flat
        tensor with the pieces received from rank 0, 1, ... concatenated."""
        es = send.element_size()
        W = self.world
        buf = self.recv[self._flip]
        self._flip ^= 1
        dst_off, so, aligned_send, mine, aligned_recv, ctas = self._layout(es, send_counts, recv_counts_matrix)
        if aligned_send:
            packed = send.view(torch.uint8)
        else:                                   # pad every segment to a 16-byte boundary
            packed = torch.zeros(so[-1], dtype=torch.uint8, device=send.device)
            src = send.view(torch.uint8)
            o = 0
            for p in range(W):
                nb = int(send_counts[p]) * es
                packed[so[p]:so[p] + nb] = src[o:o + nb]
                o += nb
        self._C.p2p_alltoall(packed, so, buf.peer_ptrs(), dst_off, ctas)
        self.barrier()
        total = sum(mine)
        raw = buf.view([self.capacity], torch.uint8)
        if aligned_recv:                        # padded layout == dense layout: one copy out of the window
            window = raw[:total * es].view(send.dtype)
            return window.clone() if copy else window
        out = torch.empty(total, dtype=send.dtype, device=send.device)
        o_b, o_e = 0, 0
        for s in range(W):
            n = mine[s]
            if n:
                out[o_e:o_e + n] = raw[o_b:o_b + n * es].view(send.dtype)
            o_b += self._pad16(n * es)
            o_e += n
        return out
