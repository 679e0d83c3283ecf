"""Truncated DFT operators as real matrices acting on interleaved (re, im) data.

Every stage of the distributed spectral convolution is ``out = A @ Op^T`` with ``A`` the
field viewed as ``[lines, K]`` and ``Op`` one of the matrices below (built in float64,
rounded to bf16 for the tensor cores).  Conventions are ``torch.fft``'s: forward unscaled,
inverse scaled by ``1/N``; the retained modes of a two-sided axis are ``[0, m) u [N-m, N)``
in that order, of the one-sided (rfft) axis ``[0, m)`` (reference ``dfno/dfno.py:104-111``).

Because complex numbers are stored as adjacent (re, im) pairs, a complex DFT is ONE real
GEMM against ``[[c, s], [-s, c]]`` blocks -- no 3M trick, no de-interleave pass.  The
adjoint (backward) operators are plain transposes of these real matrices; in particular the
adjoint of the Hermitian-weighted inverse real transform is *not* a forward rfft, which is
why it is derived here rather than borrowed from an FFT library.
"""
from __future__ import annotations

import math

import torch

__all__ = ["retained_frequencies", "fwd_real_to_complex", "fwd_complex", "inv_complex",
           "inv_complex_hermitian", "inv_complex_to_real"]


def retained_frequencies(N: int, m: int, two_sided: bool) -> torch.Tensor:
    """Actual DFT frequency index of every retained mode, in storage order."""
    if two_sided:
        return torch.cat([torch.arange(m), torch.arange(N - m, N)]).to(torch.float64)
    return torch.arange(m, dtype=torch.float64)


def _angles(N: int, m: int, two_sided: bool) -> torch.Tensor:
    k = retained_frequencies(N, m, two_sided)
    n = torch.arange(N, dtype=torch.float64)
    return 2.0 * math.pi * torch.outer(k, n) / N          # [K, N]


def fwd_real_to_complex(N: int, m: int, two_sided: bool = True) -> torch.Tensor:
    """``[2K, N]``: real samples -> retained modes ``sum_n x[n] exp(-i th)`` as (re, im)."""
    th = _angles(N, m, two_sided)
    K = th.shape[0]
    op = torch.empty(K, 2, N, dtype=torch.float64)
    op[:, 0] = torch.cos(th)
    op[:, 1] = -torch.sin(th)
    return op.reshape(2 * K, N)


def fwd_complex(N: int, m: int, two_sided: bool = True) -> torch.Tensor:
    """``[2K, 2N]``: complex samples (re, im interleaved) -> retained modes."""
    th = _angles(N, m, two_sided)
    K = th.shape[0]
    c, s = torch.cos(th), torch.sin(th)
    op = torch.empty(K, 2, N, 2, dtype=torch.float64)
    op[:, 0, :, 0] = c      # out_r += c * in_r + s * in_i      (w = c - i s)
    op[:, 0, :, 1] = s
    op[:, 1, :, 0] = -s     # out_i += -s * in_r + c * in_i
    op[:, 1, :, 1] = c
    return op.reshape(2 * K, 2 * N)


def _inv_blocks(N: int, m: int, two_sided: bool, weights: torch.Tensor) -> torch.Tensor:
    th = _angles(N, m, two_sided).t()                     # [N, K]
    K = th.shape[1]
    c, s = torch.cos(th) * weights, torch.sin(th) * weights
    op = torch.empty(N, 2, K, 2, dtype=torch.float64)
    op[:, 0, :, 0] = c      # out_r += c * in_r - s * in_i      (w = c + i s)
    op[:, 0, :, 1] = -s
    op[:, 1, :, 0] = s
    op[:, 1, :, 1] = c
    return op


def inv_complex(N: int, m: int, two_sided: bool = True) -> torch.Tensor:
    """``[2N, 2K]``: zero-padded inverse complex DFT ``(1/N) sum_k X[k] exp(+i th)``."""
    K = 2 * m if two_sided else m
    return _inv_blocks(N, m, two_sided, torch.full((K,), 1.0 / N, dtype=torch.float64)).reshape(2 * N, 2 * K)


def inv_complex_hermitian(N: int, m: int) -> torch.Tensor:
    """``[2N, 2m]``: the complex half of a C2R transform along the rfft axis when another
    axis is still to be inverted afterwards: ``U[n] = (1/N) sum_k a_k Y[k] exp(+i th)`` with
    ``a_0 = 1``, ``a_{N/2} = 1`` and ``a_k = 2`` otherwise (the mirrored half folded in);
    the real part is taken by the *last* inverse stage."""
    k = torch.arange(m)
    a = torch.where((k == 0) | (2 * k == N), 1.0, 2.0).to(torch.float64) / N
    return _inv_blocks(N, m, False, a).reshape(2 * N, 2 * m)


def inv_complex_to_real(N: int, m: int, two_sided: bool = True) -> torch.Tensor:
    """``[N, 2K]``: ``Re[(1/N) sum_k U[k] exp(+i th)]``."""
    K = 2 * m if two_sided else m
    blocks = _inv_blocks(N, m, two_sided, torch.full((K,), 1.0 / N, dtype=torch.float64))
    return blocks[:, 0].reshape(N, 2 * K)
