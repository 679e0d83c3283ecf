"""Native FFT along the last axis with the FNO's truncation / zero padding fused in
(``csrc/fft_radix.cu``: shared-memory Stockham, radix 4).

The fused engine expresses *truncated* transforms as tensor-core GEMMs (``ops/operators.py``), which is the
right trade while few modes are kept (``m <= N/4``).  These functions are the complementary path -- wide spectra,
un-truncated transforms, power-of-two axes up to 4096 samples -- and what the portable backend uses on a GPU when
built with ``fft_impl="native"`` (no cuFFT on that path).  Complex data is interleaved ``[..., n, 2]``
(``torch.view_as_real`` layout); fp32 or bf16 storage, fp32 arithmetic.  CPU tensors, other dtypes and
non-power-of-two lengths fall back to ``torch.fft`` with identical semantics
(reference ops: reference ``dfno/dfno.py:252-258,273-285``)."""
from __future__ import annotations

import torch

__all__ = ["rfft_trunc", "fft_trunc", "ifft_pad", "irfft_pad", "native_ok"]


def native_ok(t: torch.Tensor, N: int) -> bool:
    return bool(t.is_cuda and t.dtype in (torch.float32, torch.bfloat16) and 2 <= N <= 4096 and N & (N - 1) == 0)


def _launch(x, out, N, inverse, in_real, out_real, one_sided, m):
    from . import build
    lines = x.numel() // (N if (in_real and not inverse) else (x.shape[-2] * 2))
    build.load().fft_radix(x, out, N, lines, inverse, in_real, out_real, one_sided, m)
    return out


def rfft_trunc(x: torch.Tensor, m: int = 0) -> torch.Tensor:
    """Real ``[..., N]`` -> modes ``[0, m)`` (all ``N/2+1`` for ``m = 0``) as ``[..., m, 2]``."""
    N = x.shape[-1]
    keep = m or N // 2 + 1
    if not native_ok(x, N):
        return torch.view_as_real(torch.fft.rfft(x.float(), dim=-1)[..., :keep]).to(x.dtype).contiguous()
    x = x.contiguous()
    out = torch.empty(*x.shape[:-1], keep, 2, device=x.device, dtype=x.dtype)
    return _launch(x, out, N, False, True, False, True, m)


def fft_trunc(x: torch.Tensor, m: int = 0) -> torch.Tensor:
    """Complex ``[..., N, 2]`` -> modes ``[0, m) u [N-m, N)`` (all for ``m = 0``) as ``[..., 2m, 2]``."""
    N = x.shape[-2]
    if not native_ok(x, N):
        X = torch.fft.fft(torch.view_as_complex(x.float().contiguous()), dim=-1)
        X = X if not m else torch.cat([X[..., :m], X[..., N - m:]], dim=-1)
        return torch.view_as_real(X).to(x.dtype).contiguous()
    x = x.contiguous()
    out = torch.empty(*x.shape[:-2], 2 * m if m else N, 2, device=x.device, dtype=x.dtype)
    return _launch(x, out, N, False, False, False, False, m)


def ifft_pad(X: torch.Tensor, N: int) -> torch.Tensor:
    """Two-sided modes ``[..., 2m, 2]`` (or a full spectrum ``[..., N, 2]``) -> complex ``[..., N, 2]`` (1/N scaling)."""
    kept = X.shape[-2]
    m = 0 if kept == N else kept // 2
    if not native_ok(X, N):
        Xc = torch.view_as_complex(X.float().contiguous())
        if m:
            full = Xc.new_zeros(*Xc.shape[:-1], N)
            full[..., :m], full[..., N - m:] = Xc[..., :m], Xc[..., m:]
            Xc = full
        return torch.view_as_real(torch.fft.ifft(Xc, dim=-1)).to(X.dtype).contiguous()
    X = X.contiguous()
    out = torch.empty(*X.shape[:-2], N, 2, device=X.device, dtype=X.dtype)
    return _launch(X, out, N, True, False, False, False, m)


def irfft_pad(X: torch.Tensor, N: int) -> torch.Tensor:
    """One-sided modes ``[..., m, 2]`` of a Hermitian spectrum -> real ``[..., N]`` (``torch.fft.irfft(n=N)`` of the
    zero-padded spectrum: the imaginary parts of the DC and Nyquist bins are ignored)."""
    kept = X.shape[-2]
    m = 0 if kept == N // 2 + 1 else kept
    if not native_ok(X, N):
        Xc = torch.view_as_complex(X.float().contiguous())
        return torch.fft.irfft(Xc, n=N, dim=-1).to(X.dtype).contiguous()
    X = X.contiguous()
    out = torch.empty(*X.shape[:-2], N, device=X.device, dtype=X.dtype)
    return _launch(X, out, N, True, False, True, True, m)


# ------------------------------------------------------------------------------------------------------------
# differentiable transform-along-a-dimension wrappers (complex tensors in / out), used by the portable backend
# with ``fft_impl="native"``.  Backward passes are the adjoint transforms, themselves calls into the same kernel:
#   adj(fft_trunc)  = N * ifft_pad          adj(ifft_pad)  = fft_trunc / N
#   adj(rfft_trunc) = N * Re(ifft(pad))     adj(irfft_pad) = w_k / N * rfft_trunc     (w = 1 at DC / Nyquist, else 2)
# ------------------------------------------------------------------------------------------------------------

def _to_last(x: torch.Tensor, dim: int) -> torch.Tensor:
    return x.movedim(dim, -1).contiguous()


def _from_last(x: torch.Tensor, dim: int) -> torch.Tensor:
    return x.movedim(-1, dim)


class _FwdC2C(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dim, m):
        ctx.dim, ctx.m, ctx.N = dim, m, x.shape[dim]
        y = fft_trunc(torch.view_as_real(_to_last(x, dim)), m)
        return _from_last(torch.view_as_complex(y), dim)

    @staticmethod
    def backward(ctx, g):
        gx = ifft_pad(torch.view_as_real(_to_last(g, ctx.dim)), ctx.N)
        return _from_last(torch.view_as_complex(gx), ctx.dim) * ctx.N, None, None


class _InvC2C(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, dim, N):
        ctx.dim, ctx.N = dim, N
        ctx.m = 0 if X.shape[dim] == N else X.shape[dim] // 2
        y = ifft_pad(torch.view_as_real(_to_last(X, dim)), N)
        return _from_last(torch.view_as_complex(y), dim)

    @staticmethod
    def backward(ctx, g):
        gX = fft_trunc(torch.view_as_real(_to_last(g, ctx.dim)), ctx.m)
        return _from_last(torch.view_as_complex(gX), ctx.dim) / ctx.N, None, None


class _FwdR2C(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dim, m):
        ctx.dim, ctx.N = dim, x.shape[dim]
        y = rfft_trunc(_to_last(x, dim), m)
        ctx.keep = y.shape[-2]
        return _from_last(torch.view_as_complex(y), dim)

    @staticmethod
    def backward(ctx, g):
        gl = torch.view_as_real(_to_last(g, ctx.dim))
        full = gl.new_zeros(*gl.shape[:-2], ctx.N, 2)            # one-sided modes, NO Hermitian completion
        full[..., :ctx.keep, :] = gl
        gx = ifft_pad(full, ctx.N)[..., 0] * ctx.N
        return _from_last(gx, ctx.dim), None, None


class _InvC2R(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, dim, N):
        ctx.dim, ctx.N, ctx.keep = dim, N, X.shape[dim]
        return _from_last(irfft_pad(torch.view_as_real(_to_last(X, dim)), N), dim)

    @staticmethod
    def backward(ctx, g):
        m = 0 if ctx.keep == ctx.N // 2 + 1 else ctx.keep
        gX = rfft_trunc(_to_last(g, ctx.dim), m)                  # [..., keep, 2]
        w = torch.full((ctx.keep, 1), 2.0 / ctx.N, device=g.device, dtype=gX.dtype)
        w[0] = 1.0 / ctx.N
        if ctx.N % 2 == 0 and ctx.keep == ctx.N // 2 + 1:
            w[-1] = 1.0 / ctx.N
        gX = gX * w
        gX[..., 0, 1] = 0                                         # the imaginary part of DC (and Nyquist) is ignored
        if ctx.N % 2 == 0 and ctx.keep == ctx.N // 2 + 1:
            gX[..., -1, 1] = 0
        return _from_last(torch.view_as_complex(gX.contiguous()), ctx.dim), None, None


def fwd_transform(x: torch.Tensor, dim: int, m: int, real_input: bool) -> torch.Tensor:
    """Differentiable ``keep_modes(fft(x, dim))``: one-sided ``[0, m)`` for a real input, else two-sided."""
    return _FwdR2C.apply(x, dim, m) if real_input else _FwdC2C.apply(x, dim, m)


def inv_transform(X: torch.Tensor, dim: int, N: int, real_output: bool) -> torch.Tensor:
    """Differentiable ``ifft(pad_modes(X), dim)`` / ``irfft(pad_modes(X), n=N, dim)``."""
    return _InvC2R.apply(X, dim, N) if real_output else _InvC2C.apply(X, dim, N)
