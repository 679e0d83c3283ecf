"""The forward spectral_out against float64 (H100 only), tile by tile: every padded width (16 .. 64) of the last
64-column tile, one and two U blocks, every channel width class, lines that do not fill the last tile and fewer lines
than one tile.  pre and out are views between NaN guard bands: the kernel writes its outputs in place over ring
slots and TMA-stores them from there, clipped to the tensor, so no byte outside the outputs may change.

    pre = U F^T + W h (W^T h with transpose_w),  out = gelu(pre) (gelu = 1) or pre (gelu = 0)"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
GUARD = 4096                      # bf16 elements of NaN on each side of an output
# Z: last column tiles of 16, 48, 64, 16, 32, 64 and 64 padded columns
ZS = [16, 40, 64, 80, 96, 192, 256]
CS = [4, 12, 20, 32, 48, 64]      # R = 32, 10, 6, 4, 2, 2
K1S = [16, 48, 128]
MODES = ["gelu+pre", "gelu", "plain"]


def C_():
    from dfno_b200.ops import build
    return build.load()


def _f64(t):
    return t.detach().double()


def rel(got, want):
    got, want = _f64(got), _f64(want)
    return float((got - want).norm() / want.norm().clamp_min(1e-300))


def entry(got, want):
    """largest error of one entry over its own magnitude plus the rms of the reference"""
    got, want = _f64(got), _f64(want)
    return float(((got - want).abs() / (want.abs() + want.abs().pow(2).mean().sqrt())).max())


def guarded(n):
    """(buffer of n + 2 GUARD bf16 NaNs, view of its middle n elements)"""
    buf = torch.full((n + 2 * GUARD,), float("nan"), device=DEV, dtype=torch.bfloat16)
    return buf, buf[GUARD:GUARD + n]


def guards_intact(buf):
    bits = buf.view(torch.int16)
    nan = torch.full((GUARD,), float("nan"), device=DEV, dtype=torch.bfloat16).view(torch.int16)
    return bool((bits[:GUARD] == nan).all() and (bits[-GUARD:] == nan).all())


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("Z", ZS)
def test_forward_every_tile_width(Z, C):
    from dfno_b200.ops.gemm import pad_operator
    R = 128 // C
    g = torch.Generator(device=DEV).manual_seed(1000 * Z + C)
    # fewer lines than one tile (or one line at R = 2), and enough lines for several tiles per CTA and ring pass with
    # a partial last tile
    for B, L in ((2, max(1, R - 1)), (1, 40 * 132 * R // max(1, Z // 64) + R // 2 + 1)):
        for K1 in K1S:
            bf = torch.bfloat16
            U = (torch.randn(B * C, L, K1, device=DEV, generator=g) / math.sqrt(K1)).to(bf)
            h = torch.randn(B * C, L, Z, device=DEV, generator=g).to(bf)
            Fop = torch.randn(Z, K1, device=DEV, generator=g)
            W = torch.randn(C, C, device=DEV, generator=g) / math.sqrt(C)
            spec = U.double() @ Fop.to(bf).double().t()
            for mode in MODES:
                tw = mode == "plain"
                Wr = W.to(bf).double()
                mix = torch.einsum("oi,bilz->bolz", Wr.t() if tw else Wr, h.double().view(B, C, L, Z))
                ref = spec + mix.reshape(B * C, L, Z)
                n = B * C * L * Z
                pbuf, pre = guarded(n)
                obuf, out = guarded(n)
                gelu, save = mode != "plain", mode == "gelu+pre"
                C_().spectral_out(U, h, pad_operator(Fop), W, tw, pre.view(B * C, L, Z) if save else None,
                                  out.view(B * C, L, Z), B, C, L, Z, K1, gelu, save)
                torch.cuda.synchronize()
                case = (B, L, K1, mode)
                assert guards_intact(obuf), case
                assert guards_intact(pbuf), case
                o = out.view(B * C, L, Z)
                want = F.gelu(ref) if gelu else ref
                assert not o.isnan().any(), case
                assert rel(o, want) < 8e-3 and entry(o, want) < 2e-2, (case, rel(o, want), entry(o, want))
                if save:
                    p = pre.view(B * C, L, Z)
                    assert not p.isnan().any(), case
                    assert rel(p, ref) < 6e-3 and entry(p, ref) < 2e-2, (case, rel(p, ref), entry(p, ref))
                    # the GELU is evaluated on the same accumulator pair that pre rounds: out is gelu of exactly
                    # that pre's fp32 source, so it never strays from gelu(pre) by more than bf16 + packed-GELU error
                    assert entry(o, F.gelu(p.double())) < 2e-2, case
                else:
                    assert guards_intact(pbuf) and pre.view(torch.int16).eq(
                        torch.full((1,), float("nan"), dtype=torch.bfloat16, device=DEV).view(torch.int16)).all(), case
