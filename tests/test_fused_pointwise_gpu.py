"""Round-2 fused pointwise kernels (packed-fp16 GELU, spectral_out, dpre_dw, channel-major projection head)
against plain PyTorch fp32 references of the same ops (H100 only)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def C_():
    from dfno_b200.ops import build
    return build.load()


def rel(a, b):
    return float((a.detach().float() - b.detach().float()).norm() / b.detach().float().norm().clamp_min(1e-30))


def bf(t):
    return t.to(torch.bfloat16)


def gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def test_packed_fp16_gelu_tracks_erf_gelu():
    x = torch.cat([torch.linspace(-12, 12, 200001, device="cuda"), torch.tensor([300.0, -300.0, 7e4, -7e4, 0.0], device="cuda")])
    x = x[: x.numel() // 2 * 2].contiguous()
    y, dy = C_().gelu_probe_h2(x)
    ref, dref = F.gelu(x), gelu_grad(x)
    assert torch.isfinite(y).all() and torch.isfinite(dy).all()     # inputs beyond the fp16 range saturate
    ok = x.abs() < 6e4
    err = ((y - ref).abs() / x.abs().clamp_min(1.0))[ok]
    derr = (dy - dref).abs()[ok]
    assert float(err.max()) < 2.5e-3, float(err.max())          # fp16 arithmetic: ~1e-3 * max(1, |x|)
    assert float(derr.max()) < 8e-3, float(derr.max())


@pytest.mark.parametrize("B,C,L,Z,K1,mode", [
    (1, 20, 301, 128, 48, "fwd"), (1, 20, 301, 128, 48, "fwd_nopre"), (1, 20, 301, 128, 48, "adj"),
    (2, 8, 97, 64, 24, "fwd"), (1, 32, 50, 256, 48, "fwd"), (1, 12, 33, 40, 16, "adj"), (1, 24, 64, 192, 64, "fwd"), (1, 16, 40, 64, 128, "fwd"),
])
def test_spectral_out_matches_reference(B, C, L, Z, K1, mode):
    from dfno_b200.ops.gemm import pad_operator
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(11)
    U = bf(torch.randn(B * C, L, K1, device=dev, generator=g))
    h = bf(torch.randn(B * C, L, Z, device=dev, generator=g))
    Fop = torch.randn(Z, K1, device=dev, generator=g) / math.sqrt(K1)
    W = torch.randn(C, C, device=dev, generator=g) / math.sqrt(C)
    pre = torch.full((B * C, L, Z), 9.0, device=dev, dtype=torch.bfloat16)
    out = torch.full((B * C, L, Z), 9.0, device=dev, dtype=torch.bfloat16)
    adj = mode == "adj"
    C_().spectral_out(U, h, pad_operator(Fop), W, adj, None if mode != "fwd" else pre, out, B, C, L, Z, K1,
                      not adj, mode == "fwd")
    torch.cuda.synchronize()
    Wr = bf(W).float()
    spec = U.float() @ bf(Fop).float().t()
    mix = torch.einsum("oi,bilz->bolz", Wr.t() if adj else Wr, h.float().view(B, C, L, Z)).reshape(B * C, L, Z)
    ref_pre = spec + mix
    if adj:
        assert rel(out, ref_pre) < 6e-3
    else:
        assert rel(out, F.gelu(ref_pre)) < 8e-3
        if mode == "fwd":
            assert rel(pre, ref_pre) < 6e-3
        else:
            assert (pre == 9.0).all()


@pytest.mark.parametrize("B,C,L,Z", [(1, 20, 301, 128), (2, 8, 97, 64), (1, 32, 40, 256), (1, 12, 33, 40)])
def test_dpre_dw_matches_reference(B, C, L, Z):
    dev = "cuda"
    gen = torch.Generator(device=dev).manual_seed(12)
    g = bf(torch.randn(B * C, L, Z, device=dev, generator=gen) * 1e-6)       # loss gradients are tiny
    pre = bf(torch.randn(B * C, L, Z, device=dev, generator=gen) * 1.5)
    h = bf(torch.randn(B * C, L, Z, device=dev, generator=gen))
    dW = torch.full((C, C), 0.0, device=dev)
    dpre = pre.clone()
    C_().dpre_dw(g, dpre, h, dW, B, C, L, Z)
    C_().dpre_dw(g, pre.clone(), h, dW, B, C, L, Z)                          # accumulates
    torch.cuda.synchronize()
    ref = g.float() * gelu_grad(pre.float())
    assert rel(dpre, ref) < 8e-3
    refq = dpre.float().view(B, C, L * Z)
    dW_ref = 2 * torch.einsum("bos,bis->oi", refq, h.float().view(B, C, L * Z))
    assert rel(dW, dW_ref) < 2e-3, rel(dW, dW_ref)


@pytest.mark.parametrize("B,X,Y,Z,T,C", [(2, 4, 3, 8, 4, 20), (1, 3, 5, 16, 6, 8), (1, 2, 2, 8, 30, 32),
                                         (1, 40, 32, 64, 10, 20)])     # 6400 tiles: ~48 per CTA on 132 SMs, both epilogue groups
def test_channel_major_head_forward_backward(B, X, Y, Z, T, C):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(3)
    H = 128
    S = X * Y * T * Z
    h = bf(torch.randn(B * C, S, device=dev, generator=g))
    W3 = torch.randn(H, C, device=dev, generator=g) / math.sqrt(C)
    b3 = torch.randn(H, device=dev, generator=g) * 0.2
    w4b4 = torch.randn(H + 1, device=dev, generator=g) / math.sqrt(H)
    KR = (C + 1 + 15) // 16 * 16
    w3a = torch.zeros(H, 64, device=dev, dtype=torch.bfloat16)
    w3a[:, :C] = bf(W3); w3a[:, C] = bf(b3)
    w3t = torch.zeros(KR, H, device=dev, dtype=torch.float16)
    w3t[:C] = bf(W3).float().t().to(torch.float16)
    out = torch.full((B, 1, X, Y, Z, T), 5.0, device=dev)
    R, SR = [Z, T, B * X * Y], [T, 1, Z * T]
    C_().head_fwd(h, w3a, w4b4, out, B, C, S, R, SR)
    hin = h.float().view(B, C, S).permute(0, 2, 1).reshape(B * S, C).requires_grad_()   # rows (b, x, y, t, z)
    W3r, b3r, w4r = bf(W3).float().requires_grad_(), bf(b3).float().requires_grad_(), w4b4.clone().requires_grad_()
    ref = F.gelu(hin @ W3r.t() + b3r) @ w4r[:H] + w4r[H]
    ref_pub = ref.view(B, X, Y, T, Z).permute(0, 1, 2, 4, 3).unsqueeze(1)
    assert rel(out, ref_pub) < 5e-3, rel(out, ref_pub)
    dy = torch.randn(B, 1, X, Y, Z, T, device=dev, generator=g) * 3e-7       # a realistic loss-gradient scale
    ref_pub.backward(dy)
    gout = torch.full((B * C, S), 7.0, device=dev, dtype=torch.bfloat16)
    gW3, gb3, gW4, gb4 = (torch.zeros(H, C, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev),
                          torch.zeros(1, device=dev))
    ws = torch.zeros(1, device=dev, dtype=torch.int32)
    C_().head_bwd2(h, w3a, w3t, w4b4[:H].contiguous(), dy.contiguous(), ws, gout, gW3, gb3, gW4, gb4, B, C, S, R, SR)
    torch.cuda.synchronize()
    gref = hin.grad.view(B, S, C).permute(0, 2, 1).reshape(B * C, S)
    assert rel(gout, gref) < 1e-2, rel(gout, gref)
    assert rel(gW3, W3r.grad) < 1e-2 and rel(gb3, b3r.grad) < 1e-2, (rel(gW3, W3r.grad), rel(gb3, b3r.grad))
    assert rel(gW4, w4r.grad[:H]) < 6e-3 and rel(gb4, w4r.grad[H:]) < 1e-4, (rel(gW4, w4r.grad[:H]), rel(gb4, w4r.grad[H:]))
