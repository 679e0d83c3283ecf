"""Every channel width the engine supports, through every kernel templated on it, against float64 references
(H100 only).  Each kernel is instantiated for C in SUPPORTED_WIDTHS; a width that never runs in a test is a
width whose code nobody has seen execute."""
import math

import pytest
import torch
import torch.nn.functional as F

from dfno_b200.models.fused import LIFT_MAX_W, SUPPORTED_WIDTHS

pytestmark = pytest.mark.gpu

DEV = "cuda"


def C_():
    from dfno_b200.ops import build
    return build.load()


def bf(t):
    return t.to(torch.bfloat16)


def _f64(t):
    return t.detach().to(torch.complex128 if t.is_complex() else torch.float64)


def rel(got, want):
    got, want = _f64(got), _f64(want)
    return float((got - want).norm() / want.norm().clamp_min(1e-300))


def entry(got, want):
    """Largest error of one entry over its own magnitude plus the rms of the reference: a bf16 output is good to
    2^-8 of its value, and outliers of a product of normals reach many rms."""
    got, want = _f64(got), _f64(want)
    return float(((got - want).abs() / (want.abs() + want.abs().pow(2).mean().sqrt())).max())


def gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------ spectral mix
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("C", SUPPORTED_WIDTHS)
def test_spectral_mix_widths(C, accumulate):
    """B = 2 (the per-batch weight-gradient sum runs), Q = 1037 (not a multiple of 64)."""
    B, Q = 2, 1037
    g = gen(C)
    x = bf(torch.randn(B, C, Q, 2, device=DEV, generator=g))
    w = torch.randn(C, C, Q, 2, device=DEV, generator=g) / math.sqrt(C)
    xc, wc = torch.view_as_complex(x.double()), torch.view_as_complex(w.double())
    y = torch.full_like(x, 9.0)
    C_().spectral_mix_fwd(x.view(-1), w, y.view(-1), B, C, Q)
    yref = torch.einsum("biq,ioq->boq", xc, wc)
    yc = torch.view_as_complex(y.double())
    assert rel(yc, yref) < 5e-3 and entry(yc, yref) < 2e-2, (rel(yc, yref), entry(yc, yref))
    dy = bf(torch.randn(B, C, Q, 2, device=DEV, generator=g))
    dyc = torch.view_as_complex(dy.double())
    dw0 = torch.randn(C, C, Q, 2, device=DEV, generator=g)
    dx, dw = torch.full_like(x, 9.0), dw0.clone()
    C_().spectral_mix_bwd(x.view(-1), w, dy.view(-1), dx.view(-1), dw, accumulate, B, C, Q)
    dxref = torch.einsum("boq,ioq->biq", dyc, wc.conj())
    dxc = torch.view_as_complex(dx.double())
    assert rel(dxc, dxref) < 5e-3 and entry(dxc, dxref) < 2e-2, (rel(dxc, dxref), entry(dxc, dxref))
    dwref = torch.einsum("biq,boq->ioq", xc.conj(), dyc)
    if accumulate:
        dwref = dwref + torch.view_as_complex(dw0.double())
    dwc = torch.view_as_complex(dw.double())
    assert rel(dwc, dwref) < 1e-6 and entry(dwc, dwref) < 1e-5, (rel(dwc, dwref), entry(dwc, dwref))


# ------------------------------------------------------------------------------------------ lift
def _lift_T(C, Cin, Tin):
    if Tin < 64:
        return 12
    T = (LIFT_MAX_W - 2 * (C * Cin + C)) // (Tin + 1)       # just inside the kernel's shared-memory budget
    return T - T % 2


@pytest.mark.parametrize("xdt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("Tin", [1, 5, 64])
@pytest.mark.parametrize("Cin", [1, 2, 3, 4])
@pytest.mark.parametrize("C", SUPPORTED_WIDTHS)
def test_lift_widths(C, Cin, Tin, xdt):
    B, X, Y, Z = 2, 3, 4, 16
    T = _lift_T(C, Cin, Tin)
    assert T * Tin + T + 2 * (C * Cin + C) <= LIFT_MAX_W
    g = gen(100 * C + 10 * Cin + Tin)
    x = torch.randn(B, Cin, X, Y, Z, Tin, device=DEV, generator=g).to(xdt)
    W1 = torch.randn(T, Tin, device=DEV, generator=g) / math.sqrt(Tin)
    b1 = torch.randn(T, device=DEV, generator=g) * 0.3
    W2 = torch.randn(C, Cin, device=DEV, generator=g) / math.sqrt(Cin)
    b2 = torch.randn(C, device=DEV, generator=g) * 0.3
    h = torch.full((B * C * X * Y * T * Z,), 9.0, device=DEV, dtype=torch.bfloat16)
    dims = [B, Cin, Tin, C, T, X, Y, Z]
    C_().lift_fwd(x, W1, b1, W2, b2, h, dims)
    params = [p.double().requires_grad_() for p in (W1, b1, W2, b2)]
    a1 = F.gelu(torch.einsum("ti,bcxyzi->bcxyzt", params[0], x.double()) + params[1])
    ref = F.gelu(torch.einsum("oc,bcxyzt->boxyzt", params[2], a1) + params[3].view(1, C, 1, 1, 1, 1))
    ref_eng = ref.permute(0, 1, 2, 3, 5, 4)                                  # engine layout [B,C,X,Y,T,Z]
    got = h.view(B, C, X, Y, T, Z)
    assert rel(got, ref_eng) < 6e-3 and entry(got, ref_eng) < 2e-2, (rel(got, ref_eng), entry(got, ref_eng))
    dh = bf(torch.randn(B, C, X, Y, T, Z, device=DEV, generator=g))
    ref_eng.backward(dh.double())
    grads = [torch.zeros_like(p) for p in (W1, b1, W2, b2)]
    C_().lift_bwd(x, W1, b1, W2, b2, dh.view(-1), *grads, dims)
    for name, got, p in zip(("W1", "b1", "W2", "b2"), grads, params):
        assert rel(got, p.grad) < 1e-2, (name, rel(got, p.grad))          # packed fp16 GELU' (sm90_ptx.cuh)


# ------------------------------------------------------------------------------------------ bypass + GELU
def _pad(M):
    out = torch.zeros(32, 64, device=DEV, dtype=torch.bfloat16)
    out[:M.shape[0], :M.shape[1]] = bf(M)
    return out


@pytest.mark.parametrize("tc,S", [(False, 642), (False, 704), (True, 640)], ids=["cuda_core_642", "cuda_core_704", "tc_640"])
@pytest.mark.parametrize("C", SUPPORTED_WIDTHS)
def test_bypass_gelu_widths(C, tc, S):
    """CUDA-core bypass with S even but not a multiple of 128 (704 = 5.5 x 128, the engine's kreduce route; 642 also
    not a multiple of 8), and the tensor-core bypass (S a multiple of 128).  B = 2."""
    B = 2
    g = gen(C + S)
    h = bf(torch.randn(B, C, S, device=DEV, generator=g))
    spec = bf(torch.randn(B, C, S, device=DEV, generator=g))
    W = torch.randn(C, C, device=DEV, generator=g) / math.sqrt(C)
    Wr = bf(W).double() if tc else W.double()                                 # the tensor-core path rounds W to bf16
    pre_ref = spec.double() + torch.einsum("oi,bis->bos", Wr, h.double())
    out_ref = F.gelu(pre_ref)
    CP = (C + 7) // 8 * 8
    for cl in (False, True):
        pre = spec.clone().view(-1)
        out = torch.full((B * C * S,), 9.0, device=DEV, dtype=torch.bfloat16)
        out_cl = torch.zeros(B * S, CP, device=DEV, dtype=torch.bfloat16)          # the engine allocates it zeroed
        if tc:
            C_().bypass_fwd_tc(h.view(-1), pre, _pad(W), None if cl else out, out_cl if cl else None, CP, B, C, S, True)
        else:
            C_().bypass_gelu_fwd(h.view(-1), pre, W, None if cl else out, out_cl if cl else None, CP, B, C, S, True)
        assert rel(pre.view(B, C, S), pre_ref) < 6e-3 and entry(pre.view(B, C, S), pre_ref) < 2e-2
        if cl:
            got = out_cl.view(B, S, CP)[:, :, :C].permute(0, 2, 1)
            assert (out_cl.view(B, S, CP)[:, :, C:] == 0).all()
        else:
            got = out.view(B, C, S)
        assert rel(got, out_ref) < 8e-3 and entry(got, out_ref) < 2e-2, (cl, rel(got, out_ref), entry(got, out_ref))
    dout = bf(torch.randn(B, C, S, device=DEV, generator=g))
    pre_b = bf(pre_ref)
    gpre_ref = dout.double() * gelu_grad(pre_b.double())
    dhb_ref = torch.einsum("oi,bos->bis", Wr, gpre_ref)
    for cl in (False, True):
        dpre = pre_b.clone().view(-1)
        dhb = torch.full((B * C * S,), 9.0, device=DEV, dtype=torch.bfloat16)
        dW = torch.zeros(C, C, device=DEV)
        dcl = torch.zeros(B * S, CP, device=DEV, dtype=torch.bfloat16)
        dcl.view(B, S, CP)[:, :, :C] = dout.permute(0, 2, 1)
        args_in = (None, dcl, CP) if cl else (dout.view(-1), None, CP)
        if tc:
            C_().bypass_bwd_tc(*args_in, dpre, h.view(-1), _pad(W.t()), dhb, dW, B, C, S)
        else:
            C_().bypass_gelu_bwd(*args_in, dpre, W, dpre, dhb, B, C, S)
        assert rel(dpre.view(B, C, S), gpre_ref) < 8e-3
        assert rel(dhb.view(B, C, S), dhb_ref) < 1e-2
        if not tc and S % 8:
            continue                                   # kreduce_gemm needs 16-byte row pitches (S % 8 == 0)
        if not tc:
            for b in range(B):
                C_().kreduce_gemm(dpre.view(B, C, S)[b], S, C, h[b], S, C, S, dW)
        dW_ref = torch.einsum("bos,bis->oi", dpre.double().view(B, C, S), h.double())
        assert rel(dW, dW_ref) < 2e-3, (cl, rel(dW, dW_ref))


# ------------------------------------------------------------------------------------------ fused pointwise kernels
@pytest.mark.parametrize("mode", ["fwd", "adj"])
@pytest.mark.parametrize("C", SUPPORTED_WIDTHS)
def test_spectral_out_widths(C, mode):
    from dfno_b200.ops.gemm import pad_operator
    B, L, Z, K1 = 2, 97, 64, 24
    g = gen(200 + C)
    U = bf(torch.randn(B * C, L, K1, device=DEV, generator=g))
    h = bf(torch.randn(B * C, L, Z, device=DEV, generator=g))
    Fop = torch.randn(Z, K1, device=DEV, generator=g) / math.sqrt(K1)
    W = torch.randn(C, C, device=DEV, generator=g) / math.sqrt(C)
    pre = torch.full((B * C, L, Z), 9.0, device=DEV, dtype=torch.bfloat16)
    out = torch.full((B * C, L, Z), 9.0, device=DEV, dtype=torch.bfloat16)
    adj = mode == "adj"
    C_().spectral_out(U, h, pad_operator(Fop), W, adj, None if adj else pre, out, B, C, L, Z, K1, not adj, not adj)
    torch.cuda.synchronize()
    Wr = bf(W).double()
    spec = U.double() @ bf(Fop).double().t()
    mix = torch.einsum("oi,bilz->bolz", Wr.t() if adj else Wr, h.double().view(B, C, L, Z)).reshape(B * C, L, Z)
    ref_pre = spec + mix
    if adj:
        assert rel(out, ref_pre) < 6e-3 and entry(out, ref_pre) < 2e-2
    else:
        assert rel(out, F.gelu(ref_pre)) < 8e-3 and entry(out, F.gelu(ref_pre)) < 2e-2
        assert rel(pre, ref_pre) < 6e-3 and entry(pre, ref_pre) < 2e-2


@pytest.mark.parametrize("C", SUPPORTED_WIDTHS)
def test_dpre_dw_widths(C):
    B, L, Z = 2, 97, 64
    gn = gen(300 + C)
    g = bf(torch.randn(B * C, L, Z, device=DEV, generator=gn) * 1e-6)
    pre = bf(torch.randn(B * C, L, Z, device=DEV, generator=gn) * 1.5)
    h = bf(torch.randn(B * C, L, Z, device=DEV, generator=gn))
    dW0 = torch.randn(C, C, device=DEV, generator=gn) * 1e-4
    dW = dW0.clone()
    dpre = pre.clone()
    C_().dpre_dw(g, dpre, h, dW, B, C, L, Z)
    torch.cuda.synchronize()
    ref = g.double() * gelu_grad(pre.double())
    assert rel(dpre, ref) < 8e-3
    dW_ref = dW0.double() + torch.einsum("bos,bis->oi", dpre.double().view(B, C, L * Z), h.double().view(B, C, L * Z))
    assert rel(dW, dW_ref) < 2e-3, rel(dW, dW_ref)


@pytest.mark.parametrize("C", SUPPORTED_WIDTHS)
def test_channel_major_head_widths(C):
    B, X, Y, Z, T, H = 2, 4, 3, 8, 6, 128
    g = gen(400 + C)
    S = X * Y * T * Z
    h = bf(torch.randn(B * C, S, device=DEV, generator=g))
    W3 = torch.randn(H, C, device=DEV, generator=g) / math.sqrt(C)
    b3 = torch.randn(H, device=DEV, generator=g) * 0.2
    w4b4 = torch.randn(H + 1, device=DEV, generator=g) / math.sqrt(H)
    w3a = torch.zeros(H, 64, device=DEV, dtype=torch.bfloat16)
    w3a[:, :C] = bf(W3); w3a[:, C] = bf(b3)
    w3t = torch.zeros((C + 1 + 15) // 16 * 16, H, device=DEV, dtype=torch.float16)
    w3t[:C] = bf(W3).float().t().to(torch.float16)
    out = torch.full((B, 1, X, Y, Z, T), 5.0, device=DEV)
    R, SR = [Z, T, B * X * Y], [T, 1, Z * T]
    C_().head_fwd(h, w3a, w4b4, out, B, C, S, R, SR)
    hin = h.double().view(B, C, S).permute(0, 2, 1).reshape(B * S, C).requires_grad_()   # rows (b, x, y, t, z)
    W3r, b3r = bf(W3).double().requires_grad_(), bf(b3).double().requires_grad_()
    w4r = w4b4.double().requires_grad_()
    ref = F.gelu(hin @ W3r.t() + b3r) @ w4r[:H] + w4r[H]
    ref_pub = ref.view(B, X, Y, T, Z).permute(0, 1, 2, 4, 3).unsqueeze(1)
    assert rel(out, ref_pub) < 5e-3, rel(out, ref_pub)
    dy = torch.randn(B, 1, X, Y, Z, T, device=DEV, generator=g) * 3e-7       # a realistic loss-gradient scale
    ref_pub.backward(dy.double())
    gout = torch.full((B * C, S), 7.0, device=DEV, dtype=torch.bfloat16)
    gW3, gb3, gW4, gb4 = (torch.zeros(H, C, device=DEV), torch.zeros(H, device=DEV), torch.zeros(H, device=DEV),
                          torch.zeros(1, device=DEV))
    ws = torch.zeros(1, device=DEV, dtype=torch.int32)
    C_().head_bwd2(h, w3a, w3t, w4b4[:H].contiguous(), dy.contiguous(), ws, gout, gW3, gb3, gW4, gb4, B, C, S, R, SR)
    torch.cuda.synchronize()
    gref = hin.grad.view(B, S, C).permute(0, 2, 1).reshape(B * C, S)
    assert rel(gout, gref) < 1e-2, rel(gout, gref)
    assert rel(gW3, W3r.grad) < 1e-2 and rel(gb3, b3r.grad) < 1e-2, (rel(gW3, W3r.grad), rel(gb3, b3r.grad))
    assert rel(gW4, w4r.grad[:H]) < 6e-3 and rel(gb4, w4r.grad[H:]) < 1e-4, (rel(gW4, w4r.grad[:H]), rel(gb4, w4r.grad[H:]))
