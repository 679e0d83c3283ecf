"""Every sm_90a kernel against a plain PyTorch fp32 reference of the same op (H100 only)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def C_():
    from dfno_b200.ops import build
    return build.load()


def rel(a, b):
    a = torch.view_as_real(a) if a.is_complex() else a
    b = torch.view_as_real(b) if b.is_complex() else b
    return float((a.detach().float() - b.detach().float()).norm() / b.detach().float().norm().clamp_min(1e-30))


def bf(t):
    return t.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------ lift
@pytest.mark.parametrize("B,Cin,Tin,C,T,X,Y,Z", [(1, 1, 1, 20, 20, 8, 6, 16), (2, 2, 3, 8, 12, 4, 4, 8)])
def test_lift_forward_backward(B, Cin, Tin, C, T, X, Y, Z):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, Cin, X, Y, Z, Tin, device=dev, generator=g)
    W1 = torch.randn(T, Tin, device=dev, generator=g) * 0.7
    b1 = torch.randn(T, device=dev, generator=g) * 0.3
    W2 = torch.randn(C, Cin, device=dev, generator=g) * 0.7
    b2 = torch.randn(C, device=dev, generator=g) * 0.3
    h = torch.empty(B * C * X * Y * T * Z, device=dev, dtype=torch.bfloat16)
    dims = [B, Cin, Tin, C, T, X, Y, Z]
    C_().lift_fwd(x, W1, b1, W2, b2, h, dims)
    params = [p.clone().requires_grad_() for p in (W1, b1, W2, b2)]
    a1 = F.gelu(torch.einsum("ti,bcxyzi->bcxyzt", params[0], x) + params[1])
    ref = F.gelu(torch.einsum("oc,bcxyzt->boxyzt", params[2], a1) + params[3].view(1, C, 1, 1, 1, 1))
    ref_eng = ref.permute(0, 1, 2, 3, 5, 4)                                  # engine layout [B,C,X,Y,T,Z]
    assert rel(h.view(B, C, X, Y, T, Z), ref_eng) < 6e-3
    dh = torch.randn(B, C, X, Y, T, Z, device=dev, generator=g)
    ref_eng.backward(bf(dh).float())
    grads = [torch.zeros_like(p) for p in (W1, b1, W2, b2)]
    C_().lift_bwd(x, W1, b1, W2, b2, bf(dh).contiguous().view(-1), *grads, dims)
    for got, p in zip(grads, params):
        assert rel(got, p.grad) < 5e-3, (got.shape, rel(got, p.grad))     # packed fp16 GELU' (sm90_ptx.cuh)


# ------------------------------------------------------------------------------------------ bypass + GELU
@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("B,C,S", [(1, 20, 128 * 37), (2, 8, 128 * 5)])
def test_bypass_gelu_forward_backward(tc, B, C, S):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(1)
    h = bf(torch.randn(B, C, S, device=dev, generator=g))
    spec = bf(torch.randn(B, C, S, device=dev, generator=g))
    W = torch.randn(C, C, device=dev, generator=g) / math.sqrt(C)
    pad = lambda M: torch.zeros(32, 64, device=dev, dtype=torch.bfloat16).index_put_(
        (torch.arange(M.shape[0], device=dev)[:, None], torch.arange(M.shape[1], device=dev)[None, :]), bf(M))
    Wr = bf(W).float() if tc else W                                           # the tc path rounds W to bf16
    pre_ref = spec.float() + torch.einsum("oi,bis->bos", Wr, h.float())
    out_ref = F.gelu(pre_ref)
    CP = (C + 7) // 8 * 8
    for cl in (False, True):
        pre = spec.clone().view(-1)
        out = torch.empty(B * C * S, device=dev, dtype=torch.bfloat16)
        out_cl = torch.zeros(B * S, CP, device=dev, dtype=torch.bfloat16)
        if tc:
            C_().bypass_fwd_tc(h.view(-1), pre, pad(W), None if cl else out, out_cl if cl else None, CP, B, C, S, True)
        else:
            C_().bypass_gelu_fwd(h.view(-1), pre, W, None if cl else out, out_cl if cl else None, CP, B, C, S, True)
        assert rel(pre.view(B, C, S), pre_ref) < 6e-3
        if cl:
            got = out_cl.view(B, S, CP)[:, :, :C].permute(0, 2, 1)
            assert (out_cl.view(B, S, CP)[:, :, C:] == 0).all()
        else:
            got = out.view(B, C, S)
        assert rel(got, out_ref) < 8e-3, (tc, cl, rel(got, out_ref))
    # backward
    dout = bf(torch.randn(B, C, S, device=dev, generator=g))
    pre_b = bf(pre_ref)
    gpre_ref = dout.float() * (0.5 * (1 + torch.erf(pre_b.float() / math.sqrt(2))) +
                               pre_b.float() * torch.exp(-0.5 * pre_b.float() ** 2) / math.sqrt(2 * math.pi))
    dhb_ref = torch.einsum("oi,bos->bis", Wr, gpre_ref)
    dW_ref = torch.einsum("bos,bis->oi", gpre_ref, h.float())
    for cl in (False, True):
        dpre = pre_b.clone().view(-1)
        dhb = torch.empty(B * C * S, device=dev, dtype=torch.bfloat16)
        dW = torch.zeros(C, C, device=dev)
        dcl = torch.zeros(B * S, CP, device=dev, dtype=torch.bfloat16)
        dcl.view(B, S, CP)[:, :, :C] = dout.permute(0, 2, 1)
        args_in = (None, dcl, CP) if cl else (dout.view(-1), None, CP)
        if tc:
            C_().bypass_bwd_tc(*args_in, dpre, h.view(-1), pad(W.t()), dhb, dW, B, C, S)
        else:
            C_().bypass_gelu_bwd(*args_in, dpre, W, dpre, dhb, B, C, S)
            for b in range(B):
                C_().kreduce_gemm(dpre.view(B, C, S)[b], S, C, h[b], S, C, S, dW)
        assert rel(dpre.view(B, C, S), gpre_ref) < 8e-3
        assert rel(dhb.view(B, C, S), dhb_ref) < 1e-2
        assert rel(dW, dW_ref) < 1e-2, (tc, cl, rel(dW, dW_ref))


# ------------------------------------------------------------------------------------------ spectral mix
@pytest.mark.parametrize("B,C,Q", [(1, 20, 5000), (3, 8, 777)])
def test_spectral_mix_forward_backward(B, C, Q):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(2)
    x = bf(torch.randn(B, C, Q, 2, device=dev, generator=g))
    w = torch.randn(C, C, Q, 2, device=dev, generator=g) / C
    xc, wc = torch.view_as_complex(x.float().contiguous()), torch.view_as_complex(w.contiguous())
    y = torch.empty_like(x)
    C_().spectral_mix_fwd(x.view(-1), w, y.view(-1), B, C, Q)
    yref = torch.einsum("biq,ioq->boq", xc, wc)
    assert rel(torch.view_as_complex(y.float().contiguous()), yref) < 6e-3
    dy = bf(torch.randn(B, C, Q, 2, device=dev, generator=g))
    dyc = torch.view_as_complex(dy.float().contiguous())
    dx, dw = torch.empty_like(x), torch.full_like(w, 7.0)
    C_().spectral_mix_bwd(x.view(-1), w, dy.view(-1), dx.view(-1), dw, False, B, C, Q)
    assert rel(torch.view_as_complex(dx.float().contiguous()), torch.einsum("boq,ioq->biq", dyc, wc.conj())) < 6e-3
    dwref = torch.einsum("biq,boq->ioq", xc.conj(), dyc)
    assert rel(torch.view_as_complex(dw.contiguous()), dwref) < 1e-5
    C_().spectral_mix_bwd(x.view(-1), w, dy.view(-1), dx.view(-1), dw, True, B, C, Q)      # accumulate
    assert rel(torch.view_as_complex(dw.contiguous()), 2 * dwref) < 1e-5


# ------------------------------------------------------------------------------------------ projection head
def test_head_forward_backward():
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(3)
    B, X, Y, Z, T, C, H, CP = 2, 4, 3, 8, 4, 20, 128, 24
    npos = B * X * Y * T * Z
    hcl = torch.zeros(npos, CP, device=dev, dtype=torch.bfloat16)
    hcl[:, :C] = bf(torch.randn(npos, C, device=dev, generator=g))
    W3 = torch.randn(H, C, device=dev, generator=g) / math.sqrt(C)
    b3 = torch.randn(H, device=dev, generator=g) * 0.2
    w4b4 = torch.randn(H + 1, device=dev, generator=g) / math.sqrt(H)
    w3p = torch.zeros(H, 64, device=dev, dtype=torch.bfloat16); w3p[:, :C] = bf(W3)
    w3t = torch.zeros(32, H, device=dev, dtype=torch.bfloat16); w3t[:C] = bf(W3.t())
    out = torch.empty(B, 1, X, Y, Z, T, device=dev)
    R, SR = [Z, T, B * X * Y], [T, 1, Z * T]
    epi = [2, 1, 0, 3, *R, 1, *SR, 0, 1, 1, 0, 0, 0, 0, 1, 0]
    C_().dft_gemm(hcl, npos, C, CP, w3p, H, epi, [out.data_ptr()], None, 0, 0, b3, w4b4, 0.0)
    hin = hcl[:, :C].float().requires_grad_()
    W3r, b3r, w4r = bf(W3).float().requires_grad_(), b3.clone().requires_grad_(), w4b4.clone().requires_grad_()
    ref = F.gelu(hin @ W3r.t() + b3r) @ w4r[:H] + w4r[H]                     # rows in (b, x, y, t, z) order
    ref_pub = ref.view(B, X, Y, T, Z).permute(0, 1, 2, 4, 3).unsqueeze(1)
    assert rel(out, ref_pub) < 5e-3
    dy = torch.randn(B, 1, X, Y, Z, T, device=dev, generator=g)
    ref_pub.backward(dy)
    gcl = torch.empty(npos, CP, device=dev, dtype=torch.bfloat16)
    gW3, gb3, gW4, gb4 = (torch.zeros(H, C, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev),
                          torch.zeros(1, device=dev))
    C_().head_bwd(hcl, npos, C, CP, w3p, w3t, b3, w4b4[:H].contiguous(), dy.contiguous(), R, SR, gcl, gW3, gb3, gW4, gb4)
    assert rel(gcl[:, :C], hin.grad) < 1e-2
    assert (gcl[:, C:] == 0).all()
    assert rel(gW3, W3r.grad) < 1e-2 and rel(gb3, b3r.grad) < 1e-2
    assert rel(gW4, w4r.grad[:H]) < 5e-3 and rel(gb4, w4r.grad[H:]) < 1e-4


# ------------------------------------------------------------------------------------------ K-reduction GEMM
@pytest.mark.parametrize("Ma,Nb,K", [(20, 20, 128 * 1000 + 40), (128, 40, 70000), (7, 33, 4096)])
def test_kreduce_gemm(Ma, Nb, K):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(4)
    K8 = (K + 7) // 8 * 8
    A = bf(torch.randn(Ma, K8, device=dev, generator=g))
    Bm = bf(torch.randn(Nb, K8, device=dev, generator=g))
    D = torch.full((Ma, Nb), 3.0, device=dev)
    C_().kreduce_gemm(A, K8, Ma, Bm, K8, Nb, K, D)
    ref = 3.0 + A[:, :K].float() @ Bm[:, :K].float().t()
    assert rel(D, ref) < 2e-3


# ------------------------------------------------------------------------------------------ Adam
def test_adam_kernel_matches_torch():
    dev = "cuda"
    n = 100003
    p0 = torch.randn(n, device=dev)
    p, m, v = p0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    pt = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([pt], lr=3e-3, betas=(0.8, 0.95), eps=1e-7, weight_decay=1e-2)
    for step in range(1, 4):
        gr = torch.randn(n, device=dev)
        C_().adam_step(p, gr, m, v, 3e-3, 0.8, 0.95, 1e-7, 1e-2, step, 1.0)
        pt.grad = gr.clone()
        opt.step()
    assert torch.allclose(p, pt.detach(), atol=2e-6, rtol=1e-5)


def test_permute_u32_matches_torch_permute():
    """Strided 32-bit-word permutation used after the staged pencil transposes."""
    C = C_()
    dev = torch.device("cuda")
    a = torch.randn(3, 4, 5, 6, 2, device=dev).to(torch.bfloat16)          # words = (re, im) bf16 pairs
    want = a.permute(0, 2, 1, 3, 4).contiguous()
    out = torch.zeros_like(want)
    # dst[i0, i2, i1, i3] <- src[i0, i1, i2, i3]; digits innermost first, strides in words
    C.permute_u32(a.view(-1), out.view(-1), [6, 4, 5, 3], [1, 6 * 5, 6, 6 * 5 * 4], [1, 6, 6 * 4, 6 * 4 * 5])
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    # padded destination pitch: untouched words keep their old content
    out2 = torch.full((3, 5, 4, 8, 2), 7.0, device=dev, dtype=torch.bfloat16)
    C.permute_u32(a.view(-1), out2.view(-1), [6, 4, 5, 3], [1, 6 * 5, 6, 6 * 5 * 4], [1, 8, 8 * 4, 8 * 4 * 5])
    torch.cuda.synchronize()
    assert torch.equal(out2[..., :6, :], want) and bool((out2[..., 6:, :] == 7.0).all())
    # 16-byte vector path (inner run of 8 words), 6 digits like the T1 permutation, and an odd inner run (scalar path)
    for inner in (8, 5):
        b = torch.randn(2, 3, 2, 4, 3, inner, 2, device=dev).to(torch.bfloat16)
        wantb = b.permute(0, 4, 2, 1, 3, 5, 6).contiguous()
        outb = torch.zeros_like(wantb)
        sz = list(b.shape[:6])                      # src dims [n0..n5], n5 innermost
        sst = [1] * 6
        for i in range(4, -1, -1):
            sst[i] = sst[i + 1] * sz[i + 1]
        perm = [0, 4, 2, 1, 3, 5]                   # dst dim k is src dim perm[k]
        dsz = [sz[k] for k in perm]
        dst_ = [1] * 6
        for i in range(4, -1, -1):
            dst_[i] = dst_[i + 1] * dsz[i + 1]
        # digits innermost first, walking dst
        size = [dsz[k] for k in range(5, -1, -1)]
        dstr = [dst_[k] for k in range(5, -1, -1)]
        sstr = [sst[perm[k]] for k in range(5, -1, -1)]
        C.permute_u32(b.view(-1), outb.view(-1), size, sstr, dstr)
        torch.cuda.synchronize()
        assert torch.equal(outb, wantb), inner


# ------------------------------------------------------------------------------------------ losses (csrc/loss.cu)
@pytest.mark.parametrize("shape", [(2, 1, 12, 10, 16, 7), (1, 1, 33, 5, 9), (3, 2, 1031)])
def test_native_losses_match_the_autograd_formulation(shape):
    import dfno_b200 as d
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(3)
    P = d.Partition([0], [1] * len(shape))
    y = torch.randn(*shape, device=dev, generator=g)
    yh = (y + 0.3 * torch.randn(*shape, device=dev, generator=g)).requires_grad_()
    yh64 = yh.detach().double().requires_grad_()
    B = shape[0]
    for crit, ref in ((d.DistributedRelativeLpLoss(P), lambda a, b: ((a - b).reshape(B, -1).norm(dim=1)
                                                                       / b.reshape(B, -1).norm(dim=1)).mean()),
                      (d.DistributedMSELoss(P), lambda a, b: ((a - b) ** 2).mean())):
        assert crit.local
        yh.grad = None; yh64.grad = None
        out = crit(yh, y)
        out.backward()
        want = ref(yh64, y.double())
        want.backward()
        assert abs(float(out) - float(want)) <= 2e-6 * abs(float(want))
        assert rel(yh.grad, yh64.grad) < 1e-5
    # non-contiguous / half-precision inputs keep the portable formulation
    out = d.DistributedRelativeLpLoss(P)(yh.to(torch.bfloat16), y.to(torch.bfloat16))
    assert torch.isfinite(out)
