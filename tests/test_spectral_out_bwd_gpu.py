"""The adjoint spectral_out with the backward's pointwise tail folded in (H100 only).

``spectral_out(..., pre_prev=, h_dw=, dW=)`` forms, besides the adjoint accumulator g = U F'^T + W^T dpre_k,
* dpre_{k-1} = g * gelu'(pre_{k-1}) over pre_{k-1} (instead of storing g), and/or
* dW_k += sum dpre_k h_k^T.
Checked against the composition of the existing kernels on the same inputs (plain adjoint, then dpre_dw): dpre and g
bitwise, dW to fp32 reordering and against float64; that nothing outside the outputs is written; and the engine's
gradients with the fold on and off, and against the float64 portable backend, at 1 .. 4 blocks.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

VARIANTS = ["dpre", "dpre_dw", "dw"]       # top block, middle blocks, block 0


def C_():
    from dfno_b200.ops import build
    return build.load()


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _inputs(B, C, L, Z, K1, seed=0):
    from dfno_b200.ops.gemm import pad_operator
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    bf = torch.bfloat16
    U = (torch.randn(B * C, L, K1, device=dev, generator=g) * 1e-3).to(bf)
    dpre = (torch.randn(B * C, L, Z, device=dev, generator=g) * 1e-3).to(bf)     # dpre_k: the MMA2 operand
    pre = (torch.randn(B * C, L, Z, device=dev, generator=g) * 1.5).to(bf)       # pre_{k-1}
    h = torch.randn(B * C, L, Z, device=dev, generator=g).to(bf)                 # h_k
    Fop = pad_operator(torch.randn(Z, K1, device=dev, generator=g) / math.sqrt(K1))
    W = torch.randn(C, C, device=dev, generator=g) / math.sqrt(C)
    return U, dpre, pre, h, Fop, W


def _reference(U, dpre, pre, h, Fop, W, B, C, L, Z, K1):
    """The two-kernel path: plain adjoint (g), then dpre_dw (dpre_{k-1} over a copy of pre_{k-1}).  Where the plain
    adjoint's 128-column tiles do not fit shared memory (two U blocks at Z > 64), g comes from the block-0 variant,
    checked against an fp32 reference here, so the other two variants are still held bitwise to dpre_dw."""
    g = torch.empty_like(dpre)
    try:
        C_().spectral_out(U, dpre, Fop, W, True, None, g, B, C, L, Z, K1, False, False)
    except RuntimeError as e:
        if "does not fit" not in str(e):
            raise
        C_().spectral_out(U, dpre, Fop, W, True, None, g, B, C, L, Z, K1, False, False, None, h,
                          torch.zeros(C, C, device="cuda"))
        spec = U.float() @ Fop[:Z, :K1].float().t()
        mix = torch.einsum("oi,bolz->bilz", W.to(torch.bfloat16).float(), dpre.float().view(B, C, L, Z))
        assert _rel(g, spec + mix.reshape(B * C, L, Z)) < 6e-3
    dp = pre.clone()
    C_().dpre_dw(g, dp, torch.zeros_like(pre), torch.zeros(C, C, device="cuda"), B, C, L, Z)
    return g, dp


# (B, C, L, Z, K1): every width class (R = 32 .. 2, RC = 96 .. 128), one to four 64-column blocks with a partial
# last block (Z = 96), one and two U blocks, L not a multiple of R, B > 1
SHAPES = [
    (1, 20, 301, 128, 24), (2, 20, 97, 96, 48), (1, 4, 77, 64, 24), (2, 8, 61, 256, 48), (1, 32, 50, 128, 128),
    (1, 48, 41, 96, 48), (2, 64, 33, 128, 24), (1, 12, 45, 256, 24), (1, 20, 39, 96, 128), (1, 64, 30, 256, 48),
]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("B,C,L,Z,K1", SHAPES)
def test_folded_adjoint_matches_the_two_kernels(B, C, L, Z, K1, variant):
    U, dpre, pre, h, Fop, W = _inputs(B, C, L, Z, K1)
    g_ref, dp_ref = _reference(U, dpre, pre, h, Fop, W, B, C, L, Z, K1)
    kd, kw = "dpre" in variant, "dw" in variant
    g = torch.full_like(dpre, float("nan"))
    pp = pre.clone()
    dW = torch.full((C, C), 0.5, device="cuda")                            # accumulates
    C_().spectral_out(U, dpre, Fop, W, True, None, g, B, C, L, Z, K1, False, False,
                      pp if kd else None, h if kw else None, dW if kw else None)
    torch.cuda.synchronize()
    if kd:
        assert torch.equal(pp, dp_ref)
        assert torch.isnan(g.float()).all()                                 # g is not stored
    else:
        assert torch.equal(g, g_ref) and torch.equal(pp, pre)
    if kw:
        ref64 = torch.einsum("bolz,bilz->oi", dpre.double().view(B, C, L, Z), h.double().view(B, C, L, Z)) + 0.5
        ref32 = torch.einsum("bos,bis->oi", dpre.float().view(B, C, L * Z), h.float().view(B, C, L * Z)) + 0.5
        assert _rel(dW, ref64) < 1e-4, _rel(dW, ref64)
        assert _rel(dW, ref32) < 1e-4, _rel(dW, ref32)
    else:
        assert (dW == 0.5).all()


@pytest.mark.parametrize("variant", VARIANTS)
def test_folded_adjoint_writes_only_its_outputs(variant):
    """Every buffer sits between NaN guard bands; only pre_prev (dpre variants), g (dW-only variant) and dW change."""
    B, C, L, Z, K1 = 2, 20, 53, 96, 48
    U, dpre, pre, h, Fop, W = _inputs(B, C, L, Z, K1, seed=3)
    kd, kw = "dpre" in variant, "dw" in variant
    band = 4096

    def banded(t):
        flat = t.reshape(-1)
        buf = torch.full((flat.numel() + 2 * band,), float("nan"), device="cuda", dtype=t.dtype)
        buf[band:band + flat.numel()] = flat
        return buf, buf[band:band + flat.numel()].view(t.shape)
    bufs = {n: banded(t) for n, t in dict(U=U, dpre=dpre, pre=pre, h=h, W=W,
                                          g=torch.zeros_like(dpre), dW=torch.zeros(C, C, device="cuda")).items()}
    before = {n: b.clone() for n, (b, _) in bufs.items()}
    v = {n: t for n, (_, t) in bufs.items()}
    C_().spectral_out(v["U"], v["dpre"], Fop, v["W"], True, None, v["g"], B, C, L, Z, K1, False, False,
                      v["pre"] if kd else None, v["h"] if kw else None, v["dW"] if kw else None)
    torch.cuda.synchronize()
    written = {"pre"} if kd else {"g"}
    if kw:
        written.add("dW")
    for n, (b, t) in bufs.items():
        same = torch.equal(b.view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32),
                           before[n].view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32))
        if n in written:
            n_body = t.numel()
            assert torch.isnan(b[:band].float()).all() and torch.isnan(b[band + n_body:].float()).all(), n
            assert not same, n
        else:
            assert same, n


def _engine(in_shape, nt, width, modes, blocks, padding=None, seed=0):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    torch.manual_seed(seed)
    dev = torch.device("cuda")
    kw = dict(padding=padding) if padding else {}
    ref = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev, dtype=torch.float64,
                           backend="torch", input_grad=True, **kw)
    fused = FusedDistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev, input_grad=True, **kw)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    return d, ref, fused


def _grads(fused, x, t, fold):
    fused.fold_bwd = fold
    fused.theta.grad = None
    xx = x.clone().requires_grad_()
    ((fused(xx) - t) ** 2).mean().backward()
    return fused.theta.grad.clone(), xx.grad.clone()


CASES = [
    ([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), None),
    ([2, 2, 12, 8, 24, 3], 12, 20, (2, 4, 6, 7), None),
    ([1, 2, 12, 8, 24, 3], 12, 20, (2, 4, 6, 7), (4, 0, 8, 4)),        # padded plan
]


@pytest.mark.parametrize("blocks", [1, 2, 3, 4])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_engine_gradients_with_the_fold(case, blocks):
    in_shape, nt, width, modes, padding = CASES[case]
    d, ref, fused = _engine(in_shape, nt, width, modes, blocks, padding)
    assert fused.fused_pw and fused.fold_bwd
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(*in_shape, device="cuda", generator=g)
    oshape = list(in_shape); oshape[1] = 1; oshape[-1] = nt
    t = torch.randn(*oshape, device="cuda", generator=g)
    g_off, dx_off = _grads(fused, x, t, False)
    g_on, dx_on = _grads(fused, x, t, True)
    # dpre and g are bitwise those of the two-kernel path, so dx is too; the bypass weight gradients differ by the
    # fp32 summation order only, and the rest of theta only by the order of their atomics
    assert torch.equal(dx_on, dx_off)
    for name, (off, shape) in fused.plan.segments.items():
        n = int(torch.tensor(shape).prod())
        assert _rel(g_on[off:off + n], g_off[off:off + n]) < 1e-4, name
    # against float64, with the loss and tolerances of the engine's other parity tests (test_fused_gpu, test_padding_gpu)
    xx = x.double().requires_grad_()
    ((ref(xx) - t.double()) ** 2).mean().backward()
    assert _rel(dx_on, xx.grad) < 3e-2
    for p in ref.parameters():
        p.data = p.grad if p.grad is not None else torch.zeros_like(p.data)
    G = d.gather_global_state(ref, to_all=True)
    for name, (off, shape) in fused.plan.segments.items():
        got = g_on[off:off + int(torch.tensor(shape).prod())].view(shape).cpu()
        if name.endswith(".spectral"):
            Gs = G[name] if G[name].dim() == 6 else G[name].unsqueeze(2)
            want = torch.view_as_real(Gs.permute(0, 1, 4, 5, 3, 2).contiguous()).reshape(shape)
        else:
            want = G[name].reshape(shape)
        assert _rel(got, want) < 3e-2, (name, _rel(got, want))


def test_frozen_backward_with_the_fold():
    """theta frozen: dx is bitwise the dx of the two-kernel path and theta.grad is left alone."""
    in_shape, nt, width, modes, padding = CASES[0]
    d, ref, fused = _engine(in_shape, nt, width, modes, 3, padding)
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(*in_shape, device="cuda", generator=g)
    w = torch.randn(1, 1, 16, 16, 16, nt, device="cuda", generator=g)
    fused.theta.requires_grad_(False)
    dx = {}
    for fold in (False, True):
        fused.fold_bwd = fold
        xx = x.clone().requires_grad_()
        (dx[fold],) = torch.autograd.grad((fused(xx) * w).sum(), xx)
        assert fused.theta.grad is None
    assert torch.equal(dx[True], dx[False])
