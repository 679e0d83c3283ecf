"""Widths 48 and 64 (WIDE_WIDTHS, round-2 route only) through every kernel that depends on the width, and the fused
engine at those widths against the float64 portable backend (H100 only).

Kernel bounds are those of test_kernel_widths_gpu.py / test_head_gpu.py; engine bounds those of
test_fused_input_grad_gpu.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from dfno_b200.models.fused import LIFT_MAX_W, WIDE_WIDTHS

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 128


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
    got, want = _f64(got), _f64(want)
    return float(((got - want).abs() / (want.abs() + want.abs().pow(2).mean().sqrt())).max())


def worst(got, want):
    got, want = _f64(got), _f64(want)
    return float((got - want).abs().max() / want.pow(2).mean().sqrt().clamp_min(1e-300))


def gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------ spectral mix
@pytest.mark.parametrize("dw", [True, False], ids=["dw", "frozen"])
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("C", WIDE_WIDTHS)
def test_spectral_mix_wide(C, accumulate, dw):
    """B = 2, Q = 1037 (not a multiple of 64); the frozen backward (no dw) is the kDw = false kernel"""
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
    dx, dwt = torch.full_like(x, 9.0), dw0.clone()
    C_().spectral_mix_bwd(x.view(-1), w, dy.view(-1), dx.view(-1), dwt if dw else None, accumulate, B, C, Q)
    dxref = torch.einsum("boq,ioq->biq", dyc, wc.conj())
    dxc = torch.view_as_complex(dx.double())
    assert rel(dxc, dxref) < 5e-3 and entry(dxc, dxref) < 2e-2, (rel(dxc, dxref), entry(dxc, dxref))
    if not dw:
        assert torch.equal(dwt, dw0)
        return
    dwref = torch.einsum("biq,boq->ioq", xc.conj(), dyc)
    if accumulate:
        dwref = dwref + torch.view_as_complex(dw0.double())
    dwc = torch.view_as_complex(dwt.double())
    assert rel(dwc, dwref) < 1e-6 and entry(dwc, dwref) < 1e-5, (rel(dwc, dwref), entry(dwc, dwref))


# ------------------------------------------------------------------------------------------ lift
@pytest.mark.parametrize("with_dx", [False, True], ids=["no_dx", "dx"])
@pytest.mark.parametrize("xdt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("Tin", [1, 5, 64])
@pytest.mark.parametrize("Cin", [1, 2, 3, 4])
@pytest.mark.parametrize("C", WIDE_WIDTHS)
def test_lift_wide(C, Cin, Tin, xdt, with_dx):
    B, X, Y, Z = 2, 3, 4, 16
    T = 12 if Tin < 64 else (LIFT_MAX_W - 2 * (C * Cin + C)) // (Tin + 1) // 2 * 2
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
    xr = x.double().requires_grad_()
    params = [p.double().requires_grad_() for p in (W1, b1, W2, b2)]
    a1 = F.gelu(torch.einsum("ti,bcxyzi->bcxyzt", params[0], xr) + params[1])
    ref = F.gelu(torch.einsum("oc,bcxyzt->boxyzt", params[2], a1) + params[3].view(1, C, 1, 1, 1, 1))
    ref_eng = ref.permute(0, 1, 2, 3, 5, 4)
    got = h.view(B, C, X, Y, T, Z)
    assert rel(got, ref_eng) < 6e-3 and entry(got, ref_eng) < 2e-2, (rel(got, ref_eng), entry(got, ref_eng))
    dh = bf(torch.randn(B, C, X, Y, T, Z, device=DEV, generator=g))
    ref_eng.backward(dh.double())
    grads = [torch.zeros_like(p) for p in (W1, b1, W2, b2)]
    dx = torch.full(x.shape, float("nan"), device=DEV) if with_dx else None
    C_().lift_bwd(x, W1, b1, W2, b2, dh.view(-1), *grads, dims, dx)
    for name, got, p in zip(("W1", "b1", "W2", "b2"), grads, params):
        assert rel(got, p.grad) < 1e-2, (name, rel(got, p.grad))
    if with_dx:
        assert bool(torch.isfinite(dx).all())
        assert rel(dx, xr.grad) < 1e-2 and worst(dx, xr.grad) < 0.2, (rel(dx, xr.grad), worst(dx, xr.grad))


# ------------------------------------------------------------------------------------------ spectral_out, dpre_dw
@pytest.mark.parametrize("mode", ["fwd", "fwd_nopre", "adj"])
@pytest.mark.parametrize("C", WIDE_WIDTHS)
def test_spectral_out_wide(C, mode):
    """R = 2 lines per tile (RC = 96 / 128 rows); L = 97 leaves a partial last tile"""
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
    save = mode == "fwd"
    C_().spectral_out(U, h, pad_operator(Fop), W, adj, pre if save else None, out, B, C, L, Z, K1, not adj, save)
    torch.cuda.synchronize()
    Wr = bf(W).double()
    spec = U.double() @ bf(Fop).double().t()
    mix = torch.einsum("oi,bilz->bolz", Wr.t() if adj else Wr, h.double().view(B, C, L, Z)).reshape(B * C, L, Z)
    ref_pre = spec + mix
    if adj:
        assert rel(out, ref_pre) < 6e-3 and entry(out, ref_pre) < 2e-2, (rel(out, ref_pre), entry(out, ref_pre))
    else:
        assert rel(out, F.gelu(ref_pre)) < 8e-3 and entry(out, F.gelu(ref_pre)) < 2e-2
        if save:
            assert rel(pre, ref_pre) < 6e-3 and entry(pre, ref_pre) < 2e-2


@pytest.mark.parametrize("C", WIDE_WIDTHS)
def test_dpre_dw_wide(C):
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


# ------------------------------------------------------------------------------------------ channel-major head
NORM = {"out": 5e-3, "g": 1e-2, "dW3": 1e-2, "db3": 1e-2, "dW4": 6e-3, "db4": 1e-3}
WORST = {"out": 0.1, "g": 0.1, "dW3": 0.1, "db3": 0.1, "dW4": 0.1}


def _head_case(B, C, X, Y, Z, T, seed):
    g = gen(seed)
    S = X * Y * Z * T
    return dict(B=B, C=C, dims=(X, Y, Z, T), S=S, gen=g,
                h=bf(torch.randn(B * C, S, device=DEV, generator=g)),
                W3=bf(torch.randn(H, C, device=DEV, generator=g) / math.sqrt(C)),
                b3=bf(torch.randn(H, device=DEV, generator=g) * 0.2),
                w4b4=torch.randn(H + 1, device=DEV, generator=g) / math.sqrt(H))


def _head_operands(W3, b3, C):
    """as FusedDistributedFNO._head_operators_cm: W3aug [H, 64] ([H, 128] when C + 1 > 64), W3^T fp16"""
    w3a = torch.zeros(H, 64 if C + 1 <= 64 else 128, device=DEV, dtype=torch.bfloat16)
    w3a[:, :C] = W3
    w3a[:, C] = b3
    w3t = torch.zeros((C + 1 + 15) // 16 * 16, H, device=DEV, dtype=torch.float16)
    w3t[:C] = W3.float().t().to(torch.float16)
    return w3a, w3t


def _head_check(case, dscale, W3_kernel=None):
    B, C, S = case["B"], case["C"], case["S"]
    X, Y, Z, T = case["dims"]
    dy_pub = torch.randn(B, 1, X, Y, Z, T, device=DEV, generator=case["gen"]) * dscale
    rows = dy_pub.squeeze(1).permute(0, 1, 2, 4, 3).reshape(B * S).double()
    hin = case["h"].double().view(B, C, S).permute(0, 2, 1).reshape(B * S, C)
    W3, b3 = case["W3"].double(), case["b3"].double()
    w4, b4 = case["w4b4"][:H].double(), case["w4b4"][H].double()
    pre = hin @ W3.t() + b3
    a = 0.5 * pre * (1 + torch.erf(pre / math.sqrt(2)))
    dpre = (rows[:, None] * w4[None, :]) * gelu_grad(pre)
    ref = dict(out=a @ w4 + b4, dW4=a.t() @ rows, db4=rows.sum().reshape(1), dW3=dpre.t() @ hin, db3=dpre.sum(0),
               g=(dpre @ W3).view(B, S, C).permute(0, 2, 1).reshape(B * C, S))
    del pre, a, dpre
    w3a, w3t = _head_operands(case["W3"] if W3_kernel is None else W3_kernel, case["b3"], C)
    R, SR = [Z, T, B * X * Y], [T, 1, Z * T]
    out = torch.full((B, 1, X, Y, Z, T), float("nan"), device=DEV)
    C_().head_fwd(case["h"], w3a, case["w4b4"], out, B, C, S, R, SR)
    g = torch.full((B * C, S), float("nan"), device=DEV, dtype=torch.bfloat16)
    init = {k: torch.randn(*shape, device=DEV, generator=case["gen"]) * float(ref[k].abs().max())
            for k, shape in (("dW3", (H, C)), ("db3", (H,)), ("dW4", (H,)), ("db4", (1,)))}
    grads = {k: v.clone() for k, v in init.items()}
    ws = torch.zeros(1, device=DEV, dtype=torch.int32)
    C_().head_bwd2(case["h"], w3a, w3t, case["w4b4"][:H].contiguous(), dy_pub.contiguous(), ws, g,
                   grads["dW3"], grads["db3"], grads["dW4"], grads["db4"], B, C, S, R, SR)
    torch.cuda.synchronize()
    got = {"out": out.squeeze(1).permute(0, 1, 2, 4, 3).reshape(B * S), "g": g}
    got.update({k: grads[k] - init[k] for k in init})
    m = {k: rel(got[k], ref[k]) for k in NORM}
    m.update({k + "_worst": worst(got[k], ref[k]) for k in WORST})
    bad = [k for k in ("out", "g") if not bool(torch.isfinite(got[k]).all())]
    bad += [k for k in NORM if not m[k] < NORM[k]] + [k + "_worst" for k in WORST if not m[k + "_worst"] < WORST[k]]
    return m, bad


@pytest.mark.parametrize("dscale", [3e-7, 1.0])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("C", WIDE_WIDTHS)
def test_head_wide(C, B, dscale):
    """S = 720: five full tiles and a partial one of 80 positions; dout at a loss-gradient scale and at O(1)"""
    m, bad = _head_check(_head_case(B, C, 3, 5, 8, 6, seed=1000 + 10 * C + B), dscale)
    print(f"C={C} B={B} dout~{dscale:g}: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("C", WIDE_WIDTHS)
def test_head_wide_many_tiles(C):
    """S = 244800 with B = 2: 3826 tiles, so the TMA ring (2 stages at width 64) wraps many times"""
    m, bad = _head_check(_head_case(2, C, 17, 15, 32, 30, seed=2000 + C), 3e-7)
    print(f"C={C} many tiles: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("C", WIDE_WIDTHS)
def test_head_wide_checker_sees_swapped_w3_columns(C):
    """The kernels see W3 with two channel columns swapped (one of them in the second W3aug block at width 64); the
    checks against the clean reference must fail, dW3 among them"""
    case = _head_case(1, C, 3, 5, 8, 6, seed=4000 + C)
    a, b = 3, C - 2
    W3_bad = case["W3"].clone()
    W3_bad[:, [a, b]] = W3_bad[:, [b, a]]
    m, bad = _head_check(case, 3e-7, W3_kernel=W3_bad)
    print(f"C={C} swapped W3 columns {a}, {b}: failed={bad}")
    assert "dW3" in bad or "dW3_worst" in bad, (bad, m)
    assert "out" in bad or "out_worst" in bad, (bad, m)


# ------------------------------------------------------------------------------------------ the engine
FRO, POS = 9e-2, 0.95            # as test_fused_input_grad_gpu.py: dx / output vs float64
GRAD = 5e-2                      # pointwise weight gradients vs float64 (relative Frobenius)

# (id, public in_shape, T, C, modes)
ENGINE = [
    ("3d_w48", [1, 1, 16, 16, 16, 1], 8, 48, (4, 4, 4, 3)),
    ("3d_w64", [2, 2, 12, 8, 24, 3], 12, 64, (2, 4, 6, 7)),
    ("t30_w64", [1, 2, 12, 12, 16, 1], 30, 64, (4, 4, 4, 8)),
    ("2d_time_w48", [2, 1, 32, 32, 10], 16, 48, (4, 4, 4)),
    ("2d_time_w64", [1, 1, 32, 32, 10], 16, 64, (4, 4, 4)),
]
ENG = {c[0]: c for c in ENGINE}


def _models(case, seed=0, blocks=2):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    name, in_shape, T, C, modes = case
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    dev = torch.device("cuda")
    torch.manual_seed(seed)
    ref = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev, dtype=torch.float64,
                           backend="torch", input_grad=True)
    fused = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev, input_grad=True)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    assert fused.fused_pw
    return d, ref, fused


def _inputs(case, seed):
    g = torch.Generator(device="cuda").manual_seed(1000 + seed)
    x = torch.randn(*case[1], device="cuda", generator=g)
    oshape = list(case[1]); oshape[1] = 1; oshape[-1] = case[2]
    return x, torch.randn(*oshape, device="cuda", generator=g)


def _errors(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm()), float((a - b).abs().max() / b.pow(2).mean().sqrt())


@pytest.mark.parametrize("case", ENGINE, ids=[c[0] for c in ENGINE])
def test_engine_wide_matches_float64(case):
    """forward, dx and the pointwise weight gradients; then the frozen (dx-only) backward gives the same dx"""
    d, ref, fused = _models(case)
    x, w = _inputs(case, 0)
    xx = x.clone().requires_grad_()
    y = fused(xx)
    (y * w).sum().backward()
    xr = x.double().requires_grad_()
    yr = ref(xr)
    (yr * w.double()).sum().backward()
    f, p = _errors(y, yr)
    print(f"\n{case[0]} out fro={f:.3e} pos={p:.3e}")
    assert f < 2e-2 and p < 0.2, (f, p)
    f, p = _errors(xx.grad, xr.grad)
    print(f"{case[0]} dx fro={f:.3e} pos={p:.3e}")
    assert f < FRO and p < POS, (f, p)
    canon = fused.theta_to_canonical(fused.theta.grad.detach().cpu(), fused.engine_meta())
    refp = dict(ref.named_parameters())
    for name in ["linear1.W", "linear1.b", "linear2.W", "linear2.b", "linear3.W", "linear3.b", "linear4.W",
                 "linear4.b", "blocks.0.linear.W", "blocks.1.linear.W"]:
        got, want = canon[name].reshape(-1), refp[name].grad.detach().cpu().reshape(-1)
        e = rel(got, want)
        print(f"{case[0]} d{name} {e:.3e}")
        assert e < GRAD, (name, e)
    fused.theta.requires_grad_(False)
    xf = x.clone().requires_grad_()
    (fused(xf) * w).sum().backward()
    assert torch.equal(xf.grad, xx.grad)


def test_engine_wide_trainer_cuda_graph_and_inference():
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    in_shape = [1, 1, 16, 16, 16, 1]
    torch.manual_seed(0)
    net = d.DistributedFNO(P_x, in_shape, 8, 64, (4, 4, 4, 3), num_blocks=2, device=dev, dtype=torch.bfloat16)
    assert isinstance(net, d.FusedDistributedFNO) and net.width == 64
    opt = d.FusedAdam(net, lr=1e-3)
    crit = d.DistributedRelativeLpLoss(P_x, engine=net)
    tr = d.Trainer(net, crit, opt, device=dev, cuda_graph=True)
    x = torch.randn(*in_shape).pin_memory()
    y = torch.randn(1, 1, 16, 16, 16, 8).pin_memory()
    losses = [tr.step(x, y, next_batch=(x, y)) for _ in range(12)]
    print("losses", losses)
    assert tr._graph is not None
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0], losses
    sess = d.InferenceSession(net, device=dev, cuda_graph=True)
    xs = [torch.randn(*in_shape).pin_memory() for _ in range(2)]
    outs = [sess.run(v).clone() for v in xs]
    with torch.no_grad():
        for v, o in zip(xs, outs):
            want = net(v.to(dev)).cpu()
            assert torch.allclose(o, want, atol=1e-5, rtol=1e-4), float((o - want).abs().max())


def test_engine_wide_checkpoint_round_trip():
    """fused -> canonical state -> portable -> canonical state -> fused at width 64: the same outputs"""
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    case = ENG["3d_w64"]
    _, in_shape, T, C, modes = case
    _, P_x, _ = d.create_standard_partitions([1] * 6)
    dev = torch.device("cuda")
    a = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=2, device=dev, init_seed=5)
    port = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=2, device=dev, dtype=torch.float32,
                            backend="torch")
    d.load_global_state(port, d.gather_global_state(a, to_all=True), strict=False)
    b = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=2, device=dev, init_seed=6)
    d.load_global_state(b, d.gather_global_state(port, to_all=True), strict=False)
    x, _ = _inputs(case, 3)
    with torch.no_grad():
        ya, yb, yp = a(x), b(x), port(x)
    assert torch.equal(ya, yb)
    f, p = _errors(ya, yp)
    assert f < 2e-2 and p < 0.2, (f, p)
