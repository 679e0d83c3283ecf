"""5 <= Cin <= 16 input channels: the many-channel lift kernels against float64, and the fused engine with many input
fields against the float64 portable backend (H100 only).

Kernel bounds are those of test_kernel_widths_gpu.py / test_wide_widths_gpu.py; engine bounds those of
test_wide_widths_gpu.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from dfno_b200.models.fused import LIFT_MAX_W, SUPPORTED_WIDTHS, WIDE_WIDTHS

pytestmark = pytest.mark.gpu

DEV = "cuda"
WIDTHS = SUPPORTED_WIDTHS + WIDE_WIDTHS


def C_():
    from dfno_b200.ops import build
    return build.load()


def _f64(t):
    return t.detach().to(torch.float64)


def rel(got, want):
    got, want = _f64(got), _f64(want)
    return float((got - want).norm() / want.norm().clamp_min(1e-300))


def entry(got, want):
    got, want = _f64(got), _f64(want)
    return float(((got - want).abs() / (want.abs() + want.abs().pow(2).mean().sqrt())).max())


def worst(got, want):
    got, want = _f64(got), _f64(want)
    return float((got - want).abs().max() / want.pow(2).mean().sqrt().clamp_min(1e-300))


def _tin_limit(C, Cin, T=12):
    """largest Tin <= 64 whose lift weights fit kLiftMaxW at T output steps"""
    return min(64, (LIFT_MAX_W - 2 * (C * Cin + C) - T) // T)


def _lift_case(C, Cin, Tin, xdt, seed, shape=(2, 3, 4, 16)):
    B, X, Y, Z = shape
    T = 12
    assert T * Tin + T + 2 * (C * Cin + C) <= LIFT_MAX_W
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, Cin, X, Y, Z, Tin, device=DEV, generator=g).to(xdt)
    W1 = torch.randn(T, Tin, device=DEV, generator=g) / math.sqrt(Tin)
    b1 = torch.randn(T, device=DEV, generator=g) * 0.3
    W2 = torch.randn(C, Cin, device=DEV, generator=g) / math.sqrt(Cin)
    b2 = torch.randn(C, device=DEV, generator=g) * 0.3
    dh = torch.randn(B, C, X, Y, T, Z, device=DEV, generator=g).to(torch.bfloat16)
    return dict(x=x, params=(W1, b1, W2, b2), dh=dh, dims=[B, Cin, Tin, C, T, X, Y, Z])


def _lift_check(case, with_dx, x_kernel=None):
    """runs lift_fwd / lift_bwd on x_kernel (default: the case's x) and checks them against float64 on the case's x;
    returns the names of the failed checks and the errors"""
    x, (W1, b1, W2, b2), dh = case["x"], case["params"], case["dh"]
    B, Cin, Tin, C, T, X, Y, Z = case["dims"]
    xk = x if x_kernel is None else x_kernel
    h = torch.full((B * C * X * Y * T * Z,), 9.0, device=DEV, dtype=torch.bfloat16)
    C_().lift_fwd(xk, W1, b1, W2, b2, h, case["dims"])
    xr = x.double().requires_grad_()
    params = [p.double().requires_grad_() for p in (W1, b1, W2, b2)]
    a1 = F.gelu(torch.einsum("ti,bcxyzi->bcxyzt", params[0], xr) + params[1])
    ref = F.gelu(torch.einsum("oc,bcxyzt->boxyzt", params[2], a1) + params[3].view(1, C, 1, 1, 1, 1))
    ref_eng = ref.permute(0, 1, 2, 3, 5, 4)
    got = h.view(B, C, X, Y, T, Z)
    m = {"h": rel(got, ref_eng), "h_entry": entry(got, ref_eng)}
    ref_eng.backward(dh.double())
    grads = [torch.zeros_like(p) for p in (W1, b1, W2, b2)]
    dx = torch.full(x.shape, float("nan"), device=DEV) if with_dx else None
    C_().lift_bwd(xk, W1, b1, W2, b2, dh.view(-1), *grads, case["dims"], dx)
    for name, gr, p in zip(("W1", "b1", "W2", "b2"), grads, params):
        m["d" + name] = rel(gr, p.grad)
    bad = [k for k in ("h",) if not m[k] < 6e-3] + (["h_entry"] if not m["h_entry"] < 2e-2 else [])
    bad += [k for k in ("dW1", "db1", "dW2", "db2") if not m[k] < 1e-2]
    if with_dx:
        m["dx"], m["dx_worst"] = rel(dx, xr.grad), worst(dx, xr.grad)
        if not bool(torch.isfinite(dx).all()):
            bad.append("dx_finite")
        bad += [k for k, lim in (("dx", 1e-2), ("dx_worst", 0.2)) if not m[k] < lim]
    return bad, m


@pytest.mark.parametrize("with_dx", [False, True], ids=["no_dx", "dx"])
@pytest.mark.parametrize("xdt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("tin", ["1", "5", "limit"])
@pytest.mark.parametrize("Cin", [5, 8, 13, 16])
@pytest.mark.parametrize("C", WIDTHS)
def test_lift_many_inputs(C, Cin, tin, xdt, with_dx):
    Tin = {"1": 1, "5": 5, "limit": _tin_limit(C, Cin)}[tin]
    case = _lift_case(C, Cin, Tin, xdt, seed=1000 * Cin + 10 * C + Tin)
    bad, m = _lift_check(case, with_dx)
    assert not bad, (bad, m)


@pytest.mark.parametrize("Tin", [1, 5])
@pytest.mark.parametrize("C", [20, 64])
def test_lift_many_checker_sees_swapped_input_channels(C, Tin):
    """The kernels see x with input channels 2 and 11 swapped; the checks against the clean reference must fail, so a
    channel-stride error in the kernels cannot pass them"""
    case = _lift_case(C, 13, Tin, torch.float32, seed=77 + C + Tin)
    xs = case["x"].clone()
    xs[:, [2, 11]] = xs[:, [11, 2]]
    bad, m = _lift_check(case, True, x_kernel=xs)
    print(f"C={C} Tin={Tin} swapped input channels: failed={bad}")
    assert "h" in bad and "dW2" in bad and "dx" in bad, (bad, m)


@pytest.mark.parametrize("with_dx", [False, True], ids=["no_dx", "dx"])
@pytest.mark.parametrize("Tin", [1, 5])
@pytest.mark.parametrize("Cin", [8, 16])
def test_lift_many_inputs_several_items_per_warp(Cin, Tin, with_dx):
    """B = 1, 32 x 32 x 64: 8192 items, more than the grid's warps (4224 on 132 SMs), so each warp runs its
    grid-stride loop at least twice: the dW2 / db2 sums carried across items, the per-item x slice, dx reset and t = 0
    stores, and the a1 / dv tiles reused for a second item"""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    assert 32 * 32 * 64 // 8 > 32 * nsm
    case = _lift_case(20, Cin, Tin, torch.float32, seed=500 + Cin + Tin, shape=(1, 32, 32, 64))
    bad, m = _lift_check(case, with_dx)
    assert not bad, (bad, m)


# ------------------------------------------------------------------------------------------ the engine
FRO, POS = 9e-2, 0.95            # as test_wide_widths_gpu.py: dx / output vs float64
GRAD = 5e-2                      # pointwise weight gradients vs float64 (relative Frobenius)

# (id, public in_shape, T, C, modes, fused_pw)
ENGINE = [
    ("3d_cin16", [1, 16, 16, 16, 16, 1], 8, 20, (4, 4, 4, 3), True),
    ("2d_time_cin8_tin10", [2, 8, 32, 32, 10], 16, 20, (4, 4, 4), True),
    ("t30_cin5", [1, 5, 12, 12, 16, 2], 30, 16, (4, 4, 4, 8), True),
    ("round1_cin12", [1, 12, 16, 16, 80, 1], 8, 20, (4, 4, 34, 3), False),
    ("3d_cin16_w64", [1, 16, 16, 16, 16, 3], 12, 64, (4, 4, 4, 3), True),
]
ENG = {c[0]: c for c in ENGINE}


def _models(case, seed=0, blocks=2):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    name, in_shape, T, C, modes, fused_pw = case
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    dev = torch.device("cuda")
    torch.manual_seed(seed)
    ref = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev, dtype=torch.float64,
                           backend="torch", input_grad=True)
    fused = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev, input_grad=True)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    assert fused.fused_pw == fused_pw
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
def test_engine_many_inputs_matches_float64(case):
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


def test_engine_many_inputs_trainer_cuda_graph_and_inference():
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    in_shape = [1, 8, 16, 16, 16, 1]
    torch.manual_seed(0)
    net = d.DistributedFNO(P_x, in_shape, 8, 20, (4, 4, 4, 3), num_blocks=2, device=dev, dtype=torch.bfloat16)
    assert isinstance(net, d.FusedDistributedFNO)
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


def test_engine_many_inputs_checkpoint_round_trip():
    """fused -> canonical state -> portable -> canonical state -> fused at Cin = 16: the same outputs"""
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, in_shape, T, C, modes, _ = ENG["3d_cin16"]
    _, P_x, _ = d.create_standard_partitions([1] * 6)
    dev = torch.device("cuda")
    a = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=2, device=dev, init_seed=5)
    port = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=2, device=dev, dtype=torch.float32,
                            backend="torch")
    d.load_global_state(port, d.gather_global_state(a, to_all=True), strict=False)
    b = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=2, device=dev, init_seed=6)
    d.load_global_state(b, d.gather_global_state(port, to_all=True), strict=False)
    x, _ = _inputs(ENG["3d_cin16"], 3)
    with torch.no_grad():
        ya, yb, yp = a(x), b(x), port(x)
    assert torch.equal(ya, yb)
    f, p = _errors(ya, yp)
    assert f < 2e-2 and p < 0.2, (f, p)
