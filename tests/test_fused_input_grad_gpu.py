"""Input gradients (dL/dx) of the fused engine built with ``input_grad=True``, against float64 (H100 only).

The float64 portable backend gets the engine's weights, and both differentiate the same scalar ``sum(y * w)`` with a
fixed random cotangent ``w``.  A case passes when dx meets two bounds: its relative Frobenius error, and its worst
single position over the reference's rms.  The second bound catches a local error that the norm averages away.  Also
checked:
* the checker rejects a dx with one input channel zeroed, and a reference with one t term of the lift dropped;
* dx does not change theta.grad, and a frozen theta (``requires_grad_(False)``) keeps theta.grad as it was while
  dx stays bitwise equal to the trainable-theta dx;
* a double backward (``create_graph=True``) raises, and so does a second backward through one forward
  (``retain_graph=True``), which would otherwise read gradients where the saved pre-activations were;
* gradient descent on the input of a frozen engine (inversion) tracks the same descent on the fp32 portable backend.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

# Bounds, measured on an H100 80GB HBM3 over seeds 0, 1, 2 and set at about 4x the worst value seen (in brackets).
# The worst case is large_mz (legacy route, tensor-core bypass) at seed 1; every other case stays at or below
# 1.9e-2 / 0.11 (legacy_t30: 1.3e-2 / 0.107).
FRO = 9e-2          # relative Frobenius error of dx                                      [2.16e-2]
POS = 0.95          # worst |dx - ref| at one position over the rms of ref                  [0.232]

# (id, public in_shape, T, C, modes, expected fused_pw)
CASES = [
    ("cin1_tin1", [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), True),
    ("cin2_tin3", [2, 2, 12, 8, 24, 3], 12, 20, (2, 4, 6, 7), True),
    ("cin3_tin10", [1, 3, 16, 8, 16, 10], 40, 12, (2, 2, 4, 4), True),
    ("cin4_tin1_c32", [1, 4, 16, 8, 16, 1], 8, 32, (2, 2, 4, 4), True),
    ("lift_budget", [1, 1, 8, 8, 16, 64], 62, 8, (2, 2, 4, 4), True),   # test_spectral_conv_gpu.ROUTES
    ("cin4_tin64", [1, 4, 8, 8, 16, 64], 60, 8, (2, 2, 4, 4), True),
    ("t30_padded_pitch", [1, 2, 12, 12, 16, 1], 30, 20, (4, 4, 4, 8), True),
    ("2d_time", [2, 1, 32, 32, 10], 16, 20, (4, 4, 4), True),
    ("large_mz", [2, 1, 8, 8, 128, 1], 8, 12, (2, 2, 34, 3), False),   # legacy route, tensor-core bypass
    ("2d_time_cuda_core", [2, 1, 12, 72, 1], 2, 16, (4, 34, 2), False),  # legacy route, CUDA-core bypass
    ("legacy_t30", [1, 2, 8, 8, 72, 1], 30, 20, (2, 2, 34, 8), False),  # legacy route, padded t pitch (Tp = 32)
]
CASE = {c[0]: c for c in CASES}


def _models(case, seed=0, blocks=2, ref_dtype=torch.float64):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    name, in_shape, T, C, modes, fused_pw = case
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    dev = torch.device("cuda")
    torch.manual_seed(seed)
    ref = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev, dtype=ref_dtype,
                           backend="torch", input_grad=True)
    fused = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev, input_grad=True)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    assert fused.fused_pw == fused_pw, (name, fused.fused_pw)
    return d, ref, fused


def _inputs(case, seed, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(1000 + seed)
    x = torch.randn(*case[1], device="cuda", generator=g).to(dtype)
    oshape = list(case[1]); oshape[1] = 1; oshape[-1] = case[2]
    w = torch.randn(*oshape, device="cuda", generator=g)
    return x, w


def _dx(net, x, w):
    xx = x.detach().clone().requires_grad_()
    (dx,) = torch.autograd.grad((net(xx) * w).sum(), xx)
    return dx


def _ref_dx(ref, x, w, drop_t=None):
    """float64 dx of the portable backend; ``drop_t``: minus the lift's term t (a deliberately wrong reference)."""
    store = {}

    def hook(mod, inp, out):
        out.retain_grad()
        store["a"] = out
    h = ref.linear1.register_forward_hook(hook)
    xx = x.detach().to(torch.float64).requires_grad_()
    (ref(xx) * w.double()).sum().backward()
    h.remove()
    dx = xx.grad
    if drop_t is not None:
        e = store["a"].grad[..., drop_t]                            # dL/d(linear1 output) at t
        W1 = ref.linear1.W.detach().double().reshape(-1, x.shape[-1])[drop_t]
        dx = dx - e.unsqueeze(-1) * W1
    return dx


def errors(dx, ref):
    """(relative Frobenius error, worst single position over the rms of the reference)"""
    a, b = dx.detach().double(), ref.detach().double()
    rms = b.pow(2).mean().sqrt()
    return float((a - b).norm() / b.norm()), float((a - b).abs().max() / rms)


def passes(dx, ref, fro=FRO, pos=POS):
    f, p = errors(dx, ref)
    return f < fro and p < pos


# ------------------------------------------------------------------------------------------------ dx vs float64
@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_input_gradient_matches_float64(case, seed):
    d, ref, fused = _models(case, seed=seed)
    x, w = _inputs(case, seed)
    dx = _dx(fused, x, w)
    assert dx.shape == x.shape and dx.dtype == x.dtype
    want = _ref_dx(ref, x, w)
    f, p = errors(dx, want)
    print(f"\nDXERR {case[0]} seed={seed} fro={f:.3e} pos={p:.3e}")
    assert f < FRO and p < POS, (case[0], f, p)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float64], ids=["bf16", "fp64"])
@pytest.mark.parametrize("name", ["cin1_tin1", "cin3_tin10", "2d_time"])
def test_input_gradient_in_the_input_dtype(name, dtype):
    """bf16 inputs are read as bf16 by the lift; fp64 inputs run as fp32.  dx comes back in the input's dtype."""
    case = CASE[name]
    d, ref, fused = _models(case)
    x, w = _inputs(case, 0, dtype)
    dx = _dx(fused, x, w)
    assert dx.dtype == dtype and dx.shape == x.shape
    f, p = errors(dx, _ref_dx(ref, x, w))
    print(f"\nDXERR {name} {dtype} fro={f:.3e} pos={p:.3e}")
    assert f < FRO and p < POS, (name, dtype, f, p)


def test_the_checker_fails_on_a_wrong_input_gradient():
    """One input channel of dx zeroed, and one t term (of T = 40) dropped from the reference, are both rejected."""
    case = CASE["cin3_tin10"]
    d, ref, fused = _models(case)
    x, w = _inputs(case, 0)
    dx = _dx(fused, x, w)
    want = _ref_dx(ref, x, w)
    assert passes(dx, want)
    bad = dx.clone()
    bad[:, 1] = 0
    print("\nzeroed channel", errors(bad, want))
    assert not passes(bad, want)
    dropped = _ref_dx(ref, x, w, drop_t=17)
    print("dropped t term", errors(dx, dropped))
    assert not passes(dx, dropped)


# ------------------------------------------------------------------------------------------------ theta
@pytest.mark.parametrize("name", ["cin2_tin3", "large_mz", "2d_time_cuda_core"])
def test_input_gradient_leaves_the_weight_gradients_alone(name):
    case = CASE[name]
    d, ref, fused = _models(case)
    x, w = _inputs(case, 0)
    (fused(x) * w).sum().backward()
    g0 = fused.theta.grad.clone()
    fused.theta.grad = None
    xx = x.clone().requires_grad_()
    (fused(xx) * w).sum().backward()
    assert xx.grad is not None
    g1 = fused.theta.grad
    assert torch.allclose(g0, g1, rtol=1e-3, atol=1e-6 * float(g0.abs().max()))


@pytest.mark.parametrize("name", ["cin2_tin3", "cin3_tin10", "large_mz", "2d_time_cuda_core"])
def test_frozen_weights_give_dx_only(name):
    """theta.requires_grad_(False): theta.grad stays None, or bitwise equal to what a training backward left there,
    and dx is bitwise equal to the dx of a trainable theta (nothing on the dx path is atomic)."""
    case = CASE[name]
    d, ref, fused = _models(case)
    x, w = _inputs(case, 0)
    fused.theta.requires_grad_(False)
    dx_frozen = _dx(fused, x, w)
    assert fused.theta.grad is None
    fused.theta.requires_grad_(True)
    xx = x.clone().requires_grad_()
    (fused(xx) * w).sum().backward()
    dx_train = xx.grad
    before = fused.theta.grad.clone()
    fused.theta.requires_grad_(False)
    dx_frozen2 = _dx(fused, x, w)
    assert torch.equal(fused.theta.grad, before)
    assert torch.equal(dx_frozen, dx_train) and torch.equal(dx_frozen2, dx_train)
    assert passes(dx_frozen, _ref_dx(ref, x, w))


def test_double_backward_raises():
    case = CASE["cin1_tin1"]
    d, ref, fused = _models(case)
    x, w = _inputs(case, 0)
    xx = x.clone().requires_grad_()
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad((fused(xx) * w).sum(), xx, create_graph=True)


@pytest.mark.parametrize("name", ["cin1_tin1", "large_mz"])
def test_second_backward_through_one_forward_raises(name):
    """The backward overwrites the saved pre-activations with their gradients (both routes), so a second backward
    through the same forward (``retain_graph=True``) would return a wrong dx without a word; it raises instead."""
    case = CASE[name]
    d, ref, fused = _models(case)
    x, w = _inputs(case, 0)
    xx = x.clone().requires_grad_()
    loss = (fused(xx) * w).sum()
    (dx,) = torch.autograd.grad(loss, xx, retain_graph=True)
    assert passes(dx, _ref_dx(ref, x, w))
    with pytest.raises(RuntimeError, match="second backward"):
        torch.autograd.grad(loss, xx)


def test_default_engine_still_refuses_input_gradients():
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    fused = FusedDistributedFNO(P_x, [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), num_blocks=1)
    with pytest.raises(RuntimeError, match="input gradients"):
        fused(torch.randn(1, 1, 16, 16, 16, 1, device="cuda", requires_grad=True))


# ------------------------------------------------------------------------------------------------ inversion
def test_inversion_descends_and_tracks_the_fp32_backend():
    """Surrogate inversion: freeze the network and run Adam on its input towards y* = f(x*), where f is the network
    being inverted.  The loss of the frozen bf16 engine must fall >= 5x and track the same descent on the fp32
    portable backend within 10 %.  The comparison covers the first 40 steps (1.36 -> ~0.04): below a relative loss
    of about 2e-2, the bf16 activations' resolution, the engine's descent stalls while fp32 goes on (measured on an
    H100: 0.0205 against 0.0090 after 200 steps)."""
    import dfno_b200 as d
    case = ("inv", [2, 1, 16, 16, 16, 1], 8, 12, (4, 4, 4, 3), True)
    _, ref, fused = _models(case, seed=11, ref_dtype=torch.float32)
    for p in ref.parameters():
        p.requires_grad_(False)
    fused.theta.requires_grad_(False)
    g = torch.Generator(device="cuda").manual_seed(0)
    k = torch.ones(1, 1, 3, 3, 3, device="cuda") / 27

    def smooth(v):
        return torch.nn.functional.conv3d(torch.nn.functional.pad(v, (1, 1, 1, 1, 1, 1), mode="circular"), k)
    x_star = smooth(torch.randn(2, 1, 16, 16, 16, device="cuda", generator=g)).unsqueeze(-1)
    x0 = smooth(torch.randn(2, 1, 16, 16, 16, device="cuda", generator=g)).unsqueeze(-1)
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    crit = d.DistributedRelativeLpLoss(P_x)
    curves = []
    for net in (fused, ref):
        with torch.no_grad():
            y_star = net(x_star)
        x = x0.clone().requires_grad_()
        opt = torch.optim.Adam([x], lr=5e-2)
        ls = []
        for _ in range(40):
            opt.zero_grad()
            loss = crit(net(x), y_star)
            loss.backward()
            opt.step()
            ls.append(float(loss))
        curves.append(ls)
    lf, lr_ = curves
    print("\nINVERSION", " ".join(f"{i}: {lf[i]:.4f}/{lr_[i]:.4f}" for i in (0, 10, 20, 30, 39)))
    assert fused.theta.grad is None
    assert lf[-1] < lf[0] / 5, (lf[0], lf[-1])
    for i in (len(lf) // 2, len(lf) - 1):
        assert abs(lf[i] - lr_[i]) < 0.1 * lr_[i] + 5e-3, (i, lf[i], lr_[i])
