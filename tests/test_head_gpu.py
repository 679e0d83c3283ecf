"""The channel-major projection head (head_fwd / head_bwd2) against a float64 reference, on every operand width
(H100 only).

The head is out = W4 . gelu(W3 h + b3) + b4 over the positions of h [B*C, S]; head_bwd2 writes the input gradient g
and accumulates dW3, db3, dW4 and db4.  Each case checks norms and, so that one mis-mapped lane, row or tile cannot
hide in a norm, the worst single position (out), element (g) and gradient entry, each relative to the reference rms.
Outputs start as NaN sentinels (every element must be written) and gradient buffers start non-zero (the kernels
accumulate)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 128

# bounds: norm error relative to the reference norm, worst entry relative to the reference rms
NORM = {"out": 5e-3, "g": 1e-2, "dW3": 1e-2, "db3": 1e-2, "dW4": 6e-3, "db4": 1e-3}
WORST = {"out": 0.1, "g": 0.1, "dW3": 0.1, "db3": 0.1, "dW4": 0.1}


def C_():
    from dfno_b200.ops import build
    return build.load()


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def gelu_grad64(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def make_case(B, C, X, Y, Z, T, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    S = X * Y * Z * T
    h = torch.randn(B * C, S, device=DEV, generator=g).to(torch.bfloat16)
    W3 = (torch.randn(H, C, device=DEV, generator=g) / math.sqrt(C)).to(torch.bfloat16)
    b3 = (torch.randn(H, device=DEV, generator=g) * 0.2).to(torch.bfloat16)
    w4b4 = torch.randn(H + 1, device=DEV, generator=g) / math.sqrt(H)
    return dict(B=B, C=C, dims=(X, Y, Z, T), S=S, h=h, W3=W3, b3=b3, w4b4=w4b4, gen=g)


def operands(W3, b3, C):
    w3a = torch.zeros(H, 64, device=DEV, dtype=torch.bfloat16)
    w3a[:, :C] = W3
    w3a[:, C] = b3
    w3t = torch.zeros((C + 1 + 15) // 16 * 16, H, device=DEV, dtype=torch.float16)
    w3t[:C] = W3.float().t().to(torch.float16)
    return w3a, w3t


def row_digits(B, X, Y, Z, T):
    """engine row (b, x, y, t, z) -> offset in the public [B, 1, X, Y, Z, T] layout, digits innermost first"""
    return [Z, T, B * X * Y], [T, 1, Z * T]


def to_public(v, B, X, Y, Z, T):
    """[B*S] in engine row order -> [B, 1, X, Y, Z, T]"""
    return v.reshape(B, X, Y, T, Z).permute(0, 1, 2, 4, 3).unsqueeze(1)


def from_public(v, B, X, Y, Z, T):
    return v.squeeze(1).permute(0, 1, 2, 4, 3).reshape(B * X * Y * T * Z)


def reference(case, dy_rows):
    """float64 forward and backward; dy_rows: [B*S] in engine row order"""
    B, C, S = case["B"], case["C"], case["S"]
    hin = case["h"].double().view(B, C, S).permute(0, 2, 1).reshape(B * S, C)
    W3, b3 = case["W3"].double(), case["b3"].double()
    w4, b4 = case["w4b4"][:H].double(), case["w4b4"][H].double()
    pre = hin @ W3.t() + b3
    a = gelu64(pre)
    out = a @ w4 + b4
    dy = dy_rows.double()
    dpre = (dy[:, None] * w4[None, :]) * gelu_grad64(pre)
    del pre
    ref = dict(out=out, dW4=a.t() @ dy, db4=dy.sum().reshape(1), dW3=dpre.t() @ hin, db3=dpre.sum(0))
    del a
    ref["g"] = (dpre @ W3).view(B, S, C).permute(0, 2, 1).reshape(B * C, S)
    return ref


def run_kernels(case, dy_pub, init_scale, W3=None):
    """head_fwd + head_bwd2 on the case; W3 overrides the weights the kernels see (the reference keeps its own)"""
    B, C, S = case["B"], case["C"], case["S"]
    X, Y, Z, T = case["dims"]
    w3a, w3t = operands(case["W3"] if W3 is None else W3, case["b3"], C)
    R, SR = row_digits(B, X, Y, Z, T)
    out = torch.full((B, 1, X, Y, Z, T), float("nan"), device=DEV)
    C_().head_fwd(case["h"], w3a, case["w4b4"], out, B, C, S, R, SR)
    g = torch.full((B * C, S), float("nan"), device=DEV, dtype=torch.bfloat16)
    gen = case["gen"]
    init = {"dW3": torch.randn(H, C, device=DEV, generator=gen) * init_scale["dW3"],
            "db3": torch.randn(H, device=DEV, generator=gen) * init_scale["db3"],
            "dW4": torch.randn(H, device=DEV, generator=gen) * init_scale["dW4"],
            "db4": torch.randn(1, device=DEV, generator=gen) * init_scale["db4"]}
    grads = {k: v.clone() for k, v in init.items()}
    ws = torch.zeros(1, device=DEV, dtype=torch.int32)
    C_().head_bwd2(case["h"], w3a, w3t, case["w4b4"][:H].contiguous(), dy_pub.contiguous(), ws, g,
                   grads["dW3"], grads["db3"], grads["dW4"], grads["db4"], B, C, S, R, SR)
    torch.cuda.synchronize()
    got = {"out": from_public(out, B, X, Y, Z, T), "g": g}
    got.update({k: grads[k] - init[k] for k in init})      # what the kernel added
    finite = {"out": bool(torch.isfinite(out).all()), "g": bool(torch.isfinite(g).all())}
    return got, finite


def measure(got, ref):
    m = {}
    for k in NORM:
        d = got[k].double() - ref[k]
        m[k] = float(d.norm() / ref[k].norm().clamp_min(1e-300))
        if k in WORST:
            m[k + "_worst"] = float(d.abs().max() / ref[k].pow(2).mean().sqrt().clamp_min(1e-300))
    return m


def failures(m, finite):
    bad = [k for k, v in finite.items() if not v]
    bad += [k for k in NORM if not m[k] < NORM[k]]
    bad += [k + "_worst" for k in WORST if not m[k + "_worst"] < WORST[k]]
    return bad


def check(case, dscale, W3_kernel=None):
    B, S = case["B"], case["S"]
    X, Y, Z, T = case["dims"]
    dy_pub = torch.randn(B, 1, X, Y, Z, T, device=DEV, generator=case["gen"]) * dscale
    ref = reference(case, from_public(dy_pub, B, X, Y, Z, T))
    init_scale = {k: float(ref[k].abs().max()) for k in ("dW3", "db3", "dW4", "db4")}
    got, finite = run_kernels(case, dy_pub, init_scale, W3=W3_kernel)
    m = measure(got, ref)
    return m, failures(m, finite)


# C + 1 (the ones row) padded to 16 gives KR = 16, 32 and 48 on both sides of each boundary
WIDTHS = [1, 8, 15, 16, 20, 31, 32]


@pytest.mark.parametrize("dscale", [3e-7, 1.0])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("C", WIDTHS)
def test_head_widths(C, B, dscale):
    """S = 720: five full tiles and a partial one of 80 positions"""
    case = make_case(B, C, 3, 5, 8, 6, seed=1000 + 10 * C + B)
    m, bad = check(case, dscale)
    print(f"C={C} B={B} dout~{dscale:g}: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("C", [16, 20, 32])
def test_head_many_tiles(C):
    """S = 244800 with B = 2: 3826 tiles (the last of each batch partial), so every consumer warpgroup of every CTA
    takes many tiles and the TMA ring wraps many times"""
    case = make_case(2, C, 17, 15, 32, 30, seed=2000 + C)
    m, bad = check(case, 3e-7)
    print(f"C={C} many tiles: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("C", [33, 40, 47])
def test_head_fwd_wide(C):
    """head_fwd alone takes C up to 47 (KR = 48)"""
    case = make_case(2, C, 3, 5, 8, 6, seed=3000 + C)
    B, S = case["B"], case["S"]
    X, Y, Z, T = case["dims"]
    w3a, _ = operands(case["W3"], case["b3"], C)
    R, SR = row_digits(B, X, Y, Z, T)
    out = torch.full((B, 1, X, Y, Z, T), float("nan"), device=DEV)
    C_().head_fwd(case["h"], w3a, case["w4b4"], out, B, C, S, R, SR)
    torch.cuda.synchronize()
    ref = reference(case, torch.zeros(B * S, device=DEV))["out"]
    got = from_public(out, B, X, Y, Z, T).double()
    assert bool(torch.isfinite(got).all())
    norm = float((got - ref).norm() / ref.norm())
    worst = float((got - ref).abs().max() / ref.pow(2).mean().sqrt())
    assert norm < NORM["out"] and worst < WORST["out"], (norm, worst)


def test_head_checker_sees_one_corrupted_weight():
    """The kernels see W3 with one entry changed; the checks against the clean reference must fail, dW3 among them"""
    case = make_case(1, 20, 3, 5, 8, 6, seed=4000)
    j, c = 37, 11
    W3_bad = case["W3"].clone()
    W3_bad[j, c] += 1.0
    m, bad = check(case, 3e-7, W3_kernel=W3_bad)
    print("corrupted W3[37, 11]: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()) + f" failed={bad}")
    assert "dW3" in bad or "dW3_worst" in bad, (bad, m)
    assert len(bad) >= 2, (bad, m)
