"""The multi-output projection head (head_fwd_multi / head_bwd_multi) against a float64 reference, for O = 1..4 output
channels on every operand width (H100 only).

out[o] = W4[o] . gelu(W3 h + b3) + b4[o] over the positions of h [B*C, S], written as O planes of the public
[B, O, X, Y, Z, T] layout; head_bwd_multi writes the input gradient g and accumulates dW3, db3, dW4 [O, 128] and
db4 [O].  Checks as in test_head_gpu.py: norms and worst entries relative to the reference rms, NaN sentinels in out
and g, non-zero initial gradients."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 128
NORM = {"out": 5e-3, "g": 1e-2, "dW3": 1e-2, "db3": 1e-2, "dW4": 6e-3, "db4": 1e-3}
WORST = {"out": 0.1, "g": 0.1, "dW3": 0.1, "db3": 0.1, "dW4": 0.1}


def C_():
    from dfno_b200.ops import build
    return build.load()


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def gelu_grad64(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def make_case(B, C, O, X, Y, Z, T, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    S = X * Y * Z * T
    h = torch.randn(B * C, S, device=DEV, generator=g).to(torch.bfloat16)
    W3 = (torch.randn(H, C, device=DEV, generator=g) / math.sqrt(C)).to(torch.bfloat16)
    b3 = (torch.randn(H, device=DEV, generator=g) * 0.2).to(torch.bfloat16)
    W4 = torch.randn(O, H, device=DEV, generator=g) / math.sqrt(H)
    b4 = torch.randn(O, device=DEV, generator=g)
    return dict(B=B, C=C, O=O, dims=(X, Y, Z, T), S=S, h=h, W3=W3, b3=b3, W4=W4, b4=b4, gen=g)


def operands(W3, b3, C):
    w3a = torch.zeros(H, 64, device=DEV, dtype=torch.bfloat16)
    w3a[:, :C] = W3
    w3a[:, C] = b3
    w3t = torch.zeros((C + 1 + 15) // 16 * 16, H, device=DEV, dtype=torch.float16)
    w3t[:C] = W3.float().t().to(torch.float16)
    return w3a, w3t


def row_digits(B, O, X, Y, Z, T):
    """engine row (b, x, y, t, z) -> offset in the public [B, O, X, Y, Z, T] layout (channel 0), innermost first"""
    S = X * Y * Z * T
    return [Z, T, X * Y, B], [T, 1, Z * T, O * S]


def from_public(v, B, O, X, Y, Z, T):
    """[B, O, X, Y, Z, T] -> [B*S, O] in engine row order"""
    return v.permute(0, 2, 3, 5, 4, 1).reshape(B * X * Y * T * Z, O)


def reference(case, dy):
    """float64 forward and backward; dy: [B*S, O] in engine row order"""
    B, C, S = case["B"], case["C"], case["S"]
    hin = case["h"].double().view(B, C, S).permute(0, 2, 1).reshape(B * S, C)
    W3, b3 = case["W3"].double(), case["b3"].double()
    W4, b4 = case["W4"].double(), case["b4"].double()
    pre = hin @ W3.t() + b3
    a = gelu64(pre)
    out = a @ W4.t() + b4
    dy = dy.double()
    dpre = (dy @ W4) * gelu_grad64(pre)
    del pre
    ref = dict(out=out, dW4=dy.t() @ a, db4=dy.sum(0), dW3=dpre.t() @ hin, db3=dpre.sum(0))
    del a
    ref["g"] = (dpre @ W3).view(B, S, C).permute(0, 2, 1).reshape(B * C, S)
    return ref


def run_kernels(case, dy_pub, init_scale, W4=None, b4=None):
    """head_fwd_multi + head_bwd_multi; W4 / b4 override what the kernels see (the reference keeps its own)"""
    B, C, O, S = case["B"], case["C"], case["O"], case["S"]
    X, Y, Z, T = case["dims"]
    W4 = case["W4"] if W4 is None else W4
    b4 = case["b4"] if b4 is None else b4
    w3a, w3t = operands(case["W3"], case["b3"], C)
    R, SR = row_digits(B, O, X, Y, Z, T)
    out = torch.full((B, O, X, Y, Z, T), float("nan"), device=DEV)
    w4b4 = torch.cat([W4.reshape(-1), b4]).contiguous()
    C_().head_fwd_multi(case["h"], w3a, w4b4, out, B, C, S, O, S, R, SR)
    g = torch.full((B * C, S), float("nan"), device=DEV, dtype=torch.bfloat16)
    gen = case["gen"]
    init = {"dW3": torch.randn(H, C, device=DEV, generator=gen) * init_scale["dW3"],
            "db3": torch.randn(H, device=DEV, generator=gen) * init_scale["db3"],
            "dW4": torch.randn(O, H, device=DEV, generator=gen) * init_scale["dW4"],
            "db4": torch.randn(O, device=DEV, generator=gen) * init_scale["db4"]}
    grads = {k: v.clone() for k, v in init.items()}
    ws = torch.zeros(1, device=DEV, dtype=torch.int32)
    C_().head_bwd_multi(case["h"], w3a, w3t, W4.contiguous(), dy_pub.contiguous(), ws, g, grads["dW3"],
                        grads["db3"], grads["dW4"], grads["db4"], B, C, S, O, S, R, SR)
    torch.cuda.synchronize()
    got = {"out": from_public(out, B, O, X, Y, Z, T), "g": g}
    got.update({k: grads[k] - init[k] for k in init})
    finite = {"out": bool(torch.isfinite(out).all()), "g": bool(torch.isfinite(g).all())}
    return got, finite


def measure(got, ref):
    m = {}
    for k in NORM:
        dd = got[k].double() - ref[k]
        m[k] = float(dd.norm() / ref[k].norm().clamp_min(1e-300))
        if k in WORST:
            m[k + "_worst"] = float(dd.abs().max() / ref[k].pow(2).mean().sqrt().clamp_min(1e-300))
    return m


def check(case, dscale, **override):
    B, O = case["B"], case["O"]
    X, Y, Z, T = case["dims"]
    dy_pub = torch.randn(B, O, X, Y, Z, T, device=DEV, generator=case["gen"]) * dscale
    ref = reference(case, from_public(dy_pub, B, O, X, Y, Z, T))
    init_scale = {k: float(ref[k].abs().max()) for k in ("dW3", "db3", "dW4", "db4")}
    got, finite = run_kernels(case, dy_pub, init_scale, **override)
    m = measure(got, ref)
    bad = [k for k, v in finite.items() if not v]
    bad += [k for k in NORM if not m[k] < NORM[k]]
    bad += [k + "_worst" for k in WORST if not m[k + "_worst"] < WORST[k]]
    return m, bad


WIDTHS = [1, 8, 15, 16, 20, 31]          # KR = 16 and 32 on both sides of the boundary (the backward takes C <= 31)


@pytest.mark.parametrize("dscale", [3e-7, 1.0])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("O", [1, 2, 3, 4])
@pytest.mark.parametrize("C", WIDTHS)
def test_head_multi_widths(C, O, B, dscale):
    """S = 720: five full tiles and a partial one of 80 positions"""
    case = make_case(B, C, O, 3, 5, 8, 6, seed=5000 + 100 * C + 10 * O + B)
    m, bad = check(case, dscale)
    print(f"C={C} O={O} B={B} dout~{dscale:g}: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("C,O", [(16, 2), (20, 3), (31, 4)])
def test_head_multi_many_tiles(C, O):
    """S = 244800 with B = 2: 3826 tiles, so the TMA ring wraps many times in every consumer warpgroup"""
    case = make_case(2, C, O, 17, 15, 32, 30, seed=6000 + C)
    m, bad = check(case, 3e-7)
    print(f"C={C} O={O} many tiles: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("O", [1, 2, 3, 4])
def test_head_multi_fwd_width_32(O):
    """the forward also takes C = 32 (KR = 48), where the fused engine uses it with one output only"""
    case = make_case(2, 32, O, 3, 5, 8, 6, seed=7000 + O)
    B, S = case["B"], case["S"]
    X, Y, Z, T = case["dims"]
    w3a, _ = operands(case["W3"], case["b3"], 32)
    R, SR = row_digits(B, O, X, Y, Z, T)
    out = torch.full((B, O, X, Y, Z, T), float("nan"), device=DEV)
    C_().head_fwd_multi(case["h"], w3a, torch.cat([case["W4"].reshape(-1), case["b4"]]), out, B, 32, S, O, S, R, SR)
    torch.cuda.synchronize()
    ref = reference(case, torch.zeros(B * S, O, device=DEV))["out"]
    got = from_public(out, B, O, X, Y, Z, T).double()
    assert bool(torch.isfinite(got).all())
    assert float((got - ref).norm() / ref.norm()) < NORM["out"]
    assert float((got - ref).abs().max() / ref.pow(2).mean().sqrt()) < WORST["out"]


def test_head_multi_checker_sees_swapped_output_rows():
    """the kernels see W4 with outputs 0 and 2 swapped: out (per plane) and the gradients that flow through W4 must
    fail against the clean reference (dW4 and db4 do not depend on W4)"""
    case = make_case(1, 20, 3, 3, 5, 8, 6, seed=8000)
    W4_bad = case["W4"][[2, 1, 0]].contiguous()
    m, bad = check(case, 1.0, W4=W4_bad)
    print("swapped W4 rows: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()) + f" failed={bad}")
    assert "out" in bad and "g" in bad and "dW3" in bad, (bad, m)


def test_head_multi_checker_sees_one_corrupted_bias():
    """the kernels see b4[1] shifted: the output check must fail (the bias is per plane)"""
    case = make_case(1, 20, 3, 3, 5, 8, 6, seed=8100)
    b4_bad = case["b4"].clone()
    b4_bad[1] += 0.5
    m, bad = check(case, 1.0, b4=b4_bad)
    print("corrupted b4[1]: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()) + f" failed={bad}")
    assert "out" in bad or "out_worst" in bad, (bad, m)


def test_head_multi_backward_refuses_width_32():
    case = make_case(1, 32, 2, 3, 5, 8, 6, seed=8200)
    with pytest.raises(RuntimeError, match="C <= 31"):
        check(case, 1.0)
