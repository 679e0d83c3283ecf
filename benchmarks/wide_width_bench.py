"""Width-dependent kernels at widths 32, 48 and 64, and the width-64 training step on both backends.

(a) spectral_mix fwd/bwd, lift fwd/bwd, spectral_out fwd/adj, dpre_dw, head_fwd and head_bwd2 alone, on the engine's
    1-GPU buffers of one shape (B = 1, 128 x 128 x 64 x 20, modes 12 12 12 10), timed with CUDA events; bytes are the
    entries of EnginePlan.cost_model() (one call each), as a share of H100_COPY_GBS.
(b) one training step (forward, sum-of-squares loss, backward, Adam) at width 64 on 64^3 x 20, modes 8, 4 blocks: the fused
    engine against the portable fp32 backend.

    python benchmarks/wide_width_bench.py [--iters 20] [--warmup 3]

Prints one line per measurement and one JSON line; writes nothing."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dfno_b200.models.fused import H100_COPY_GBS, EnginePlan  # noqa: E402
from dfno_b200.ops import build  # noqa: E402
from dfno_b200.ops.gemm import pad_operator  # noqa: E402

H = 128


def gpu_state():
    """name and power limit (W), read by nvidia-smi in this run"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, pl = q.stdout.strip().split(", ")
        return {"gpu": name, "power_limit_w": float(pl)}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None}


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def kernels(C_, C, iters, warmup):
    """(a) at width C: {kernel: (ms, bytes)}"""
    dev = torch.device("cuda", 0)
    B, X, Y, Z, T = 1, 128, 128, 64, 20
    pl = EnginePlan(B, 1, 1, C, T, X, Y, Z, (12, 12, 12, 10))
    pl.finish(4)
    assert pl.fused_pw
    stages = {n: b for n, _, b, _ in pl.cost_model()["stages"]}
    g = torch.Generator(device=dev).manual_seed(C)
    bf = dict(device=dev, dtype=torch.bfloat16)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
    BC, Q, S, L = pl.BC, pl.Q, pl.S, X * Y * T
    s3, s4 = rnd(pl.n_S3).to(torch.bfloat16), torch.empty(pl.n_S3, **bf)
    w = rnd(C, C, Q, 2) / C
    dw = torch.zeros_like(w)
    x = rnd(B, 1, X, Y, Z, 1)
    W1, b1, W2, b2 = rnd(T, 1), rnd(T), rnd(C, 1), rnd(C)
    gW1, gb1, gW2, gb2 = (torch.zeros_like(t) for t in (W1, b1, W2, b2))
    dims = [B, 1, 1, C, T, X, Y, Z]
    h, pre, out = (rnd(pl.n_act).to(torch.bfloat16) for _ in range(3))
    U = rnd(pl.n_U).to(torch.bfloat16)
    op = pad_operator(pl.operators()["iG1a"], device=dev)
    Wb = rnd(C, C) / math.sqrt(C)
    gW = torch.zeros(C, C, device=dev)
    W3, b3 = rnd(H, C) / math.sqrt(C), rnd(H) * 0.2
    w4b4 = rnd(H + 1) / math.sqrt(H)
    w3a = torch.zeros(H, 64 if C + 1 <= 64 else 128, **bf)
    w3a[:, :C] = W3.to(torch.bfloat16)
    w3a[:, C] = b3.to(torch.bfloat16)
    w3t = torch.zeros((C + 1 + 15) // 16 * 16, H, device=dev, dtype=torch.float16)
    w3t[:C] = W3.to(torch.bfloat16).float().t().to(torch.float16)
    R, SR = [Z, T, B * X * Y], [T, 1, Z * T]
    hout = torch.empty(B, 1, X, Y, Z, T, device=dev)
    dy = rnd(B, 1, X, Y, Z, T) * 3e-7
    ws = torch.zeros(1, device=dev, dtype=torch.int32)
    hW3, hb3, hW4, hb4 = torch.zeros(H, C, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev), \
        torch.zeros(1, device=dev)
    K1 = 2 * pl.KZ
    calls = {
        "spectral_mix fwd": lambda: C_.spectral_mix_fwd(s3, w, s4, B, C, Q),
        "spectral_mix bwd": lambda: C_.spectral_mix_bwd(s3, w, s4, s3, dw, False, B, C, Q),
        "lift fwd": lambda: C_.lift_fwd(x, W1, b1, W2, b2, h, dims),
        "lift bwd": lambda: C_.lift_bwd(x, W1, b1, W2, b2, h, gW1, gb1, gW2, gb2, dims),
        "spectral_out fwd": lambda: C_.spectral_out(U, h, op, Wb, False, pre, out, B, C, L, Z, K1, True, True),
        "spectral_out adj": lambda: C_.spectral_out(U, h, op, Wb, True, None, out, B, C, L, Z, K1, False, False),
        "dpre_dw": lambda: C_.dpre_dw(h, pre, out, gW, B, C, L, Z),
        "head fwd": lambda: C_.head_fwd(h, w3a, w4b4, hout, B, C, S, R, SR),
        "head bwd": lambda: C_.head_bwd2(h, w3a, w3t, w4b4[:H].contiguous(), dy, ws, out, hW3, hb3, hW4, hb4, B, C,
                                         S, R, SR),
    }
    return {k: (time_ms(fn, iters, warmup), stages[k]) for k, fn in calls.items()}


def step(backend, iters, warmup):
    """(b) ms per training step at width 64"""
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    in_shape, T, C, modes = [1, 1, 64, 64, 64, 1], 20, 64, (8, 8, 8, 8)
    _, P_x, _ = d.create_standard_partitions([1] * 6)
    torch.manual_seed(0)
    fused = backend == "fused"
    net = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=4, device=dev,
                           dtype=torch.bfloat16 if fused else torch.float32, backend=backend)
    assert isinstance(net, d.FusedDistributedFNO) == fused
    opt = d.FusedAdam(net, lr=1e-4) if fused else torch.optim.Adam(net.parameters(), lr=1e-4)
    x = torch.randn(*in_shape, device=dev)

    def one():
        opt.zero_grad()
        net(x).square().sum().backward()
        opt.step()
    return time_ms(one, iters, warmup)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_width_bench.py needs a GPU")
    C_ = build.load()
    state = gpu_state()
    res = {**state, "copy_gbs": H100_COPY_GBS, "kernels": {}, "step_w64_ms": {}}
    for C in (32, 48, 64):
        for k, (ms, nbytes) in kernels(C_, C, a.iters, a.warmup).items():
            gbs = nbytes / ms / 1e6
            res["kernels"][f"{k} C={C}"] = {"ms": round(ms, 4), "gbs": round(gbs, 1),
                                            "frac_copy": round(gbs / H100_COPY_GBS, 3)}
            print(f"C={C:2d} {k:17s} {ms:8.3f} ms {gbs:7.1f} GB/s {gbs / H100_COPY_GBS:6.1%} of copy")
    for backend in ("fused", "torch"):
        try:
            ms = round(step(backend, max(3, a.iters // 4), a.warmup), 2)
        except torch.cuda.OutOfMemoryError:
            ms = None                                  # not measured: the shape does not fit this backend
        torch.cuda.empty_cache()
        res["step_w64_ms"][backend] = ms
        print(f"width 64 step, {backend:5s}: {ms} ms")
    print(f"{state['gpu']}, power limit {state['power_limit_w']} W")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
