"""Projection head kernels alone at the headline shape: head_fwd and head_bwd2 on B = 1, C = 20, S = 128^3 x 20
positions, timed with CUDA events, against the bytes each must move (the head entries of the engine's traffic model,
EnginePlan.cost_model / tools/plan.py).  Prints one line per kernel and one JSON line; writes nothing.

    python benchmarks/head_bench.py [--iters 50] [--warmup 5]

head_bwd2's time includes its absmax pre-pass over dout (the power-of-two scale), as every call runs it."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dfno_b200.models.fused import H100_COPY_GBS  # noqa: E402
from dfno_b200.ops import build  # noqa: E402

H = 128


def gpu_state():
    """name, power limit (W) and current SM clock (MHz), read by nvidia-smi in this run"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1]), "sm_clock_mhz": float(q[2]), "sm_clock_max_mhz": float(q[3])}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "sm_clock_mhz": None,
                "sm_clock_max_mhz": None}


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


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("head_bench.py needs a GPU")
    C_ = build.load()
    dev = torch.device("cuda", 0)
    B, C, X, Y, Z, T = 1, 20, 128, 128, 128, 20
    S = X * Y * Z * T
    g = torch.Generator(device=dev).manual_seed(0)
    h = torch.randn(B * C, S, device=dev, generator=g).to(torch.bfloat16)
    W3 = torch.randn(H, C, device=dev, generator=g) / math.sqrt(C)
    b3 = torch.randn(H, device=dev, generator=g) * 0.2
    w4b4 = torch.randn(H + 1, device=dev, generator=g) / math.sqrt(H)
    w3a = torch.zeros(H, 64, device=dev, dtype=torch.bfloat16)
    w3a[:, :C] = W3.to(torch.bfloat16)
    w3a[:, C] = b3.to(torch.bfloat16)
    w3t = torch.zeros((C + 1 + 15) // 16 * 16, H, device=dev, dtype=torch.float16)
    w3t[:C] = W3.to(torch.bfloat16).float().t().to(torch.float16)
    R, SR = [Z, T, B * X * Y], [T, 1, Z * T]          # engine row (b, x, y, t, z) -> public [B, 1, X, Y, Z, T]
    out = torch.empty(B, 1, X, Y, Z, T, device=dev)
    dy = torch.randn(B, 1, X, Y, Z, T, device=dev, generator=g) * 3e-7
    gout = torch.empty(B * C, S, device=dev, dtype=torch.bfloat16)
    gW3, gb3, gW4, gb4 = (torch.zeros(H, C, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev),
                          torch.zeros(1, device=dev))
    ws = torch.zeros(1, device=dev, dtype=torch.int32)
    w4 = w4b4[:H].contiguous()

    def fwd():
        C_.head_fwd(h, w3a, w4b4, out, B, C, S, R, SR)

    def bwd():
        C_.head_bwd2(h, w3a, w3t, w4, dy, ws, gout, gW3, gb3, gW4, gb4, B, C, S, R, SR)

    act = B * C * S * 2                                # one bf16 channel-major activation
    npos = B * S
    need = {"head_fwd": act + npos * 4,              # read h, write out (fp32)
            "head_bwd2": 2 * act + 2 * npos * 4}     # read h and dout, write g; dout read again by the pre-pass
    ms = {"head_fwd": time_ms(fwd, a.iters, a.warmup), "head_bwd2": time_ms(bwd, a.iters, a.warmup)}
    state = gpu_state()
    res = {"shape": {"B": B, "C": C, "S": S}, "iters": a.iters, **state, "copy_gbs": H100_COPY_GBS, "kernels": {}}
    for k in ms:
        gbs = need[k] / ms[k] / 1e6
        res["kernels"][k] = {"ms": round(ms[k], 4), "bytes": need[k], "gbs": round(gbs, 1),
                             "frac_copy": round(gbs / H100_COPY_GBS, 3)}
        print(f"{k:10s} {ms[k]:8.3f} ms  {need[k] / 1e9:6.2f} GB  {gbs:7.1f} GB/s  {gbs / H100_COPY_GBS:5.1%} of copy")
    print(f"{state['gpu']}, power limit {state['power_limit_w']} W, SM clock {state['sm_clock_mhz']} MHz "
          f"(max {state['sm_clock_max_mhz']})")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
