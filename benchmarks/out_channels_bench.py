"""Cost of several output fields at the headline shape (B = 1, C = 20, S = 128^3 x 20 positions).

1. The projection head kernels alone: head_fwd / head_bwd2 (one output) and head_fwd_multi / head_bwd_multi at
   O = 1..4, timed with CUDA events, against the head bytes of the engine's traffic model (EnginePlan.cost_model).
2. The training step (forward + relative-L2 loss + backward + Adam, eager launches) of the headline network at
   O = 1 and O = 3, alternated over rounds, next to three times the O = 1 step (three single-field networks).

    python benchmarks/out_channels_bench.py [--iters 50] [--rounds 3] [--steps 10]

Prints one line per measurement and one JSON line; writes nothing."""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from head_bench import gpu_state, time_ms  # noqa: E402
from dfno_b200.models.fused import H100_COPY_GBS, EnginePlan  # noqa: E402
from dfno_b200.ops import build  # noqa: E402

H = 128
SHAPE = dict(B=1, C=20, X=128, Y=128, Z=128, T=20)
MODES = (12, 12, 12, 10)


def head_bytes(O):
    """(forward, backward) bytes of the head at the headline shape, from the traffic model"""
    s = SHAPE
    pl = EnginePlan(s["B"], 1, 1, s["C"], s["T"], s["X"], s["Y"], s["Z"], MODES, out_channels=O)
    pl.finish(4)
    st = {n: b for n, _, b, _ in pl.cost_model()["stages"]}
    return st["head fwd"], st["head bwd"]


def bench_kernels(C_, iters, warmup):
    s = SHAPE
    B, C, X, Y, Z, T = s["B"], s["C"], s["X"], s["Y"], s["Z"], s["T"]
    S = X * Y * Z * T
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    h = torch.randn(B * C, S, device=dev, generator=g).to(torch.bfloat16)
    W3 = torch.randn(H, C, device=dev, generator=g) / math.sqrt(C)
    b3 = torch.randn(H, device=dev, generator=g) * 0.2
    w3a = torch.zeros(H, 64, device=dev, dtype=torch.bfloat16)
    w3a[:, :C] = W3.to(torch.bfloat16)
    w3a[:, C] = b3.to(torch.bfloat16)
    w3t = torch.zeros((C + 1 + 15) // 16 * 16, H, device=dev, dtype=torch.float16)
    w3t[:C] = W3.to(torch.bfloat16).float().t().to(torch.float16)
    gout = torch.empty(B * C, S, device=dev, dtype=torch.bfloat16)
    gW3, gb3 = torch.zeros(H, C, device=dev), torch.zeros(H, device=dev)
    ws = torch.zeros(1, device=dev, dtype=torch.int32)
    rows = {}
    for O in (0, 1, 2, 3, 4):                       # 0: the single-output kernels head_fwd / head_bwd2
        n = max(O, 1)
        w4b4 = torch.randn(n * (H + 1), device=dev, generator=g) / math.sqrt(H)
        w4 = w4b4[:n * H].contiguous()
        out = torch.empty(B, n, X, Y, Z, T, device=dev)
        dy = torch.randn(B, n, X, Y, Z, T, device=dev, generator=g) * 3e-7
        gW4, gb4 = torch.zeros(n * H, device=dev), torch.zeros(n, device=dev)
        if O == 0:
            R, SR = [Z, T, B * X * Y], [T, 1, Z * T]
            fwd = lambda: C_.head_fwd(h, w3a, w4b4, out, B, C, S, R, SR)                       # noqa: E731
            bwd = lambda: C_.head_bwd2(h, w3a, w3t, w4, dy, ws, gout, gW3, gb3, gW4, gb4, B, C, S, R, SR)  # noqa: E731
            names = ("head_fwd", "head_bwd2")
        else:
            R, SR = [Z, T, X * Y, B], [T, 1, Z * T, O * S]
            fwd = lambda: C_.head_fwd_multi(h, w3a, w4b4, out, B, C, S, O, S, R, SR)          # noqa: E731
            bwd = lambda: C_.head_bwd_multi(h, w3a, w3t, w4, dy, ws, gout, gW3, gb3, gW4, gb4, B, C, S, O, S,  # noqa: E731
                                            R, SR)
            names = (f"head_fwd_multi O={O}", f"head_bwd_multi O={O}")
        need = head_bytes(n)
        for name, fn, nb in zip(names, (fwd, bwd), need):
            ms = time_ms(fn, iters, warmup)
            gbs = nb / ms / 1e6
            rows[name] = {"ms": round(ms, 4), "bytes": nb, "gbs": round(gbs, 1), "frac_copy": round(gbs / H100_COPY_GBS, 3)}
            print(f"{name:22s} {ms:8.3f} ms  {nb / 1e9:6.2f} GB  {gbs:7.1f} GB/s  {gbs / H100_COPY_GBS:5.1%} of copy")
        del out, dy
    return rows


def bench_steps(rounds, steps):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam, FusedDistributedFNO
    s = SHAPE
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    dev = torch.device("cuda", 0)
    in_shape = [s["B"], 1, s["X"], s["Y"], s["Z"], 1]
    x = torch.randn(*in_shape, device=dev)
    times = {1: [], 3: []}
    for _ in range(rounds):
        for O in (1, 3):
            net = FusedDistributedFNO(P_x, in_shape, s["T"], s["C"], MODES, num_blocks=4, device=dev, init_seed=0,
                                      out_channels=O)
            opt = FusedAdam(net, lr=1e-3)
            crit = d.DistributedRelativeLpLoss(P_x, engine=net)
            t = torch.randn(s["B"], O, s["X"], s["Y"], s["Z"], s["T"], device=dev)

            def step():
                opt.zero_grad()
                crit(net(x), t).backward()
                opt.step()
            times[O].append(time_ms(step, steps, 2))
            del net, opt, crit, t
            torch.cuda.empty_cache()
    med = {O: statistics.median(v) for O, v in times.items()}
    for O in (1, 3):
        print(f"training step O={O}: median {med[O]:.2f} ms over {rounds} rounds {['%.2f' % v for v in times[O]]}")
    print(f"three single-field networks (3 x O=1): {3 * med[1]:.2f} ms")
    return {"step_ms": {str(O): [round(v, 3) for v in times[O]] for O in times},
            "median_ms": {str(O): round(v, 3) for O, v in med.items()}, "three_single_ms": round(3 * med[1], 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("out_channels_bench.py needs a GPU")
    torch.cuda.set_device(0)
    state = gpu_state()
    res = {"shape": SHAPE, **state, "copy_gbs": H100_COPY_GBS, "kernels": bench_kernels(build.load(), a.iters, a.warmup)}
    res["training"] = bench_steps(a.rounds, a.steps)
    print(f"{state['gpu']}, power limit {state['power_limit_w']} W, SM clock {state['sm_clock_mhz']} MHz "
          f"(max {state['sm_clock_max_mhz']})")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
