"""The backward's pointwise tail at the headline shape (B = 1, C = 20, 128^3 x 20, K1 = 48): today's pair (adjoint
spectral_out, then dpre_dw) against the adjoint spectral_out with that work folded in -- the top-block variant (GELU'
of the block below), the middle-block variant (also the bypass weight gradient) and the block-0 variant (weight
gradient, g stored).  CUDA events over --iters calls per variant, in --rounds alternating rounds; the median round
against the bytes of the engine's traffic model entries (EnginePlan.cost_model(fold_bwd=True)), as a share of
H100_COPY_GBS.  Prints one line per variant and one JSON line; writes nothing.

    python benchmarks/spectral_out_bwd_bench.py [--iters 30] [--warmup 3] [--rounds 3]"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from head_bench import gpu_state, time_ms  # noqa: E402
from dfno_b200.models.fused import H100_COPY_GBS  # noqa: E402
from dfno_b200.ops import build  # noqa: E402
from dfno_b200.ops.gemm import pad_operator  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spectral_out_bwd_bench.py needs a GPU")
    C_ = build.load()
    dev = torch.device("cuda", 0)
    B, C, X, Y, Z, T, K1 = 1, 20, 128, 128, 128, 20, 48
    L = X * Y * T
    bf = torch.bfloat16
    g = torch.Generator(device=dev).manual_seed(0)
    U = (torch.randn(B * C, L, K1, device=dev, generator=g) * 1e-3).to(bf)
    dpre = (torch.randn(B * C, L, Z, device=dev, generator=g) * 1e-3).to(bf)
    pre = (torch.randn(B * C, L, Z, device=dev, generator=g) * 1.5).to(bf)
    h = torch.randn(B * C, L, Z, device=dev, generator=g).to(bf)
    gbuf = torch.empty_like(dpre)
    Fop = pad_operator(torch.randn(Z, K1, device=dev, generator=g) / math.sqrt(K1))
    W = torch.randn(C, C, device=dev, generator=g) / math.sqrt(C)
    dW = torch.zeros(C, C, device=dev)
    act, u = dpre.numel() * 2, U.numel() * 2

    def adj(pre_prev=None, h_dw=None, dw=None):
        C_.spectral_out(U, dpre, Fop, W, True, None, gbuf, B, C, L, Z, K1, False, False, pre_prev, h_dw, dw)

    def pair():
        adj()
        C_.dpre_dw(gbuf, pre, h, dW, B, C, L, Z)

    # (name, call, bytes it must move): pre is overwritten with dpre by every call, which changes no byte count
    variants = [("adjoint + dpre_dw (today)", pair, u + 2 * act + 4 * act),
                ("adj+dpre (top block)", lambda: adj(pre), u + 3 * act),
                ("adj+dpre+dW (middle blocks)", lambda: adj(pre, h, dW), u + 4 * act),
                ("adj+dW (block 0)", lambda: adj(None, h, dW), u + 3 * act)]
    times = {n: [] for n, _, _ in variants}
    for _ in range(a.rounds):
        for n, fn, _ in variants:
            times[n].append(time_ms(fn, a.iters, a.warmup))
    state = gpu_state()
    out = {"shape": dict(B=B, C=C, L=L, Z=Z, K1=K1), **state, "copy_gbs": H100_COPY_GBS, "variants": {}}
    print(f"{state['gpu']}  power limit {state['power_limit_w']} W  SM clock {state['sm_clock_mhz']} / "
          f"{state['sm_clock_max_mhz']} MHz")
    for n, _, nbytes in variants:
        ms = statistics.median(times[n])
        share = nbytes / (H100_COPY_GBS * 1e9) * 1e3 / ms
        out["variants"][n] = {"ms": ms, "rounds_ms": times[n], "gb": nbytes / 1e9, "copy_share": share}
        print(f"  {n:30s} {ms:7.3f} ms  (rounds {', '.join('%.3f' % t for t in times[n])})  {nbytes / 1e9:6.2f} GB  "
              f"{share:6.1%} of copy rate")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
