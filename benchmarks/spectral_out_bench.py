"""spectral_out, forward and adjoint, at the headline shape (B = 1, C = 20, 128^3 x 20, K1 = 48) and at the local
lines of 2, 4 and 8 pencil ranks on one GPU (Y_local = 64, 32, 16): the training forward (GELU, pre saved), the plain
adjoint and the three folded adjoints of the backward (top block: GELU' of the block below; middle blocks: also the
bypass weight gradient; block 0: weight gradient, g stored).  CUDA events over --iters calls per variant, in --rounds
alternating rounds; the median round against the bytes of the engine's traffic model (EnginePlan.cost_model(
fold_bwd=True), per call), as a share of H100_COPY_GBS.  Every output's bytes (pre, out, g, dpre) are checksummed on
fixed seeded inputs, so that two builds run in one session can be compared bit for bit.  Prints one line per variant
and one JSON line; writes nothing.

    python benchmarks/spectral_out_bench.py [--iters 20] [--warmup 3] [--rounds 3] [--ranks 1 2 4 8]"""
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
from dfno_b200.models.fused import H100_COPY_GBS, EnginePlan  # noqa: E402
from dfno_b200.ops import build  # noqa: E402
from dfno_b200.ops.gemm import pad_operator  # noqa: E402

B, C, X, Y, Z, T, MODES = 1, 20, 128, 128, 128, 20, (12, 12, 12, 10)


def checksum(t):
    """position-weighted sum of the tensor's 32-bit words (wrapping int64), computed on the device"""
    v = t.contiguous().view(torch.int32).reshape(-1).to(torch.int64)
    w = torch.arange(v.numel(), device=v.device, dtype=torch.int64) % 65521 + 1
    return "%016x" % (int((v * w).sum()) & (2 ** 64 - 1))


def shape_case(C_, P, dev, a):
    pl = EnginePlan(B, 1, 1, C, T, X, Y, Z, MODES, world=P, rank=0)
    pl.finish(4)
    L = X * pl.Yl * T
    K1 = pl.n_U // (B * C * L)
    fold = {n: b for n, _, b, _ in pl.cost_model(fold_bwd=True)["stages"]}
    plain = {n: b for n, _, b, _ in pl.cost_model()["stages"]}
    bf = torch.bfloat16
    g = torch.Generator(device=dev).manual_seed(0)
    U = (torch.randn(B * C, L, K1, device=dev, generator=g) * 0.05).to(bf)
    h = torch.randn(B * C, L, Z, device=dev, generator=g).to(bf)
    dpre = (torch.randn(B * C, L, Z, device=dev, generator=g) * 1e-3).to(bf)
    pre0 = (torch.randn(B * C, L, Z, device=dev, generator=g) * 1.5).to(bf)
    Fop = pad_operator(torch.randn(Z, K1, device=dev, generator=g) / math.sqrt(K1))
    Fadj = pad_operator(torch.randn(Z, K1, device=dev, generator=g) / math.sqrt(K1))
    W = torch.randn(C, C, device=dev, generator=g) / math.sqrt(C)
    pre, out, gbuf, pp = (torch.empty_like(h) for _ in range(4))
    dW = torch.zeros(C, C, device=dev)

    def fwd():
        C_.spectral_out(U, h, Fop, W, False, pre, out, B, C, L, Z, K1, True, True, None, None, None)

    def adj(pre_prev=None, h_dw=None, dw=None):
        C_.spectral_out(U, dpre, Fadj, W, True, None, gbuf, B, C, L, Z, K1, False, False, pre_prev, h_dw, dw)

    # (name, call, bytes per call, {output: tensor}); the folded dpre variants overwrite pp (a copy of pre0) in place,
    # so pp is refilled before the checksummed call
    variants = [("fwd (gelu, pre)", fwd, fold["spectral_out fwd"], {"pre": pre, "out": out}),
                ("adj", lambda: adj(), plain["spectral_out adj"], {"g": gbuf}),
                ("adj+dpre (top)", lambda: adj(pp), fold["spectral_out adj+dpre"], {"dpre": pp}),
                ("adj+dpre+dW (middle)", lambda: adj(pp, h, dW), fold["spectral_out adj+dpre+dW"], {"dpre": pp}),
                ("adj+dW (block 0)", lambda: adj(None, h, dW), fold["spectral_out adj+dW"], {"g": gbuf})]
    sums = {}
    for n, fn, _, outs in variants:
        pp.copy_(pre0)
        fn()
        torch.cuda.synchronize()
        sums[n] = {k: checksum(t) for k, t in outs.items()}
    pp.copy_(pre0)
    times = {n: [] for n, _, _, _ in variants}
    for _ in range(a.rounds):
        for n, fn, _, _ in variants:
            times[n].append(time_ms(fn, a.iters, a.warmup))
    res = {}
    print(f"P = {P}: L = {L} lines (Y_local = {pl.Yl}), K1 = {K1}")
    for n, _, nbytes, _ in variants:
        ms = statistics.median(times[n])
        share = nbytes / (H100_COPY_GBS * 1e9) * 1e3 / ms
        res[n] = {"ms": ms, "rounds_ms": times[n], "gb": nbytes / 1e9, "copy_share": share, "checksums": sums[n]}
        print(f"  {n:22s} {ms:7.3f} ms  (rounds {', '.join('%.3f' % t for t in times[n])})  {nbytes / 1e9:6.2f} GB  "
              f"{share:6.1%} of copy rate  {' '.join(f'{k}={v}' for k, v in sums[n].items())}")
    return {"L": L, "K1": K1, "variants": res}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ranks", type=int, nargs="+", default=[1, 2, 4, 8])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spectral_out_bench.py needs a GPU")
    C_ = build.load()
    dev = torch.device("cuda", 0)
    out = {"shape": dict(B=B, C=C, X=X, Y=Y, Z=Z, T=T, modes=MODES), "copy_gbs": H100_COPY_GBS, "ranks": {}}
    for P in a.ranks:
        out["ranks"][P] = shape_case(C_, P, dev, a)
        torch.cuda.empty_cache()
    state = gpu_state()
    out.update(state)
    print(f"{state['gpu']}  power limit {state['power_limit_w']} W  SM clock {state['sm_clock_mhz']} / "
          f"{state['sm_clock_max_mhz']} MHz")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
