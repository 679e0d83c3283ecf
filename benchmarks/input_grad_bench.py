"""Cost of input gradients (dL/dx) on the fused engine, timed with CUDA events on one GPU.  Prints one line per
measurement, the device name and power limit read in the same run, and one JSON line; writes nothing.

    python benchmarks/input_grad_bench.py [--iters 10] [--warmup 3] [--rounds 3] [--only headline|navier_stokes]

Two shapes, both with 4 Fourier blocks and width 20:
* headline: 128^3 x 20, modes (12, 12, 12, 10), Tin = 1, batch 1 (bench.py's flagship configuration);
* navier_stokes: [10, 1, 64, 64, 10] -> T = 40, modes (4, 4, 4) (the reference Navier-Stokes trainer's default).

For each, a forward plus backward (a) with weight gradients only, as in training, (b) with dx as well, (c) with frozen
weights and dx only (inversion), and lift_bwd alone with and without dx.  The three steps are alternated over
``--rounds`` rounds and the median is reported."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchmarks.head_bench import gpu_state, time_ms  # noqa: E402

SHAPES = {
    "headline": dict(in_shape=[1, 1, 128, 128, 128, 1], T=20, modes=(12, 12, 12, 10)),
    "navier_stokes": dict(in_shape=[10, 1, 64, 64, 10], T=40, modes=(4, 4, 4)),
}


def run_shape(name, cfg, a):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    dev = torch.device("cuda", 0)
    _, P_x, _ = d.create_standard_partitions([1] * len(cfg["in_shape"]))
    net = FusedDistributedFNO(P_x, cfg["in_shape"], cfg["T"], 20, cfg["modes"], num_blocks=4, device=dev,
                              init_seed=0, input_grad=True)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(*cfg["in_shape"], device=dev, generator=g)
    oshape = list(cfg["in_shape"]); oshape[1] = 1; oshape[-1] = cfg["T"]
    w = torch.randn(*oshape, device=dev, generator=g) * 1e-6          # a loss gradient of realistic scale
    xg = x.clone().requires_grad_()

    def step(theta_grad, dx):
        net.theta.requires_grad_(theta_grad)
        xin = xg if dx else x
        net(xin).backward(w)
        if dx:
            xg.grad = None

    steps = {"a_theta": (True, False), "b_theta_dx": (True, True), "c_frozen_dx": (False, True)}
    ms = {k: [] for k in steps}
    for _ in range(a.rounds):
        for k, (tg, dx) in steps.items():
            ms[k].append(time_ms(lambda: step(tg, dx), a.iters, a.warmup))
    net.theta.requires_grad_(True)
    # lift_bwd alone, on the block-0 input gradient the last backward left in the engine's workspace
    pl = net.plan
    x6 = x.view(pl.B, pl.Cin, pl.X, pl.Yl, pl.Z, pl.Tin)
    scratch = torch.zeros(pl.n_small, device=dev)
    segs = [net._seg(n) for n in ("linear1.W", "linear1.b", "linear2.W", "linear2.b")]
    gsegs = [net._seg(n, scratch) for n in ("linear1.W", "linear1.b", "linear2.W", "linear2.b")]
    dxbuf = torch.empty(x6.shape, device=dev)
    lift = {}
    for k, dx in (("lift_bwd", None), ("lift_bwd_dx", dxbuf)):
        lift[k] = time_ms(lambda: net._C.lift_bwd(x6, *segs, net.ws["g"], *gsegs, net._lift_dims(), dx),
                          a.iters * 5, a.warmup)
    res = {k: round(statistics.median(v), 3) for k, v in ms.items()}
    res.update({k: round(v, 4) for k, v in lift.items()})
    res["rounds"] = {k: [round(t, 3) for t in v] for k, v in ms.items()}
    for k, v in ms.items():
        print(f"{name:14s} {k:12s} {statistics.median(v):9.3f} ms   (rounds: {', '.join(f'{t:.3f}' for t in v)})")
    for k, v in lift.items():
        print(f"{name:14s} {k:12s} {v:9.4f} ms")
    del net
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", choices=sorted(SHAPES), default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("input_grad_bench.py needs a GPU")
    torch.cuda.set_device(0)
    out = {"iters": a.iters, "warmup": a.warmup, "shapes": {}}
    for name, cfg in SHAPES.items():
        if a.only in (None, name):
            out["shapes"][name] = run_shape(name, cfg, a)
    out.update(gpu_state())
    print(f"{out['gpu']}, power limit {out['power_limit_w']} W, SM clock {out['sm_clock_mhz']} MHz "
          f"(max {out['sm_clock_max_mhz']})")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
