"""Training step with and without ``padding``, and the padded-layout lift / head kernels at padding 0.

(a) The step (forward, loss, backward, FusedAdam) of two networks, unpadded and padded, alternated in one session:
    the Navier-Stokes default (batch 10, 64 x 64, Tin 10 -> T 40, width 20, modes 4 4 4, 4 blocks) padded by 8 in t,
    and the headline 128^3 x 20 (width 20, modes 12 12 12 10, 4 blocks) padded by 4 in t.  Printed next to the
    padded-to-interior volume ratio, the overhead the padded grid should cost.
(b) lift_fwd, lift_bwd, head_fwd and head_bwd2 alone on the headline shape without padding (the kernels every
    unpadded network runs), timed with CUDA events over many calls, to compare against a build of the parent commit.

    python benchmarks/padding_bench.py [--iters 20] [--rounds 5]

Prints one line per measurement and one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from many_inputs_bench import gpu_state, time_ms  # noqa: E402

SHAPES = {
    "navier_stokes": dict(in_shape=[10, 1, 64, 64, 10], nt=40, modes=(4, 4, 4), padding=(0, 0, 8)),
    "headline_128": dict(in_shape=[1, 1, 128, 128, 128, 1], nt=20, modes=(12, 12, 12, 10), padding=(0, 0, 0, 4)),
}


def make_step(cfg, padding):
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    _, P_x, _ = d.create_standard_partitions([1] * len(cfg["in_shape"]))
    net = d.DistributedFNO(P_x, cfg["in_shape"], cfg["nt"], 20, cfg["modes"], num_blocks=4, device=dev,
                           dtype=torch.bfloat16, padding=padding, init_seed=0)
    assert isinstance(net, d.FusedDistributedFNO)
    opt = d.FusedAdam(net, lr=1e-4)
    crit = d.DistributedRelativeLpLoss(P_x)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(*cfg["in_shape"], device=dev, generator=g)
    t = torch.randn(*cfg["in_shape"][:-1], cfg["nt"], device=dev, generator=g)

    def one():
        opt.zero_grad()
        crit(net(x), t).backward()
        opt.step()
    return net, one


def steps(cfg, a):
    nets = {}
    fns = {}
    for key, pad in (("unpadded", None), ("padded", cfg["padding"])):
        nets[key], fns[key] = make_step(cfg, pad)
        time_ms(fns[key], 1, a.warmup)
    per = {k: [] for k in fns}
    for _ in range(a.rounds):
        for k, fn in fns.items():
            per[k].append(time_ms(fn, a.iters, 1))
    ratio = nets["padded"].plan.S / nets["unpadded"].plan.S
    return per, ratio


def kernels(a):
    """(b): the four changed kernels at padding 0 on the headline shape"""
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    net, _ = make_step(SHAPES["headline_128"], None)
    pl, C_ = net.plan, net._C
    x = torch.randn(*net.in_shape, device=dev)
    g = (torch.randn(pl.n_act, device=dev) * 1e-3).to(torch.bfloat16)
    h = torch.randn(pl.n_act, device=dev).to(torch.bfloat16)
    dy = torch.randn(pl.B, 1, pl.Xi, pl.Yli, pl.Zi, pl.Ti, device=dev)
    out = torch.empty_like(dy)
    gf = torch.zeros(pl.n_theta, device=dev)
    seg = lambda n, base=None: net._seg(n, base)  # noqa: E731
    w3a, w3t = net._head_operators_cm()
    R, SR = net._head_row_digits()
    dims = net._lift_dims()
    lw = [seg("linear1.W"), seg("linear1.b"), seg("linear2.W"), seg("linear2.b")]
    lg = [seg("linear1.W", gf), seg("linear1.b", gf), seg("linear2.W", gf), seg("linear2.b", gf)]
    hg = [seg("linear3.W", gf), seg("linear3.b", gf), seg("linear4.W", gf).view(-1), seg("linear4.b", gf)]
    amax = torch.zeros(1, device=dev, dtype=torch.int32)
    gh = torch.empty_like(g)
    calls = {
        "lift_fwd": lambda: C_.lift_fwd(x, *lw, h, dims),
        "lift_bwd": lambda: C_.lift_bwd(x, *lw, g, *lg, dims, None),
        "head_fwd": lambda: C_.head_fwd(h, w3a, net._w4b4(), out, pl.B, pl.C, pl.S, R, SR),
        "head_bwd2": lambda: C_.head_bwd2(h, w3a, w3t, seg("linear4.W").view(-1), dy, amax, gh, *hg, pl.B, pl.C,
                                          pl.S, R, SR),
    }
    res = {}
    for k, fn in calls.items():
        v = [time_ms(fn, 4 * a.iters, 2) for _ in range(a.rounds)]
        res[k] = round(statistics.median(v), 4)
        print(f"{k:9s} 128^3 x 20, width 20, padding 0: median {res[k]:.4f} ms ({min(v):.4f} .. {max(v):.4f})")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the unpadded and padded steps")
    ap.add_argument("--skip-steps", action="store_true", help="only the kernels of (b)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("padding_bench.py needs a GPU")
    res = {**gpu_state(), "step_ms": {}, "kernels_ms": {}}
    if not a.skip_steps:
        for name, cfg in SHAPES.items():
            per, ratio = steps(cfg, a)
            for k, v in per.items():
                res["step_ms"][f"{name} {k}"] = round(statistics.median(v), 3)
                print(f"{name} {k:8s}: median {statistics.median(v):.3f} ms over {len(v)} windows "
                      f"({min(v):.3f} .. {max(v):.3f})")
            over = statistics.median(per["padded"]) / statistics.median(per["unpadded"])
            res["step_ms"][f"{name} overhead"] = round(over, 3)
            res["step_ms"][f"{name} volume ratio"] = round(ratio, 3)
            print(f"{name}: padded / unpadded step {over:.3f}, padded / interior volume {ratio:.3f}")
            torch.cuda.empty_cache()
    res["kernels_ms"] = kernels(a)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
