"""Cost of schedules, decoupled decay and gradient-norm clipping in FusedAdam, on the headline one-GPU step.

(a) The CUDA-graph training step (``Trainer(cuda_graph=True).step_on_device``: forward, loss, backward, optimizer) of
    the 128^3 x 20 network (width 20, modes 12 12 12 10, 4 blocks), in two variants alternated in one session:
      plain    FusedAdam(lr=1e-3)                                       -- the default kernel path
      sched    FusedAdam(lr=1e-3, weight_decay=1e-4, decoupled, max_grad_norm=1.0) + StepLR, stepped every replay
(b) The optimizer's kernels alone on that network's flat buffer, timed with CUDA events: the sum of squares of the
    gradient and both Adam instantiations.  The extra work of (a) is one read of the gradient (sumsq) and the small
    hyperparameter write before each replay.

    python benchmarks/optim_bench.py [--iters 20] [--rounds 5]

Prints one line per measurement and one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from many_inputs_bench import gpu_state, time_ms  # noqa: E402

IN_SHAPE, NT, MODES = [1, 1, 128, 128, 128, 1], 20, (12, 12, 12, 10)


def make(variant):
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    _, P_x, _ = d.create_standard_partitions([1] * 6)
    net = d.DistributedFNO(P_x, IN_SHAPE, NT, 20, MODES, num_blocks=4, device=dev, dtype=torch.bfloat16, init_seed=0)
    assert isinstance(net, d.FusedDistributedFNO)
    sched = None
    if variant == "plain":
        opt = d.FusedAdam(net, lr=1e-3)
    else:
        opt = d.FusedAdam(net, lr=1e-3, weight_decay=1e-4, decoupled_weight_decay=True, max_grad_norm=1.0)
        sched = torch.optim.lr_scheduler.StepLR(opt, step_size=10, gamma=0.9)
    crit = d.DistributedRelativeLpLoss(P_x, engine=net)
    tr = d.Trainer(net, crit, opt, device=dev, cuda_graph=True)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(*IN_SHAPE, device=dev, generator=g)
    tt = torch.arange(NT, device=dev, dtype=torch.float32)
    t = 0.5 * x * torch.cos(0.3 * tt) + 0.05 * torch.randn(*IN_SHAPE[:-1], NT, device=dev, generator=g)

    def one():
        tr.step_on_device(x, t)
        if sched is not None:
            sched.step()
    return net, opt, tr, one


def kernels(net, opt, iters):
    from dfno_b200.models.fused import SUMSQ_MAX_BLOCKS
    C_ = net._C._mod
    n = net.plan.n_theta
    dev = net.theta.device
    gr = net.grad_flat
    p, m, v = net.theta.data.clone(), torch.zeros_like(gr), torch.zeros_like(gr)
    step = torch.ones(1, device=dev)
    hp = torch.zeros(8, device=dev, dtype=torch.float64)
    C_.adam_set_hparams(hp, 1e-3, 0.9, 0.999, 1e-8, 1e-4, True, 1.0)
    sq, part = torch.zeros(1, device=dev, dtype=torch.float64), torch.zeros(SUMSQ_MAX_BLOCKS, device=dev,
                                                                            dtype=torch.float64)
    ticket, norm = torch.zeros(1, device=dev, dtype=torch.int32), torch.zeros((), device=dev)
    calls = {
        "sumsq": (lambda: C_.sumsq(gr, sq, part, ticket), 4 * n),
        "adam_step": (lambda: C_.adam_step(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, step), 7 * 4 * n),
        "adam_step_dev": (lambda: C_.adam_step_dev(p, gr, m, v, hp, step, 1.0, sq, norm), 7 * 4 * n),
    }
    out = {}
    for name, (fn, nbytes) in calls.items():
        ms = min(time_ms(fn, iters, 3) for _ in range(3))
        out[name] = {"ms": round(ms, 4), "GBs": round(nbytes / ms / 1e6, 1)}
        print(f"  {name:14s} {ms:7.3f} ms  {nbytes / 1e9:6.2f} GB  {nbytes / ms / 1e6:7.1f} GB/s")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    state = gpu_state()
    print(f"{state['gpu']}, power limit {state['power_limit_w']} W")
    runs = {}
    for k in ("plain", "sched"):
        runs[k] = make(k)
        time_ms(runs[k][3], a.warmup, 1)
    per = {k: [] for k in runs}
    for _ in range(a.rounds):
        for k, r in runs.items():
            per[k].append(time_ms(r[3], a.iters, 1))
    res = {k: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
           for k, v in per.items()}
    for k, v in res.items():
        print(f"step {k:6s} median {v['median_ms']:.3f} ms (min {v['min_ms']:.3f}, max {v['max_ms']:.3f}) "
              f"over {a.rounds} rounds of {a.iters}")
    delta = res["sched"]["median_ms"] - res["plain"]["median_ms"]
    print(f"delta (sched - plain): {delta:+.3f} ms")
    net, opt, tr, _ = runs["sched"]
    print(f"graph launches per step: plain {runs['plain'][2].graph_kernel_launches}, sched {tr.graph_kernel_launches}; "
          f"last grad norm {float(opt.grad_norm):.4f}, lr {opt.lr:.3e}")
    print(f"kernels on the {net.plan.n_theta * 4 / 2**30:.3f} GiB flat buffer:")
    ks = kernels(net, opt, a.iters)
    print(json.dumps({"bench": "optim", **state, "steps": res, "delta_ms": round(delta, 3), "kernels": ks,
                      "n_theta": net.plan.n_theta,
                      "graph_launches": {k: r[2].graph_kernel_launches for k, r in runs.items()}}))


if __name__ == "__main__":
    main()
