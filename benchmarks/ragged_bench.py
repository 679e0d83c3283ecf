"""Training step of the reference's two-phase workload on a ragged pencil.

The two-phase grid (60 x 60 x 64 x 30, width 20, modes 12 12 12 8, 4 blocks, batch 1) split over 8 GPUs leaves 7.5
y rows per GPU: the fused engine stores 8 per rank, 64 for 60 live, so 1/16 of its y-pencil work is dead.  Timed,
each on its own set of spawned ranks:

* ``fused P=8``: the fused engine on the ragged 8-GPU pencil;
* ``portable P=8``: the portable backend (cuFFT, cuBLAS, NCCL; fp32) on the same partition, which is what this shape
  ran on before ragged pencils;
* ``fused P=4``: the fused engine on the even 4-GPU pencil (15 rows per rank, nothing dead).

Each step is forward, relative-L2 loss, backward and the optimizer (FusedAdam / torch Adam), timed with CUDA events on
rank 0 after a barrier, over ``--iters`` steps per round, rounds alternating the three configurations.  A
configuration that needs more GPUs than the machine has is reported as not measured.

    python benchmarks/ragged_bench.py [--iters 20] [--rounds 3] [--warmup 5]

Prints one line per measurement and one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

SHAPE = dict(in_shape=[1, 1, 60, 60, 64, 1], nt=30, width=20, modes=(12, 12, 12, 8), blocks=4)
CONFIGS = [("fused", 8), ("portable", 8), ("fused", 4)]


def _rank(rank, world, backend, iters, warmup):
    import torch.distributed as dist
    import dfno_b200 as d
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    from many_inputs_bench import gpu_state
    dev = torch.device("cuda", torch.cuda.current_device())
    c = SHAPE
    grid = [1, 1, 1, world, 1, 1]
    _, P_x, _ = d.create_standard_partitions(grid)
    fused = backend == "fused"
    net = d.DistributedFNO(P_x, c["in_shape"], c["nt"], c["width"], c["modes"], num_blocks=c["blocks"], device=dev,
                           dtype=torch.bfloat16 if fused else torch.float32, backend="fused" if fused else "torch",
                           init_seed=0)
    assert isinstance(net, d.FusedDistributedFNO) == fused
    opt = d.FusedAdam(net, lr=1e-4) if fused else torch.optim.Adam(net.parameters(), lr=1e-4)
    crit = d.DistributedRelativeLpLoss(P_x, engine=net if fused else None)
    g = torch.Generator(device=dev).manual_seed(0)
    out_shape = [*c["in_shape"][:-1], c["nt"]]
    x = torch.randn(*c["in_shape"], device=dev, generator=g)[assemble_slices(*shard_bounds(c["in_shape"], grid, P_x.index))]
    t = torch.randn(*out_shape, device=dev, generator=g)[assemble_slices(*shard_bounds(out_shape, grid, P_x.index))]
    x, t = x.contiguous(), t.contiguous()

    def step():
        opt.zero_grad()
        crit(net(x), t).backward()
        opt.step()

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    res = {"ms": ms, **gpu_state()}
    if fused:
        pl = net.plan
        res.update(y_stored=pl.Y, y_live=pl.Yg, kz_stored=pl.KZ, kz_live=pl.KZg, rows_per_rank=pl.Yl)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    from dfno_b200.utils.testing import run_distributed
    have = torch.cuda.device_count()
    per = {f"{b} P={P}": [] for b, P in CONFIGS}
    info = {}
    for _ in range(a.rounds):
        for backend, P in CONFIGS:
            key = f"{backend} P={P}"
            if P > have:
                continue
            r0 = run_distributed(_rank, P, backend, a.iters, a.warmup, cuda=True, timeout=1800)[0]
            per[key].append(r0["ms"])
            info[key] = {k: v for k, v in r0.items() if k != "ms"}
    out = {"shape": SHAPE, "gpus": have, "results": {}}
    for key, ms in per.items():
        if not ms:
            print(f"{key:14s} not measured ({have} GPU(s) here)")
            out["results"][key] = None
            continue
        med = statistics.median(ms)
        extra = info[key]
        dead = (f"  y {extra['y_stored']} stored / {extra['y_live']} live = {extra['y_stored'] / extra['y_live']:.4f}"
                if "y_stored" in extra else "")
        print(f"{key:14s} {med:9.3f} ms/step (rounds {', '.join(f'{v:.3f}' for v in ms)}){dead}  "
              f"[{extra.get('gpu')}, {extra.get('power_limit_w')} W]")
        out["results"][key] = {"ms_median": med, "ms_rounds": ms, **extra}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
