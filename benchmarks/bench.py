#!/usr/bin/env python
"""Scaling-benchmark kernel: one (input shape, partition, width, modes, nt) point.

Same CLI and per-rank JSON contract as reference ``benchmarks/bench.py:149-161`` -- keys
``dt`` (forward), ``dt_comm`` (time in repartitions/broadcasts), ``dt_comp = dt - dt_comm``
and, for ``--benchmark-type grad``, ``dt_grad`` (backward from a ones cotangent) -- but
measured properly: warm-up iterations, a barrier, and CUDA events / synchronised clocks.
File name: ``<shape>-<partition>-<width>-<modes>-<nt>-<type>-<rank>-<size>.json``.

Launch: ``python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1
benchmarks/bench.py --input-shape 1 1 64 64 64 1 --partition_shape 1 1 1 N 1 1 ...``
"""
import json
import os
import sys
import time
import traceback
from argparse import ArgumentParser
from pathlib import Path

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import dfno_b200 as d


def dls(seq, delimiter="_"):
    return delimiter.join(str(v) for v in seq)


def print0(msg, P_0):
    if P_0.active:
        print(msg, flush=True)


def bench(input_shape, partition_shape, width, modes, nt, dev, ngpu, benchmark_type, output_dir=Path("."),
          warmup=2, iters=3, backend="auto", dtype="bf16"):
    P_world, P_x, P_0 = d.create_standard_partitions(partition_shape)
    if dev == "cpu":
        device = torch.device("cpu")
    else:
        device = torch.device("cuda", torch.cuda.current_device() if torch.distributed.is_initialized()
                              else P_x.rank % max(ngpu, 1))
        torch.cuda.set_device(device)
    assert len(input_shape) == len(partition_shape) and width > 0 and len(input_shape) - 2 == len(modes) and nt > 0
    outfile = Path(f"{dls(input_shape)}-{dls(partition_shape)}-{width}-{dls(modes)}-{nt}-{benchmark_type}-"
                   f"{P_x.rank}-{P_x.size}.json")
    if P_0.active:
        os.makedirs(output_dir, exist_ok=True)
    P_x._comm.Barrier()
    data, errors = {}, False
    try:
        info = d.compute_distribution_info(P_x, input_shape)
        tdt = {"bf16": torch.bfloat16, "fp32": torch.float32, "fp64": torch.float64}[dtype]
        if device.type == "cpu" and tdt == torch.bfloat16:
            tdt = torch.float32
        x = torch.rand(*[int(s) for s in info["shape"]], device=device, dtype=torch.float32)
        net = d.DistributedFNO(P_x, list(input_shape), nt, width, list(modes), device=device, dtype=tdt,
                               backend=backend)
        if not isinstance(net, d.FusedDistributedFNO):
            x = x.to(tdt)
        sync = torch.cuda.synchronize if device.type == "cuda" else (lambda: None)

        def timed(fn):
            P_x._comm.Barrier(); sync()
            t0 = time.perf_counter()
            out = fn()
            sync()
            return out, time.perf_counter() - t0

        if benchmark_type == "eval":
            net.eval()
            with torch.no_grad():
                for _ in range(warmup):
                    net(x)
                best = None
                for _ in range(iters):
                    _, dt = timed(lambda: net(x))
                    best = dt if best is None else min(best, dt)
            data["dt"] = best
        else:
            for _ in range(warmup):
                y = net(x); y.backward(torch.ones_like(y))
            bf, bb = None, None
            for _ in range(iters):
                y, dt = timed(lambda: net(x))
                y1 = torch.ones_like(y)
                _, dg = timed(lambda: y.backward(y1))
                bf = dt if bf is None else min(bf, dt)
                bb = dg if bb is None else min(bb, dg)
            data["dt"], data["dt_grad"] = bf, bb
        data["dt_comm"] = float(getattr(net, "dt_comm", 0.0))
        data["dt_comp"] = data["dt"] - data["dt_comm"]
        data["backend"] = type(net).__name__
        data["device"] = str(device)
        with open(Path(output_dir) / outfile, "w") as f:
            json.dump(data, f)
        print0(f"{outfile}: {data}", P_0)
    except Exception:                                     # noqa: BLE001 - never hang the other ranks
        traceback.print_exc()
        errors = True
    if errors:
        os._exit(1)                                       # abort the job (reference: MPI Abort)
    return data


if __name__ == "__main__":
    ap = ArgumentParser()
    ap.add_argument("--input-shape", "-is", type=int, nargs="+", required=True)
    ap.add_argument("--partition_shape", "-ps", type=int, nargs="+", required=True)
    ap.add_argument("--width", "-w", type=int, default=20)
    ap.add_argument("--modes", "-m", type=int, nargs="+", required=True)
    ap.add_argument("--num-timesteps", "-nt", type=int, default=10)
    ap.add_argument("--device", "-d", type=str, default="cpu")
    ap.add_argument("--num-gpus", "-ngpu", type=int, default=0)
    ap.add_argument("--benchmark-type", "-bt", type=str, default="eval", choices=["eval", "grad"])
    ap.add_argument("--output-dir", "-o", type=Path, default=Path("."))
    ap.add_argument("--backend", type=str, default=os.environ.get("DFNO_BENCH_BACKEND", "auto"),
                    choices=["auto", "fused", "torch"])
    ap.add_argument("--dtype", type=str, default="bf16", choices=["bf16", "fp32", "fp64"])
    ap.add_argument("--mydummyargument", nargs="?", required=False)
    a = ap.parse_args()
    bench(a.input_shape, a.partition_shape, a.width, a.modes, a.num_timesteps, a.device, a.num_gpus,
          a.benchmark_type, a.output_dir, backend=a.backend, dtype=a.dtype)
    d.shutdown()
