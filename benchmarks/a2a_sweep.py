#!/usr/bin/env python
"""Repartition all-to-all bandwidth sweep (BASELINE.json config 5): P2P push kernel over
NVLink peer memory vs NCCL ``all_to_all_single``, 1 MB - 1 GB per rank, device-timed, max
over ranks.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 benchmarks/a2a_sweep.py
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import dfno_b200 as d
from dfno_b200.runtime.symm import P2PAllToAll

d.ensure_process_group()
rank, world = dist.get_rank(), dist.get_world_size()
dev = torch.device("cuda", torch.cuda.current_device())
sizes = [1 << k for k in range(20, 31)]          # bytes sent per rank (all peers together)
max_bytes = int(os.environ.get("A2A_MAX_BYTES", 1 << 30))
sizes = [s for s in sizes if s <= max_bytes]
a2a = P2PAllToAll(dist.group.WORLD, rank, world, max(sizes))
rows = []


def timed(fn, iters):
    for _ in range(3):
        fn()
    dist.barrier(); torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    dist.barrier(); torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


for nbytes in sizes:
    n = nbytes // 2 // world * world                          # bf16 elements, equal split
    send = torch.randn(n, device=dev).to(torch.bfloat16)
    recv = torch.empty_like(send)
    counts = [n // world] * world
    matrix = [counts] * world
    iters = 20 if nbytes <= (1 << 26) else 5
    t_nccl = timed(lambda: dist.all_to_all_single(recv, send), iters)
    out = a2a.exchange(send, counts, matrix)
    dist.all_to_all_single(recv, send)
    assert torch.equal(out, recv), "p2p all-to-all disagrees with NCCL"
    t_p2p = timed(lambda: a2a.exchange(send, counts, matrix, copy=False), iters)   # zero-copy receive window,
    # like NCCL writing into a caller-provided buffer
    off = n * 2 * (world - 1) / world                          # bytes leaving each rank
    rows.append({"bytes_per_rank": n * 2, "nccl_ms": t_nccl, "p2p_ms": t_p2p,
                 "nccl_GBps_out": off / t_nccl / 1e6, "p2p_GBps_out": off / t_p2p / 1e6})
    if rank == 0:
        print(json.dumps(rows[-1]), flush=True)
if rank == 0:
    os.makedirs("bench_out", exist_ok=True)
    with open(f"bench_out/a2a_sweep_{world}gpu.json", "w") as f:
        json.dump({"world": world, "link_peak_GBps_per_direction_datasheet": 450, "rows": rows}, f, indent=1)
d.shutdown()
