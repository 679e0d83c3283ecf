#!/usr/bin/env python
"""Exposed all-to-all time per SpectralConv (BASELINE.json metric): time the spectral chain of
one Fourier layer on N GPUs (a) as shipped -- mode slabs scattered to their owner GPUs from
the GEMM epilogues over NVLink + flag barriers -- and (b) with the same kernels writing the
same bytes into *local* memory and no barrier (the comm-off counterfactual).  The difference
is the communication time that is not hidden behind the math.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 benchmarks/exposed_a2a.py
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import dfno_b200 as d

d.ensure_process_group()
N, rank = d.world_size(), d.world_rank()
dev = torch.device("cuda", torch.cuda.current_device())
G, T = int(os.environ.get("G", 128)), 20
_, P_x, _ = d.create_standard_partitions((1, 1, 1, N, 1, 1))


def timed(fn, iters=20):
    for _ in range(5):
        fn()
    if N > 1:
        dist.barrier()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    if N > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device=dev)
    if N > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def measure(staged):
    os.environ["DFNO_STAGED_SCATTER"] = "1" if staged else "0"
    net = d.DistributedFNO(P_x, [1, 1, G, G, G, 1], T, 20, (12, 12, 12, 10), device=dev, dtype=torch.bfloat16, backend="fused")
    net._ensure_eval_buffers()
    net._eval_mode = True
    pl = net.plan
    src = torch.randn(pl.n_act, device=dev).to(torch.bfloat16)
    dst = torch.empty_like(src)

    def chain():
        net._spectral_chain(src, dst, 0, adj=False)

    t_comm = timed(chain)
    # counterfactual: every "peer" pointer is the local buffer, barrier disabled
    world_saved, barrier_saved = net.world, net.barrier
    net.barrier = lambda: None
    peer_saved = (net.sym_S1.peer_ptrs, net.sym_T1.peer_ptrs) if N > 1 else None
    if N > 1:
        net.sym_S1.peer_ptrs = lambda off=0: [net.sym_S1.local_ptr + off] * N
        net.sym_T1.peer_ptrs = lambda off=0: [net.sym_T1.local_ptr + off] * N
    t_local = timed(chain)
    if N > 1:
        net.sym_S1.peer_ptrs, net.sym_T1.peer_ptrs = peer_saved
    net.barrier = barrier_saved
    bytes_out = (pl.n_S1 + pl.n_T1 * pl.mt // pl.mtp) * 2 * (N - 1) // N      # bf16 bytes leaving this rank per chain
    res = {"n_gpus": N, "staged_scatter": net.plan.staged, "spectral_chain_ms": t_comm, "spectral_chain_comm_off_ms": t_local,
           "exposed_all_to_all_ms_per_spectral_conv": max(t_comm - t_local, 0.0),
           "bytes_leaving_rank_per_chain": bytes_out,
           "link_time_at_450GBps_datasheet_ms": bytes_out / 450e9 * 1e3,
           "hidden_fraction": None if N == 1 else 1.0 - max(t_comm - t_local, 0.0) / max(bytes_out / 450e9 * 1e3, 1e-9)}
    return res


variants = [measure(False)] + ([measure(True)] if N > 1 and os.environ.get("AB", "1") != "0" else [])
res = dict(variants[0])
if len(variants) > 1:
    res["staged_variant"] = variants[1]
if rank == 0:
    print(json.dumps(res))
    os.makedirs("bench_out", exist_ok=True)
    json.dump(res, open(f"bench_out/exposed_a2a_{N}gpu.json", "w"), indent=1)
d.shutdown()
