#!/usr/bin/env python
"""Per-kernel time breakdown of one training step (torch.profiler / CUPTI).  Not a benchmark:
numbers taken under a profiler are only used as *shares* to decide what to optimise."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import dfno_b200 as d

ap = argparse.ArgumentParser()
ap.add_argument("--impl", default="fused")
ap.add_argument("--grid", type=int, default=128)
ap.add_argument("--out", default="bench_out/profile_step.txt")
args = ap.parse_args()

d.ensure_process_group()
N = d.world_size()
dev = torch.device("cuda", torch.cuda.current_device() if N > 1 else 0)
G, T = args.grid, 20
_, P_x, _ = d.create_standard_partitions((1, 1, 1, N, 1, 1))
net = d.DistributedFNO(P_x, [1, 1, G, G, G, 1], T, 20, (12, 12, 12, 10), device=dev, dtype=torch.bfloat16,
                       backend="fused" if args.impl == "fused" else "torch")
opt = d.FusedAdam(net) if args.impl == "fused" else torch.optim.Adam([p for p in net.parameters() if p.numel()], lr=1e-3)
crit = d.DistributedRelativeLpLoss(P_x)
x = torch.randn(1, 1, G, G // N, G, 1, device=dev, dtype=torch.float32 if args.impl == "fused" else torch.bfloat16)
y = torch.randn(1, 1, G, G // N, G, T, device=dev)


def step():
    opt.zero_grad(set_to_none=True)
    loss = crit(net(x), y)
    loss.backward()
    opt.step()


for _ in range(2):
    step()
torch.cuda.synchronize()
from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
tab = prof.key_averages().table(sort_by="cuda_time_total", row_limit=45, max_name_column_width=70)
if P_x.rank == 0:
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(tab)
    print(tab)
    # busy vs wall: how much of the step the GPU spends outside kernels (launch gaps, waits)
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    if ev:
        t0 = min(e.time_range.start for e in ev); t1 = max(e.time_range.end for e in ev)
        busy = sum(e.time_range.end - e.time_range.start for e in ev)
        print(f"GPU span {(t1 - t0) / 1e3:.3f} ms, sum of kernel durations {busy / 1e3:.3f} ms, kernels {len(ev)}")
d.shutdown()
