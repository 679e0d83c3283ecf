#!/usr/bin/env python
"""Inference with a trained two-phase model: rebuild the network, load this rank's
``model_{rank:04d}.pt``, predict one validation sample, gather input / truth / prediction onto
the root with ``Repartition(P_x, P_root)`` and save them
(reference ``training/two_phase/test_two_phase.py``; the reference's 3-vs-2 input-channel
mismatch at ``:69`` is not reproduced)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch
import dfno_b200 as d

ap = argparse.ArgumentParser()
ap.add_argument("--shape", type=int, nargs=4, default=[60, 60, 64, 30])
ap.add_argument("--width", type=int, default=20)
ap.add_argument("--modes", type=int, nargs=4, default=[12, 12, 12, 8])
ap.add_argument("--out-dir", default="data/")
ap.add_argument("--sample", type=int, default=801)
ap.add_argument("--dtype", default="auto", choices=["auto", "bf16", "fp32"])
args = ap.parse_args()

d.ensure_process_group()
n = d.world_size()
P_world, P_x, P_root = d.create_standard_partitions((1, 1, 1, n, 1, 1))
use_cuda, _, _, device, ctx = d.get_env(P_x, num_gpus=max(torch.cuda.device_count(), 1))
dtype = {"auto": torch.bfloat16 if use_cuda else torch.float32, "bf16": torch.bfloat16, "fp32": torch.float32}[args.dtype]
shape = tuple(args.shape)
collect = [d.Repartition(P_x, P_root) for _ in range(3)]
data = d.DistributedFieldDataset(P_x, [args.sample], d.SyntheticTwoPhaseStore(shape), shape)
net = d.DistributedFNO(P_x, [1, 2, *shape[:-1], 1], shape[-1], args.width, args.modes, device=device, dtype=dtype)
d.load_checkpoint(net, args.out_dir, epoch=None, restore_rng=False, map_location=device)
net.eval()
x, y = data[0]
x, y = x.unsqueeze(0).to(device), y.unsqueeze(0).to(device)
with ctx, torch.no_grad():
    fused = isinstance(net, d.FusedDistributedFNO)
    y_ = net(x if fused else x.to(dtype)).float()
    xg, yg, pg = collect[0](x), collect[1](y), collect[2](y_)
if P_root.active:
    np.savez(os.path.join(args.out_dir, "fno_sample.npz"), x=xg.cpu().numpy(), y=yg.cpu().numpy(), y_=pg.cpu().numpy())
    rel = float((pg - yg).norm() / yg.norm())
    print(f"Saved data sample! relative L2 error of the prediction: {rel:.4f}")
    try:                                                    # optional picture (matplotlib is not in this image)
        import matplotlib
        matplotlib.use("Agg")
        import matplotlib.pyplot as plt
        idx = shape[1] // 2
        fig, ax = plt.subplots(1, 3)
        ax[0].imshow(xg[0, 0, :, idx, :, 0].cpu().T); ax[1].imshow(yg[0, 0, :, idx, :, -1].cpu().T)
        ax[2].imshow(pg[0, 0, :, idx, :, -1].cpu().T)
        plt.savefig(os.path.join(args.out_dir, "pred.png"))
    except ImportError:
        pass
d.shutdown()
