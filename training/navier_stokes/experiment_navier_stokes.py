#!/usr/bin/env python
"""2-D Navier-Stokes (space x space x time) FNO experiment -- the workflow of
reference ``training/navier_stokes/experiment_navier_stokes.py``: the root rank loads and
normalises the trajectories, the data set is scattered root -> ``P_x`` with a Repartition
(``:91-93``), training uses Adam(1e-3, wd 1e-4) and the distributed MSE loss, predictions
are de-normalised before the loss, checkpoints are written per rank, and predictions can
be gathered back to the root.

The reference script does not run as shipped (undefined ``dim`` / ``generate_batch_indices``,
SURVEY.md §7.5); this one does.  Data: ``--input file.mat`` (scipy / mat73 if installed) or
``--synthetic`` (band-limited advected vorticity; there is no dataset in this environment).

    python -m torch.distributed.run --nproc-per-node 4 --master-addr 127.0.0.1 \
        training/navier_stokes/experiment_navier_stokes.py --synthetic -ps 1 1 2 2 1
"""
import os
import sys
import time
from argparse import ArgumentParser
from pathlib import Path

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch
import dfno_b200 as d

ap = ArgumentParser()
ap.add_argument("--input", "-i", type=Path, default=None)
ap.add_argument("--synthetic", action="store_true")
ap.add_argument("--grid", type=int, default=64)
ap.add_argument("--partition-shape", "-ps", type=int, default=(1, 1, 2, 2, 1), nargs=5)
ap.add_argument("--num-data", "-nd", type=int, default=1000)
ap.add_argument("--sampling-rate", "-sr", type=int, default=1)
ap.add_argument("--in-timesteps", "-it", type=int, default=10)
ap.add_argument("--out-timesteps", "-ot", type=int, default=40)
ap.add_argument("--num-gpus", "-ng", type=int, default=1)
ap.add_argument("--train-split", "-ts", type=float, default=0.8)
ap.add_argument("--width", "-w", type=int, default=20)
ap.add_argument("--modes", "-m", type=int, default=(4, 4, 4), nargs=3)
ap.add_argument("--decomposition-order", "-do", type=int, default=1)
ap.add_argument("--num-blocks", "-nb", type=int, default=4)
ap.add_argument("--num-epochs", "-ne", type=int, default=500)
ap.add_argument("--batch-size", "-bs", type=int, default=10)
ap.add_argument("--checkpoint-interval", "-ci", type=int, default=25)
ap.add_argument("--generate-visualization", "-gv", action="store_true")
ap.add_argument("--out-root", type=Path, default=Path("data"))
ap.add_argument("--dtype", default="auto", choices=["auto", "bf16", "fp32"],
                help="auto: bf16 on a GPU (the fused sm_90a engine serves 2-D + time problems), fp32 on the CPU")
d.add_optimizer_args(ap)
args = ap.parse_args()

d.ensure_process_group()
if int(np.prod(args.partition_shape)) != d.world_size():
    raise ValueError(f"The number of processes {d.world_size()} does not match the partition shape "
                     f"{tuple(args.partition_shape)}.")
P_world, P_x, P_0 = d.create_standard_partitions(args.partition_shape)
use_cuda, _, _, device, ctx = d.get_env(P_x, num_gpus=args.num_gpus)

with ctx:
    d.seed_all(P_x.rank)
    B = d.Broadcast(P_0, P_x)
    stamp = torch.tensor([int(time.time())], dtype=torch.float64) if P_0.active else d.zero_volume_tensor(dtype=torch.float64)
    timestamp = int(B(stamp).item())
    stem = args.input.stem if args.input is not None else "synthetic_ns"
    out_dir = args.out_root / f"{stem}_{timestamp}"
    if P_0.active:
        os.makedirs(out_dir, exist_ok=True)
        print(f"created output directory: {out_dir.resolve()}")

    T_in, T_out, sr = args.in_timesteps, args.out_timesteps, args.sampling_rate
    names = ["x_train", "x_test", "y_train", "y_test", "mu_y", "std_y"]
    data = {}
    if P_0.active:
        if args.input is not None:
            try:
                from mat73 import loadmat
            except ImportError:
                from scipy.io import loadmat
            u = torch.tensor(np.asarray(loadmat(str(args.input))["u"]), dtype=torch.float32)[:args.num_data]
        else:
            u = d.SyntheticNavierStokes.make(args.num_data, args.grid, T_in + T_out, seed=0)
        u = u.unsqueeze(1)[:, :, ::sr, ::sr]                                   # [N, 1, X, Y, T]
        x, mu_x, std_x = d.unit_guassian_normalize(u[..., :T_in])
        y, data["mu_y"], data["std_y"] = d.unit_guassian_normalize(u[..., T_in:T_in + T_out])
        split = int(args.train_split * u.shape[0])
        data.update(x_train=x[:split], x_test=x[split:], y_train=y[:split], y_test=y[split:])
        for k, v in data.items():
            print(f"{k}.shape = {tuple(v.shape)}")
    local = {}
    for k in names:                                         # scatter root -> P_x
        v = data[k].to(device) if P_0.active else d.zero_volume_tensor(device=device)
        local[k] = d.Repartition(P_0, P_x)(v)
    del data
    x_train, x_test, y_train, y_test = (local[k] for k in ("x_train", "x_test", "y_train", "y_test"))
    mu_y, std_y = local["mu_y"], local["std_y"]
    print(f"index = {P_x.index}, x_train.shape = {tuple(x_train.shape)}, y_train.shape = {tuple(y_train.shape)}")

    gshape = d.infer_global_shape(P_x, [args.batch_size, *x_train.shape[1:]])
    mdtype = {"auto": torch.bfloat16 if use_cuda else torch.float32, "bf16": torch.bfloat16, "fp32": torch.float32}[args.dtype]
    net = d.DistributedFNO(P_x, gshape, T_out, args.width, args.modes, num_blocks=args.num_blocks, device=device,
                           dtype=mdtype)
    fused = isinstance(net, d.FusedDistributedFNO)
    d.print0(f"backend = {'fused sm_90a engine' if fused else 'portable (torch.fft / torch.distributed)'}, dtype = {mdtype}")
    criterion, mse = d.DistributedMSELoss(P_x).to(device), d.DistributedMSELoss(P_x).to(device)
    optimizer, scheduler, clip = d.make_optimizer(net, args, fused, lr=1e-3, weight_decay=1e-4, group=P_x.group)
    if not fused:                                   # the fused engine takes fp32 / bf16 inputs as they are
        x_train, x_test = x_train.to(mdtype), x_test.to(mdtype)
    steps, train_accs, test_accs = [], [], []

    for i in range(args.num_epochs):
        net.train()
        tl, nb = 0.0, 0
        for j, (a, b) in enumerate(d.generate_batch_indices(P_x, x_train.shape[0], args.batch_size, shuffle=True, seed=i)):
            if b - a != args.batch_size:
                continue                                   # the model is built for a fixed batch size
            optimizer.zero_grad()
            y_hat = d.unit_gaussian_denormalize(net(x_train[a:b]), mu_y, std_y)
            y = d.unit_gaussian_denormalize(y_train[a:b], mu_y, std_y)
            loss = criterion(y_hat, y)
            loss.backward()
            if clip is not None:
                clip()
            optimizer.step()
            if P_0.active:
                tl, nb = tl + loss.item(), nb + 1
        if scheduler is not None:
            scheduler.step()
        if P_0.active:
            print(f"epoch = {i}, average train loss = {tl / max(nb, 1)}")
            steps.append(i); train_accs.append(tl / max(nb, 1))
        net.eval()
        y_true, y_pred, te, tm, nt_ = [], [], 0.0, 0.0, 0
        with torch.no_grad():
            for a, b in d.generate_batch_indices(P_x, x_test.shape[0], args.batch_size, shuffle=False):
                if b - a != args.batch_size:
                    continue
                y_hat = d.unit_gaussian_denormalize(net(x_test[a:b]), mu_y, std_y)
                y = d.unit_gaussian_denormalize(y_test[a:b], mu_y, std_y)
                te += criterion(y_hat, y).item(); tm += mse(y_hat, y).item(); nt_ += 1
                y_true.append(y); y_pred.append(y_hat)
        if P_0.active:
            print(f"average test loss = {te / max(nt_, 1)}\naverage test mse  = {tm / max(nt_, 1)}")
            test_accs.append(te / max(nt_, 1))
        if (i + 1) % args.checkpoint_interval == 0:
            path = d.save_checkpoint(net, str(out_dir), epoch=i + 1, optimizer=optimizer, scheduler=scheduler)
            print(f"saved model: {Path(path).resolve()}")
            if y_true:
                np.savez(out_dir / f"mat_{i + 1:04d}_{max(P_x.rank, 0):04d}.npz",
                         y_true=torch.cat(y_true).cpu().numpy(), y_pred=torch.cat(y_pred).cpu().numpy())
                if args.generate_visualization:             # gather P_x -> root (needs matplotlib to draw)
                    G = d.Repartition(P_x, P_0)
                    yt, yp = G(torch.cat(y_true)), G(torch.cat(y_pred))
                    if P_0.active:
                        np.savez(out_dir / f"gathered_{i + 1:04d}.npz", y_true=yt.cpu().numpy(), y_pred=yp.cpu().numpy(),
                                 steps=steps, train=train_accs, test=test_accs)
                        # the reference's plots (experiment_navier_stokes.py:198-227): loss curves + truth / prediction GIF
                        from dfno_b200.utils.viz import save_curves_png, save_field_gif
                        save_curves_png(str(out_dir / f"curves_{i + 1:04d}.png"), {"train": train_accs, "test": test_accs})
                        save_field_gif(str(out_dir / f"sample_{i + 1:04d}.gif"),
                                       {"truth": yt[0, 0].float().cpu().numpy(), "prediction": yp[0, 0].float().cpu().numpy()})
d.shutdown()
