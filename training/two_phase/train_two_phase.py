#!/usr/bin/env python
"""Two-phase (CO2 plume) FNO training -- the workflow of
reference ``training/two_phase/train_two_phase.py`` (4-way y-pencil, field 60x60x64x30,
width 20, modes (12,12,12,8), 2 input channels, relative-L2 loss, Adam 1e-3, checkpoint every
10 epochs, loss history on the root) on this framework:

    python -m torch.distributed.run --nproc-per-node 4 --master-addr 127.0.0.1 \
        training/two_phase/train_two_phase.py [--data-dir DIR | synthetic by default]

Differences by design: data comes from a synthetic / ``.npy`` store (no Azure blob in this
environment), training state (optimizer, RNG, epoch) is checkpointed so runs can *resume*
(``--resume``), and the loss history is written as JSON (h5py is not installed).
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
import dfno_b200 as d

ap = argparse.ArgumentParser()
ap.add_argument("--shape", type=int, nargs=4, default=[60, 60, 64, 30], help="X Y Z T")
ap.add_argument("--partition", type=int, nargs=6, default=None)
ap.add_argument("--width", type=int, default=20)
ap.add_argument("--modes", type=int, nargs=4, default=[12, 12, 12, 8])
ap.add_argument("--num-train", type=int, default=800)
ap.add_argument("--num-valid", type=int, default=200)
ap.add_argument("--epochs", type=int, default=100)
ap.add_argument("--checkpoint-interval", type=int, default=10)
ap.add_argument("--lr", type=float, default=1e-3)
ap.add_argument("--out-dir", default="data/")
ap.add_argument("--data-dir", default=None, help="directory of <name>_<i>.npy files; default: synthetic")
ap.add_argument("--cache-dir", default=None)
ap.add_argument("--resume", action="store_true")
ap.add_argument("--dtype", default="auto", choices=["auto", "bf16", "fp32"])
d.add_optimizer_args(ap)
args = ap.parse_args()

d.ensure_process_group()
n = d.world_size()
grid = tuple(args.partition) if args.partition else (1, 1, 1, n, 1, 1)
P_world, P_x, P_root = d.create_standard_partitions(grid)
use_cuda, _, _, device, ctx = d.get_env(P_x, num_gpus=max(torch.cuda.device_count(), 1))
dtype = {"auto": torch.bfloat16 if use_cuda else torch.float32, "bf16": torch.bfloat16, "fp32": torch.float32}[args.dtype]

with ctx:
    d.seed_all(P_x.rank)
    nb, shape = 1, tuple(args.shape)
    store = d.NpyDirStore(args.data_dir) if args.data_dir else d.SyntheticTwoPhaseStore(shape)
    train = d.DistributedFieldDataset(P_x, range(1, args.num_train + 1), store, shape, savepath=args.cache_dir)
    valid = d.DistributedFieldDataset(P_x, range(args.num_train + 1, args.num_train + args.num_valid + 1), store,
                                      shape, savepath=args.cache_dir)
    train_loader = torch.utils.data.DataLoader(train, batch_size=nb, shuffle=False)
    valid_loader = torch.utils.data.DataLoader(valid, batch_size=nb, shuffle=False)
    P_world._comm.Barrier()

    net = d.DistributedFNO(P_x, [nb, 2, *shape[:-1], 1], shape[-1], args.width, args.modes, device=device, dtype=dtype)
    fused = isinstance(net, d.FusedDistributedFNO)
    d.print0(f"backend = {'fused sm_90a engine' if fused else 'portable (torch.fft / torch.distributed)'}, dtype = {dtype}")
    criterion = d.DistributedRelativeLpLoss(P_x).to(device)
    optimizer, scheduler, clip = d.make_optimizer(net, args, fused, lr=args.lr, group=P_x.group)
    trainer = d.Trainer(net, criterion, optimizer, device=device, before_step=clip) if optimizer is not None else None
    start, hist = 0, {"train": [], "valid": []}
    log = d.get_logger("two_phase")
    metrics = d.MetricsWriter(args.out_dir)                 # metrics_0000.jsonl on the root
    if args.resume:
        last = d.latest_checkpoint(args.out_dir, max(P_x.rank, 0))
        if last is not None:
            info = d.load_checkpoint(net, args.out_dir, epoch=last, optimizer=optimizer, scheduler=scheduler)
            start, hist = last, info.get("history", hist)
            if P_root.active:
                print(f"resumed from epoch {last}")

    def to_in(t):
        return t.to(torch.float32 if fused else dtype)

    for epoch in range(start, args.epochs):
        net.train()
        tot, nbat = 0.0, 0
        for j, (x, y) in enumerate(train_loader):
            t0 = time.time()
            loss = trainer.step(to_in(x), y.float())
            tot, nbat = tot + loss, nbat + 1
            P_x._comm.Barrier()
            if j % 50 == 0:
                log.info(f"epoch = {epoch}, batch = {j}, loss = {loss:.6f}, dt = {time.time() - t0:.3f}")
                metrics.log(step=epoch * len(train_loader) + j, epoch=epoch, loss=loss, dt=time.time() - t0)
        if scheduler is not None:
            scheduler.step()
        net.eval()
        vtot, vbat = 0.0, 0
        for x, y in valid_loader:
            vtot, vbat = vtot + trainer.evaluate(to_in(x), y.float()), vbat + 1
        if P_root.active:
            hist["train"].append(tot / max(nbat, 1)); hist["valid"].append(vtot / max(vbat, 1))
            log.info(f"epoch = {epoch}, train loss = {hist['train'][-1]:08f}, val loss = {hist['valid'][-1]:08f}")
            metrics.log(epoch=epoch, train_loss=hist["train"][-1], valid_loss=hist["valid"][-1])
        if (epoch + 1) % args.checkpoint_interval == 0:
            path = d.save_checkpoint(net, args.out_dir, epoch=epoch + 1, optimizer=optimizer, scheduler=scheduler,
                                     extra={"history": hist, "plan": "fused" if fused else "reference"})
            if P_root.active:
                with open(os.path.join(args.out_dir, f"loss_epoch_{epoch}.json"), "w") as f:
                    json.dump(hist, f)
            print(f"rank = {P_x.rank}, saved model: {path}")
    path = d.save_checkpoint(net, args.out_dir, epoch=None, optimizer=optimizer, scheduler=scheduler,
                             extra={"history": hist})
    print(f"rank = {P_x.rank}, saved model after final iteration: {path}")
    metrics.close()
    d.print0("training finished.")
d.shutdown()
