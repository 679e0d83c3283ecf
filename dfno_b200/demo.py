"""Smoke demo: ``python -m dfno_b200.demo`` (or under torchrun with 4 ranks).

Counterpart of the ``__main__`` block of reference ``dfno/dfno.py:355-389``: build a
64^3 network with 30 output steps, run a few forward/backward passes and print per-rank
times -- device-timed instead of bare host clocks."""
import time

import torch

import dfno_b200 as d


def main(iters: int = 5) -> None:
    d.ensure_process_group()
    ws = d.world_size()
    grid = (1, 1, 1, ws, 1, 1) if torch.cuda.is_available() else (1, 1, 2, 2, 1, 1) if ws == 4 else (1, 1, ws, 1, 1, 1)
    _, P_x, P_0 = d.create_standard_partitions(grid)
    use_cuda, _, _, device, ctx = d.get_env(P_x, num_gpus=max(torch.cuda.device_count(), 1))
    n = 64 if use_cuda else 16
    width, modes, nt = 20, (4, 4, 4, 8), 30 if use_cuda else 16
    in_shape = (1, 1, n, n, n, 1)
    info = d.compute_distribution_info(P_x, in_shape)
    with ctx:
        x = torch.rand(*[int(s) for s in info["shape"]], device=device)
        net = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=4, device=device,
                               dtype=torch.bfloat16 if use_cuda else torch.float32)
        crit = d.DistributedMSELoss(P_x)
        y = net(x)
        for i in range(iters):
            sync = torch.cuda.synchronize if use_cuda else (lambda: None)
            sync(); t0 = time.perf_counter()
            y = net(x)
            sync(); t1 = time.perf_counter()
            loss = crit(y, torch.rand_like(y))
            P_x._comm.Barrier()
            sync(); t2 = time.perf_counter()
            loss.backward()
            sync(); t3 = time.perf_counter()
            print(f"rank = {P_x.rank}, backend = {type(net).__name__}, dt = {t1 - t0:.4f}, dt_grad = {t3 - t2:.4f}")
    d.shutdown()


if __name__ == "__main__":
    main()
