"""`bench.py --impl reference`: the UNMODIFIED reference (`baseline/_ref/dfno`, installed with pip from a
checkout of slimgroup/dfno) through its own public API and stock code path --

    dfno.create_standard_partitions -> dfno.DistributedFNO -> dfno.DistributedRelativeLpLoss ->
    torch.optim.Adam, the loop of the reference's training/two_phase/train_two_phase.py:99-117

-- fp32 (the only dtype the reference supports on GPU, dfno.py:80), same 128^3 x 20 config, same timing
method as the product arm.  Nothing of `dfno_b200` (models, kernels, engine, communication layer) is
imported by this module or anything it pulls in: when the real DistDL / mpi4py are importable they are
used; otherwise the reference's `import distdl` / `from mpi4py import MPI` resolve to `baseline/compat`,
a self-contained stand-in written on plain `torch.distributed` NCCL broadcast / reduce /
all_to_all_single.  At N = 1 every DistDL layer is the identity, so that point is the pure reference.
"""
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))


def _import_reference():
    """Returns (dfno module, comm description).  Real DistDL first; the torch.distributed stand-in otherwise."""
    shim_dir = os.path.join(HERE, "compat")
    candidates = [os.path.join(HERE, "_ref"), os.path.join(os.path.dirname(HERE), "oracle", "_ref")]
    ref_dir = next((d for d in candidates if os.path.isdir(os.path.join(d, "dfno"))), None)
    if ref_dir is None:
        raise ImportError("the reference package is missing: oracle/install_reference.sh <checkout of slimgroup/dfno> "
                          "(DESIGN.md, 'Reference arm')")
    for name in [m for m in sys.modules if m == "dfno" or m.startswith("dfno.")]:
        del sys.modules[name]
    sys.path.insert(0, ref_dir)
    try:
        import distdl            # noqa: F401
        import mpi4py            # noqa: F401
        comm = "DistDL on mpi4py (as installed)"
    except ImportError:
        sys.path.insert(0, shim_dir)
        import distdl            # noqa: F401
        assert os.path.abspath(distdl.__file__).startswith(shim_dir)
        comm = "stock model code on NCCL DistDL shim (baseline/compat: torch.distributed broadcast/reduce/all_to_all_single)"
    import dfno
    assert os.path.abspath(dfno.__file__).startswith(ref_dir), dfno.__file__
    return dfno, comm


def run(args, ClockSampler):
    rank = int(os.environ.get("RANK", "0"))
    try:
        import torch
        import torch.distributed as dist
        on_gpu = args.device == "cuda"
        local = int(os.environ.get("LOCAL_RANK", "0"))
        if on_gpu:
            torch.cuda.set_device(local)
        else:
            os.environ["USE_CUDA"] = "0"
        ref, comm = _import_reference()
    except Exception as e:                     # noqa: BLE001
        if rank == 0:
            print(json.dumps({"impl": "reference", "unavailable": f"{type(e).__name__}: {e}"[:300]}))
        return 0
    assert "dfno_b200" not in sys.modules, "the reference arm must not load this repository's package"

    N = args.gpus
    dev = torch.device("cuda", local) if on_gpu else torch.device("cpu")
    G, T = args.grid, args.nt
    in_shape = [args.batch, args.in_channels, G, G, G, getattr(args, 'tin', 1)]
    grid = tuple(args.partition) if args.partition else (1, 1, 1, N, 1, 1)
    _, P_x, _ = ref.create_standard_partitions(grid)          # joins the torchrun job (mpirun's role)
    world = dist.get_world_size() if dist.is_initialized() else 1
    assert world == N, f"world size {world} != --gpus {N}"
    torch.manual_seed(123 + rank)

    net = ref.DistributedFNO(P_x, in_shape, T, args.width, list(args.modes), num_blocks=args.blocks,
                             device=dev, dtype=torch.float32)
    crit = ref.DistributedRelativeLpLoss(P_x).to(dev)
    params = [p for p in net.parameters() if p.numel() > 0]    # zero-volume placeholders own nothing
    opt = torch.optim.Adam(params, lr=1e-3)

    x_shape = [int(v) for v in ref.compute_distribution_info(P_x, in_shape)["shape"]]
    y_shape = [int(v) for v in ref.compute_distribution_info(P_x, [args.batch, 1, G, G, G, T])["shape"]]
    x_host, y_host = torch.randn(*x_shape), torch.randn(*y_shape)
    if on_gpu:
        x_host, y_host = x_host.pin_memory(), y_host.pin_memory()
    x_dev, y_dev = x_host.to(dev), y_host.to(dev)

    def step(xd, yd):                          # train_two_phase.py:101-117
        opt.zero_grad()
        loss = crit(net(xd), yd)
        loss.backward()
        opt.step()
        return loss

    def step_device():
        return step(x_dev, y_dev)

    def step_e2e():                            # host batch in (pinned), loss value out
        return float(step(x_host.to(dev, non_blocking=True), y_host.to(dev, non_blocking=True)))

    def sync_all():
        if N > 1:
            dist.barrier()
        if on_gpu:
            torch.cuda.synchronize()

    def timed(fn, steps):
        sync_all()
        if on_gpu:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        if on_gpu:
            e.record()
        sync_all()
        ms = torch.tensor([s.elapsed_time(e) if on_gpu else (time.perf_counter() - t0) * 1e3],
                          device=dev, dtype=torch.float64)
        if N > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    sampler = ClockSampler(local)
    if rank == 0 and on_gpu:
        sampler.start()
    warm = max(args.warmup, 3)
    last = None
    for _ in range(warm):
        last = step_device()
    total = timed(step_device, args.steps)
    clocks = sampler.stop() if (rank == 0 and on_gpu) else None
    ms_step = total / args.steps
    e2e = None
    if not args.no_e2e:
        for _ in range(2):
            step_e2e()
        e2e_ms = timed(step_e2e, args.steps) / args.steps
        e2e = {"value": args.batch * 1000.0 / e2e_ms, "unit": "samples/s", "ms_per_step": e2e_ms,
               "h2d_bytes_per_step": x_host.numel() * 4 + y_host.numel() * 4, "d2h_bytes_per_step": 4,
               "how": "reference loop: pinned host batch -> H2D -> fwd+loss+bwd+Adam -> float(loss)"}
    peak = torch.cuda.max_memory_allocated(dev) if on_gpu else 0
    if rank == 0:
        print(json.dumps({
            "metric": "3D Navier-Stokes FNO training step (fwd+loss+bwd+Adam) samples/sec, whole job, device-timed, max over ranks",
            "value": args.batch * 1000.0 / ms_step, "unit": "samples/s", "n_gpus": N, "steps": args.steps,
            "warmup": warm, "ms_per_step": ms_step, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "fp32", "data": "synthetic (random fields, random-init weights)",
            "impl": "reference", "reference_class": comm,
            "config": {"model": f"FNO3d+t {G}^3x{T}t width {args.width} modes {tuple(args.modes)} blocks {args.blocks}",
                       "global_batch": args.batch, "seq_len": G * G * G * T,
                       "parallelism": f"P_x = {grid} (reference planner: P_m, P_y derived by dfno.py:82-97)",
                       "l2": "per-step working set (GBs of fp32 activations) exceeds the 50 MB L2 of an H100; no flush needed",
                       "step": "forward + DistributedRelativeLpLoss + backward + torch.optim.Adam"},
            "clocks": clocks, "e2e": e2e, "loss": float(last) if last is not None else None,
            "peak_mem_gb": peak / 2 ** 30, "gpu_launches": None}))
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()
    return 0
