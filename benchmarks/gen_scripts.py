#!/usr/bin/env python
"""Generate weak-scaling run scripts (``{eval,grad}_weak_scaling_{spatial,temporal}_gpu.sh``)
and a driver ``submit_<system>.sh`` -- the role of reference ``benchmarks/gen_scripts.py``
(Summit/Perlmutter tables at ``:119-161``), re-targeted at one-process-per-GPU ``torchrun``
launches on NVSwitch boxes:

* ``h100``        : one 8 x H100 box, 64^3 x 32 per GPU, the field grows in x, y and z (grids up to 2x2x2)
* ``h100-pencil`` : the same box, 1 x N y-pencils at 128 x 16 x 128 x 20 per GPU
* ``local``       : CPU/gloo development runs, N <= 4

"spatial" grows the partitioned extents (and their modes) with the grid at fixed per-GPU size; "temporal"
keeps space fixed and grows ``nt`` and ``modes_t`` with N -- the reference's two scaling modes
(``gen_scripts.py:44-52``).  Zero-size shards are rejected at generation time (``:55-63``).
"""
import os
from argparse import ArgumentParser
from pathlib import Path

ap = ArgumentParser()
ap.add_argument("--system", default="h100", choices=["h100", "h100-pencil", "local"])
ap.add_argument("--max-workers", "-mw", type=int, default=-1)
ap.add_argument("--clean-old", "-co", action="store_true")
ap.add_argument("--out", type=Path, default=Path(os.path.dirname(os.path.abspath(__file__))))
args = ap.parse_args()

SYSTEMS = {
    # per-GPU local shape (X, Y, Z, T), per-GPU modes, device, dtype, and the worker grids of the scaling series.
    # "h100": one 8 x H100 NVSwitch box.  Like the reference's Perlmutter table (gen_scripts.py:141-153: 64^3 x 32 per
    # GPU, 4 modes / axis / GPU) the volume grows in every spatial axis -- 1, 2, 4, 8 GPUs = (1,1,1), (1,2,1), (2,2,1),
    # (2,2,2) -- so the 4- and 8-GPU points exercise the general-partition path (folded onto the engine's y-pencil);
    # "h100-pencil" is the 1 x N y-pencil series (BASELINE config 2's layout) at 128 x 16 x 128 x 20 per GPU.
    "h100": dict(shape=(64, 64, 64, 32), modes=(4, 4, 4, 4), device="cuda", dtype="bf16",
                 grids={1: (1, 1, 1, 1, 1, 1), 2: (1, 1, 1, 2, 1, 1), 4: (1, 1, 2, 2, 1, 1), 8: (1, 1, 2, 2, 2, 1)}),
    "h100-pencil": dict(shape=(128, 16, 128, 20), modes=(12, 2, 12, 10), device="cuda", dtype="bf16",
                        grids={n: (1, 1, 1, n, 1, 1) for n in (1, 2, 4, 8)}),
    "local": dict(shape=(16, 8, 16, 8), modes=(4, 2, 4, 4), device="cpu", dtype="fp32",
                  grids={1: (1, 1, 1, 1, 1, 1), 2: (1, 1, 1, 2, 1, 1), 4: (1, 1, 2, 2, 1, 1)}),
}
cfg = SYSTEMS[args.system]
counts = [n for n in cfg["grids"] if args.max_workers < 0 or n <= args.max_workers]


def launcher(n):
    return (f"python -m torch.distributed.run --nnodes=1 --nproc-per-node {n} --master-addr 127.0.0.1 "
            f"--master-port $((29500 + RANDOM % 1000)) bench.py")


def point(n, mode):
    """(global input shape, modes, nt, worker grid) of one scaling point.  "spatial": per-GPU block fixed, the global
    field and its retained modes grow with the grid in every partitioned axis; "temporal": the global space of the
    LARGEST grid stays fixed and nt / modes_t grow with the worker count (reference gen_scripts.py:44-52)."""
    X, Y, Z, T = cfg["shape"]
    mx, my, mz, mt = cfg["modes"]
    part = cfg["grids"][n]
    px, py, pz = part[2], part[3], part[4]
    if mode == "spatial":
        shape, modes, nt = (1, 1, X * px, Y * py, Z * pz, 1), (mx * px, my * py, mz * pz, mt), T
    else:
        big = cfg["grids"][max(cfg["grids"])]
        shape = (1, 1, X * big[2], Y * big[3], Z * big[4], 1)
        modes, nt = (mx * big[2], my * big[3], mz * big[4], mt * n), T * n
    sp = shape[2:5]
    if any(p > s for p, s in zip((px, py, pz), sp)) or any(2 * m > s for m, s in zip(modes[:3], sp)) \
            or modes[3] > nt // 2 + 1:
        raise ValueError(f"invalid configuration {shape} / {modes} / {part}: a shard would be empty")
    return shape, modes, nt, part


def make(name, run_type, mode):
    lines = ["#!/bin/bash", "set -x", f"data_dir={name}",
             'if test "x$1" = x; then echo "Usage: $0 <numranks>"; exit 0; fi', "ranks=$1"]
    for n in counts:
        shape, modes, nt, part = point(n, mode)
        lines.append(f"[[ $ranks -eq '{n}' ]] && {launcher(n)} --input-shape {' '.join(map(str, shape))} "
                     f"--modes {' '.join(map(str, modes))} --partition_shape {' '.join(map(str, part))} --width 20 "
                     f"--num-timesteps {nt} --device {cfg['device']} --num-gpus {n} --dtype {cfg['dtype']} "
                     f"--benchmark-type {run_type} --output-dir $data_dir")
    path = args.out / f"{name}.sh"
    path.write_text("\n".join(lines) + "\n")
    os.chmod(path, 0o755)
    print(f"created script for {args.system}: {path.name}")
    return [f"./{path.name} {n}" for n in counts]


args.out.mkdir(parents=True, exist_ok=True)
if args.clean_old:
    for f in args.out.glob("*_weak_scaling_*_gpu.sh"):
        f.unlink()
jobs = []
for run_type in ("eval", "grad"):
    for mode in ("spatial", "temporal"):
        jobs += make(f"{run_type}_weak_scaling_{mode}_gpu", run_type, mode)
sub = args.out / f"submit_{args.system}.sh"
sub.write_text("#!/bin/bash\nset -x\ncd \"$(dirname \"$0\")\"\n" + "\n".join(jobs) + "\n")
os.chmod(sub, 0o755)
print(f"created batch submission script: {sub.name}")
