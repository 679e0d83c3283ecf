#!/usr/bin/env python
"""Print what the fused engine would do for a configuration -- eligibility, per-rank memory by
category against the 80 GB of an H100, and the GEMM stage chain with its NVLink scatters -- without
touching a GPU.

    python tools/plan.py --shape 128 128 128 20 --width 20 --modes 12 12 12 10 --gpus 8
    python tools/plan.py --shape 256 256 256 16 --width 32 --modes 12 12 12 8 --gpus 8 --partition 1 1 2 2 2 1
    python tools/plan.py --shape 64 64 64 30 --width 20 --modes 8 8 8 8 --padding 0 0 0 2
    python tools/plan.py --shape 128 128 128 1 --width 20 --modes 12 12 12 1 --batch 4 --in-channels 2
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dfno_b200.models.fused import H100_COPY_GBS, HBM_BUDGET, EnginePlan, supports   # noqa: E402


class _Grid:
    def __init__(self, shape):
        self.shape, self.dim = list(shape), len(shape)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shape", type=int, nargs=4, required=True, metavar=("X", "Y", "Z", "T_out"))
    ap.add_argument("--width", type=int, default=20)
    ap.add_argument("--modes", type=int, nargs=4, required=True)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--partition", type=int, nargs=6, default=None, help="P_x (default: 1 1 1 GPUS 1 1)")
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--in-channels", type=int, default=1)
    ap.add_argument("--in-timesteps", type=int, default=1)
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("--out-channels", type=int, default=1, help="fields predicted by the network (default 1)")
    ap.add_argument("--padding", type=int, nargs=4, default=None, metavar=("PX", "PY", "PZ", "PT"),
                    help="zeros appended to the lifted field along x, y, z, t (default none)")
    ap.add_argument("--hbm-gbs", type=float, default=None,
                    help="HBM copy bandwidth for the traffic floor (default: the value measured on an H100)")
    ap.add_argument("--nvlink-gbs", type=float, default=None, help="measured peer-copy rate (default: not estimated)")
    a = ap.parse_args()
    X, Y, Z, T = a.shape
    grid = a.partition or [1, 1, 1, a.gpus, 1, 1]
    in_shape = [a.batch, a.in_channels, X, Y, Z, a.in_timesteps]
    ok, why = supports(_Grid(grid), in_shape, T, a.width, a.modes, out_channels=a.out_channels, padding=a.padding)
    print(f"P_x = {tuple(grid)}  in_shape = {in_shape}  T_out = {T}  width = {a.width}  modes = {tuple(a.modes)}"
          + (f"  out_channels = {a.out_channels}" if a.out_channels != 1 else "")
          + (f"  padding = {tuple(a.padding)}" if a.padding and any(a.padding) else ""))
    print(f"fused engine: {'yes' if ok else 'no -- ' + why}")
    P = 1
    for g in grid:
        P *= g
    pad = a.padding or (0, 0, 0, 0)
    pl = EnginePlan(a.batch, a.in_channels, a.in_timesteps, a.width, T, X, Y, Z, a.modes, world=P, rank=0,
                    out_channels=a.out_channels, pad=pad)
    pl.finish(a.blocks)
    if tuple(grid) != (1, 1, 1, P, 1, 1):
        print(f"work partition: (1, 1, 1, {P}, 1, 1) (input / output re-sharded once per step)")
    # ragged pencil: every rank stores the same extents, the entries past its balanced share are dead work
    print(f"y rows: {pl.Yl} stored per rank, {pl.Y} in all for {pl.Yg} live (storage / live {pl.Y / pl.Yg:.4f}, "
          f"dead fraction {1 - pl.Yg / pl.Y:.2%});  kz modes: {pl.kzl} stored per rank, {pl.KZ} in all for {pl.KZg} "
          f"live (storage / live {pl.KZ / pl.KZg:.4f}, dead fraction {1 - pl.KZg / pl.KZ:.2%})")
    for train in (True, False):
        m = pl.memory_bytes(train=train)
        print(f"\nper-rank memory, {'training' if train else 'inference'} "
              f"({m['total'] / 2 ** 30:.2f} GiB of a {HBM_BUDGET / 2 ** 30:.0f} GiB budget):")
        for k, v in m.items():
            if k != "total" and v:
                print(f"  {k:22s} {v / 2 ** 30:9.3f} GiB")
    peaks = {"hbm": a.hbm_gbs or H100_COPY_GBS, "link": a.nvlink_gbs}
    cm = pl.cost_model(hbm_gbs=peaks["hbm"], nvlink_gbs=peaks["link"], front=True, fold_bwd=True)
    print(f"\ntraffic of one training step per rank: {cm['hbm_bytes'] / 1e9:.2f} GB HBM -> {cm['hbm_floor_ms']:.2f} ms at "
          f"{peaks['hbm']:.0f} GB/s;  {cm['nvlink_bytes'] / 1e6:.0f} MB over NVLink" +
          (f" -> {cm['nvlink_ms']:.3f} ms at {peaks['link']:.0f} GB/s (overlappable)" if peaks["link"] else
           " (no measured NVLink rate)"))
    for name, calls, hb, lb in cm["stages"]:
        print(f"  {name:24s} x{calls:<3d} {hb / 1e9:8.3f} GB/call" + (f"  + {lb / 1e6:7.1f} MB NVLink" if lb else ""))
    print(f"\nstage chain ({'staged' if pl.staged else 'direct'} peer layout), one spectral convolution" +
          (" (G1a + G1b run as ONE kernel, spectral_in, when the shape allows: T <= 64, local Y % 4 == 0):"
           if pl.has_t else " (T_out = 1: no t stages; G1a scatters into S1, the last stage reads T1):"))
    for st in pl.chain(staged=pl.staged):
        if "N" not in st:
            print(f"  {st['name']:7s} {'local permutation ' + st['src'] + ' -> ' + st['dst'] if st['name'].startswith('perm') else 'per-mode channel mixing'}")
            continue
        parts = pl.parts(st)
        where = "-> peers over NVLink, then barrier" if st.get("peer_dst") and P > 1 else ""
        print(f"  {st['name']:7s} M = {st['M']:>11,d}  K = {st['K']:>4d}  N = {st['N']:>4d}"
              f"{'  (' + str(len(parts)) + ' column parts)' if len(parts) > 1 else ''}  {st['src']:>4s} -> {st['dst']:<4s} {where}")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
