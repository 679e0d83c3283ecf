#!/usr/bin/env python
"""Taylor-remainder gradient checks, launchable stand-alone or under torchrun.

Counterparts of the reference's four driver scripts (reference ``tests/gradient_test_torch.py``,
``gradient_test_distdl.py``, ``gradient_test_distdl_bcast.py``, ``gradient_test_dfno.py``):

    python tools/gradient_check.py --case torch
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/gradient_check.py --case transpose
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/gradient_check.py --case transpose-linear
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/gradient_check.py --case bcast
    python -m torch.distributed.run --nproc-per-node 4 --master-addr 127.0.0.1 tools/gradient_check.py --case dfno

``transpose-linear`` is the network the reference reports as *failing* its own check (a Linear
between two re-shards, ``gradient_test_distdl.py:43-50``); with a globally reduced objective it
passes here.  Exit status is non-zero when any parameter fails.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn as nn

import dfno_b200 as d

CASES = ("torch", "transpose", "transpose-linear", "bcast", "dfno")


class _RootOwnedAffine(nn.Module):
    """``W @ x + b`` with ``W``/``b`` living on the root rank only (Broadcast forward, SumReduce
    adjoint) -- the smallest model of the root-owned parameter scheme."""

    def __init__(self, P_x, n_in, n_out, dtype=torch.float64):
        super().__init__()
        self.P_x, self.P_0 = P_x, d.create_root_partition(P_x)
        if self.P_0.active:
            self.W = nn.Parameter(torch.rand(n_out, n_in, dtype=dtype))
            self.b = nn.Parameter(torch.rand(n_out, dtype=dtype))
        else:
            self.W = nn.Parameter(d.zero_volume_tensor(dtype=dtype))
            self.b = nn.Parameter(d.zero_volume_tensor(dtype=dtype))
        self.BW, self.Bb = d.Broadcast(self.P_0, P_x), d.Broadcast(self.P_0, P_x)

    def forward(self, x):
        return self.BW(self.W) @ x + self.Bb(self.b)


class _Grouped(nn.Sequential):
    """Sequential that carries the partition whose group the objective is summed over."""

    def __init__(self, P_x, *mods):
        super().__init__(*mods)
        self.P_x = P_x


def build_case(case: str, world: int):
    """Return ``(module, local_input_shape)`` for ``case`` on ``world`` ranks."""
    f64 = torch.float64
    if case == "torch":
        return nn.Sequential(nn.Linear(16, 16, dtype=f64), nn.Linear(16, 16, dtype=f64)), (16, 16)
    if case in ("transpose", "transpose-linear"):
        _, P_x, _ = d.create_standard_partitions((1, world))
        _, P_y, _ = d.create_standard_partitions((world, 1))
        rows, cols = 2 * world, 16 * world                      # global [rows, cols]
        if case == "transpose":
            f = _Grouped(P_x, nn.Linear(16, 16, dtype=f64), d.DistributedTranspose(P_x, P_y),
                         d.DistributedTranspose(P_y, P_x), nn.Linear(16, 16, dtype=f64))
        else:
            f = _Grouped(P_x, nn.Linear(16, 16, dtype=f64), d.DistributedTranspose(P_x, P_y),
                         nn.Linear(cols, cols, dtype=f64), d.DistributedTranspose(P_y, P_x))
        return f, (rows, 16)
    if case == "bcast":
        _, P_x, _ = d.create_standard_partitions((world,))
        return _RootOwnedAffine(P_x, 16, 16), (16,)
    if case == "dfno":
        grid = {1: (1, 1, 1, 1, 1), 2: (1, 1, 2, 1, 1), 4: (1, 1, 2, 2, 1)}.get(world)
        if grid is None:
            raise SystemExit("--case dfno runs on 1, 2 or 4 ranks")
        _, P_x, _ = d.create_standard_partitions(grid)
        in_shape = [1, 1, 8, 8, 2]
        net = d.DistributedFNO(P_x, in_shape, 4, 3, (2, 2, 2), num_blocks=1, dtype=f64, backend="torch")
        return net, tuple(int(s) for s in d.compute_distribution_info(P_x, in_shape)["shape"])
    raise SystemExit(f"unknown case {case!r}; choose from {CASES}")


def run_case(case: str, verbose: bool = True):
    """Run one case on the current process group; returns the list of failing results (strings)."""
    world = d.world_size()
    torch.manual_seed(100 + d.world_rank())
    f, shape = build_case(case, world)
    # every rank holds its *own* nn.Linear in the transpose cases (same name, different values, acting
    # on the local shard): gradient_test perturbs all of them together and all-reduces <grad, dp>, which
    # is exactly the directional derivative of the global objective along the joint perturbation.
    bad = []
    for r in d.gradient_test(f, shape):
        if verbose and d.world_rank() == 0:
            print(str(r))
        if not r.ok:
            bad.append(str(r))
    return bad


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--case", choices=CASES, default="torch")
    args = ap.parse_args()
    if "RANK" in os.environ:
        d.ensure_process_group("gloo")
    bad = run_case(args.case)
    print(f"rank {d.world_rank()} {'failed' if bad else 'passed'} gradcheck [{args.case}]")
    d.shutdown()
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
