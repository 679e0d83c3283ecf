"""Input gradients (dL/dx) of the fused engine over all visible H100s (2, 4 or 8 ranks), on a y-pencil and on a
general partition folded onto the pencil (dx flows back through the input re-shard's adjoint), against the fp32
portable backend evaluated on the whole field.  ``DFNO_TEST_WORLD`` narrows the world."""
import gc
import os

import pytest
import torch

from dfno_b200.utils.testing import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

CFG = dict(in_shape=[1, 2, 16, 32, 16, 2], nt=8, width=8, modes=(4, 4, 4, 3), blocks=2)
DX_TOL = 3e-2


def _world() -> int:
    have = torch.cuda.device_count()
    want = int(os.environ.get("DFNO_TEST_WORLD", "0")) or have
    return max(n for n in (1, 2, 4, 8) if n <= min(have, want))


def _grids(ws):
    fold = {2: (1, 1, 2, 1, 1, 1), 4: (1, 1, 2, 1, 2, 1), 8: (1, 1, 2, 2, 2, 1)}[ws]
    return [("pencil", (1, 1, 1, ws, 1, 1)), (f"fold {fold}", fold)]


def _one(rank, ws, name, grid, frozen):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    cfg = CFG
    dev = torch.device("cuda", torch.cuda.current_device())
    _, P_x, _ = d.create_standard_partitions(tuple(grid))
    P_1 = d.Partition([rank], [1] * len(grid))
    torch.manual_seed(5)
    ref = d.DistributedFNO(P_1, cfg["in_shape"], cfg["nt"], cfg["width"], cfg["modes"], num_blocks=cfg["blocks"],
                           device=dev, dtype=torch.float32, backend="torch")
    net = FusedDistributedFNO(P_x, cfg["in_shape"], cfg["nt"], cfg["width"], cfg["modes"], num_blocks=cfg["blocks"],
                              device=dev, input_grad=True)
    d.load_global_state(net, d.gather_global_state(ref, to_all=True), strict=False)
    net.theta.requires_grad_(not frozen)
    g = torch.Generator().manual_seed(9)
    xg = torch.randn(*cfg["in_shape"], generator=g).to(dev)
    oshape = list(cfg["in_shape"]); oshape[1] = 1; oshape[-1] = cfg["nt"]
    wg = torch.randn(*oshape, generator=g).to(dev)
    lo, hi = shard_bounds(cfg["in_shape"], P_x.shape, P_x.index)
    lo_o, hi_o = shard_bounds(oshape, P_x.shape, P_x.index)
    xl = xg[assemble_slices(lo, hi)].contiguous().requires_grad_()
    wl = wg[assemble_slices(lo_o, hi_o)].contiguous()
    xr = xg.clone().requires_grad_()
    (ref(xr) * wg).sum().backward()
    (net(xl) * wl).sum().backward()           # every rank's share of the loss; the adjoint chain sums them
    want = xr.grad[assemble_slices(lo, hi)]
    err = float((xl.grad - want).norm() / want.norm())
    res = {"name": f"{name} frozen={frozen}", "dx": err, "theta_grad_none": net.theta.grad is None}
    torch.cuda.synchronize()
    del net, ref
    gc.collect()
    torch.cuda.empty_cache()
    return res


def _all(rank, ws):
    return [_one(rank, ws, name, grid, frozen) for name, grid in _grids(ws) for frozen in (False, True)]


def test_input_gradient_on_every_rank_layout_matches_the_fp32_backend():
    n = _world()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    per_rank = run_distributed(_all, n, cuda=True, timeout=900)
    print(f"\nworld = {n}")
    for i, row in enumerate(per_rank[0]):
        print(f"  {row['name']:40s} dx {max(r[i]['dx'] for r in per_rank):.2e}")
    for rows in per_rank:
        for row in rows:
            assert row["dx"] < DX_TOL, row
            assert row["theta_grad_none"] == row["name"].endswith("frozen=True"), row
