"""``clip_grad_norm_global`` on the portable backend over gloo ranks, against ``clip_grad_norm_`` on the one-rank model:
batch-partitioned (data-parallel) partitions, where every replica holds the same spectral shard and its summed
gradient, must count each shard once."""
import math

import pytest
import torch

from dfno_b200.utils.testing import run_distributed

IN_SHAPE, NT, WIDTH, MODES = [2, 1, 8, 8, 8, 2], 4, 3, (2, 2, 2, 2)


def _norms(rank, ws, grid):
    import dfno_b200 as d
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    _, P_x, _ = d.create_standard_partitions(grid)
    P_1 = d.Partition([rank], [1] * len(grid))              # a private single-rank world
    torch.manual_seed(7)
    kw = dict(num_blocks=1, dtype=torch.float64, backend="torch")
    serial = d.DistributedFNO(P_1, IN_SHAPE, NT, WIDTH, MODES, **kw)
    net = d.DistributedFNO(P_x, IN_SHAPE, NT, WIDTH, MODES, **kw)
    d.load_global_state(net, d.gather_global_state(serial, to_all=True))
    g = torch.Generator().manual_seed(1)
    xg = torch.randn(*IN_SHAPE, dtype=torch.float64, generator=g)
    out_shape = [IN_SHAPE[0], 1, *IN_SHAPE[2:-1], NT]
    tg = torch.randn(*out_shape, dtype=torch.float64, generator=g)
    (serial(xg) - tg).square().sum().backward()
    want = float(torch.nn.utils.clip_grad_norm_([p for p in serial.parameters() if p.numel()], math.inf))
    xl = xg[assemble_slices(*shard_bounds(IN_SHAPE, P_x.shape, P_x.index))]
    tl = tg[assemble_slices(*shard_bounds(out_shape, P_x.shape, P_x.index))]
    (net(xl) - tl).square().sum().backward()
    got = float(d.clip_grad_norm_global(net, 0.25 * want, P_x.group))
    after = float(d.clip_grad_norm_global(net, math.inf, P_x.group))
    return want, got, after


@pytest.mark.parametrize("ws,grid", [(2, (2, 1, 1, 1, 1, 1)), (4, (2, 1, 1, 2, 1, 1)), (2, (1, 1, 1, 2, 1, 1))],
                         ids=["data_parallel", "data_parallel_x_pencil", "pencil"])
def test_global_norm_matches_the_one_rank_model(ws, grid):
    for want, got, after in run_distributed(_norms, ws, grid, timeout=600):
        assert abs(got - want) <= 1e-6 * want, (got, want)
        assert abs(after - 0.25 * want) <= 1e-5 * want, (after, want)
