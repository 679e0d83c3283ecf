"""This framework against the UNMODIFIED reference package (slimgroup/dfno), from the same weights.

``tests/golden/reference_parity.npz`` holds what the reference computed for the cases below, recorded once by
running its own code (on the DistDL / mpi4py stand-in in ``baseline/compat``) with every real or complex
floating-point state-dict entry replaced by the seeded values of :func:`_seeded_state_dict`: per rank, the
reference's state-dict shapes and distribution info, its output, loss (root rank) and parameter gradients.
``oracle/gen_reference_parity.py`` (after ``oracle/install_reference.sh``) records it again.
Checked: identical state-dict keys and per-rank shard shapes, outputs, loss and gradients on 1, 2 and 4 ranks
(``(1,1,2,2,1,1)`` is the reference's in-module demo grid, ``dfno/dfno.py:359`` of the reference)."""
import os

import numpy as np
import pytest
import torch

from dfno_b200.utils.testing import run_distributed

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_parity.npz")


def _seeded_state_dict(sd, rank):
    """Every real or complex floating-point entry of ``sd`` replaced by seeded normal values (scale 0.3, keys in
    sorted order)."""
    out = {}
    for i, k in enumerate(sorted(sd)):
        v = sd[k]
        if v.is_floating_point() or v.is_complex():
            g = torch.Generator().manual_seed(1000 * (rank + 1) + i)
            v = 0.3 * torch.randn(v.shape, dtype=v.dtype, generator=g)
        out[k] = v
    return out


def _parity(rank, ws, grid, in_shape, nt, width, modes, blocks):
    import warnings
    warnings.filterwarnings("ignore")
    import dfno_b200 as d
    gold = np.load(GOLDEN)
    pre = f"ws{ws}/r{rank}/"
    _, P_x, _ = d.create_standard_partitions(grid)
    ours = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, dtype=torch.float64,
                            backend="torch", plan="reference")
    sd = ours.state_dict()
    ref_keys = sorted(k[len(pre + "sdshape/"):] for k in gold.files if k.startswith(pre + "sdshape/"))
    assert sorted(sd) == ref_keys, "state-dict keys differ"
    for k, v in sd.items():
        want = tuple(int(s) for s in gold[pre + "sdshape/" + k])
        assert tuple(v.shape) == want, (k, tuple(v.shape), want)
    ours.load_state_dict(_seeded_state_dict(sd, rank))
    info = d.compute_distribution_info(P_x, in_shape)
    assert tuple(info["shape"]) == tuple(int(s) for s in gold[pre + "shape"])
    assert tuple(info["start"]) == tuple(int(s) for s in gold[pre + "start"])
    g = torch.Generator().manual_seed(99)
    xg = torch.randn(*in_shape, dtype=torch.float64, generator=g)
    x = xg[tuple(info["slice"])].contiguous()
    y1 = ours(x.clone())
    y0 = torch.from_numpy(gold[pre + "y"])
    assert y1.shape == y0.shape, (tuple(y1.shape), tuple(y0.shape))
    t = torch.randn(y0.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(5 + rank))
    l1 = d.DistributedRelativeLpLoss(P_x)(y1, t)
    l1.backward()
    g0 = {k[len(pre + "grad/"):]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith(pre + "grad/")}
    g1 = {k: p.grad for k, p in ours.named_parameters() if p.grad is not None}
    assert sorted(g0) == sorted(g1)
    gerr = max([float((g0[k] - g1[k]).abs().max()) for k in g0 if g0[k].numel()] or [0.0])
    # off the root the reference's loss is mean(empty / empty) = NaN (it only ever prints the root's value);
    # ours is a well-defined 0 there
    lerr = abs(float(gold[pre + "loss"][0]) - float(l1)) if rank == 0 else float(l1)
    return float((y0 - y1.detach()).abs().max()), lerr, gerr


CFG = dict(in_shape=[1, 2, 8, 8, 8, 2], nt=4, width=3, modes=(2, 2, 2, 2), blocks=2)


@pytest.mark.parametrize("ws,grid", [(1, (1, 1, 1, 1, 1, 1)), (4, (1, 1, 2, 2, 1, 1)), (2, (1, 1, 1, 2, 1, 1))])
def test_unmodified_reference_matches_portable_backend(ws, grid):
    res = run_distributed(_parity, ws, grid, CFG["in_shape"], CFG["nt"], CFG["width"], CFG["modes"], CFG["blocks"],
                          timeout=600)
    for yerr, lerr, gerr in res:
        assert yerr < 1e-12 and lerr < 1e-12 and gerr < 1e-12, (yerr, lerr, gerr)
