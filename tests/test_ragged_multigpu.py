"""Ragged pencils on real ranks: the reference's two-phase workload (60 x 60 x 64 x 30, modes 12 12 12 8) on a pencil
of every visible GPU (8 rows of 60 stored per rank at 8 GPUs) and of 3 GPUs, against the same seeded model replayed on
one GPU by rank 0 -- the check ``bench.py`` makes of an N-rank run.  Forward, canonical weight gradients and the weights
after two FusedAdam steps are compared; a count of GPUs that divides the grid is skipped (not ragged)."""
import gc

import pytest
import torch

from dfno_b200.utils.testing import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

CFG = dict(in_shape=[1, 1, 60, 60, 64, 1], nt=30, width=20, modes=(12, 12, 12, 8), blocks=2)
FWD_TOL, GRAD_TOL = 2e-2, 3e-2
STEPS = 2


def _rel(a, b):
    a, b = a.detach().double().reshape(-1), b.detach().double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _real(t):
    return torch.view_as_real(t) if t.is_complex() else t


def _run(dev, P_x, x, t, cfg):
    """Seeded fused model on ``P_x``: (output, canonical gradients of the rel-2 loss, canonical weights after STEPS
    FusedAdam steps), the canonical states on every rank."""
    import dfno_b200 as d
    net = d.DistributedFNO(P_x, cfg["in_shape"], cfg["nt"], cfg["width"], cfg["modes"], num_blocks=cfg["blocks"],
                           device=dev, backend="fused", init_seed=3)
    crit = d.DistributedRelativeLpLoss(P_x, engine=net)
    y = net(x)
    crit(y, t).backward()
    flat = net.theta.data.clone()
    net.theta.data.copy_(net.theta.grad)
    grads = net.engine_state_to_global(to_all=True)
    net.theta.data.copy_(flat)
    opt = d.FusedAdam(net, lr=1e-3)
    for _ in range(STEPS):
        opt.zero_grad()
        crit(net(x), t).backward()
        opt.step()
    state = net.engine_state_to_global(to_all=True)
    plan = (net.plan.Y, net.plan.Yg)
    del net, opt
    gc.collect()
    torch.cuda.empty_cache()
    return y.detach(), grads, state, plan


def _one(rank, ws, cfg):
    import dfno_b200 as d
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    dev = torch.device("cuda", torch.cuda.current_device())
    grid = (1, 1, 1, ws, 1, 1)
    _, P_x, _ = d.create_standard_partitions(grid)
    P_1 = d.Partition([rank], [1] * 6)           # the one-GPU replica (run by rank 0)
    g = torch.Generator().manual_seed(9)
    xg = torch.randn(*cfg["in_shape"], generator=g).to(dev)
    oshape = [*cfg["in_shape"][:-1], cfg["nt"]]
    tg = torch.randn(*oshape, generator=g).to(dev)
    xl = xg[assemble_slices(*shard_bounds(cfg["in_shape"], grid, P_x.index))].contiguous()
    tl = tg[assemble_slices(*shard_bounds(oshape, grid, P_x.index))].contiguous()
    y, grads, state, plan = _run(dev, P_x, xl, tl, cfg)
    ys = [None] * ws
    torch.distributed.all_gather_object(ys, y.cpu())
    if rank != 0:
        return {}
    y1, grads1, state1, _ = _run(dev, P_1, xg, tg, cfg)
    res = {"plan": plan, "fwd": _rel(torch.cat(ys, dim=3), y1.cpu())}
    res["grad"] = max(_rel(_real(grads[k]), _real(grads1[k])) for k in grads1 if k in grads)
    res["steps"] = max(_rel(_real(state[k]), _real(state1[k])) for k in state1 if k in state)
    return res


@pytest.mark.parametrize("which", ["all", "three"])
def test_two_phase_on_a_ragged_pencil_matches_one_gpu(which):
    have = torch.cuda.device_count()
    ws = have if which == "all" else 3
    if ws < 3 or ws > have:
        pytest.skip(f"needs >= 3 GPUs ({have} here)")
    if ws > 8:
        ws = 8
    if CFG["in_shape"][3] % ws == 0:
        pytest.skip(f"{ws} GPUs divide the grid: not a ragged pencil")
    r0 = run_distributed(_one, ws, CFG, cuda=True, timeout=900)[0]
    print(f"\n{ws} GPUs: y stored {r0['plan'][0]} for {r0['plan'][1]} live; fwd {r0['fwd']:.2e}  grad {r0['grad']:.2e}  "
          f"after {STEPS} Adam steps {r0['steps']:.2e}")
    assert r0["plan"][0] != r0["plan"][1]
    assert r0["fwd"] < FWD_TOL and r0["grad"] < GRAD_TOL and r0["steps"] < FWD_TOL, r0
