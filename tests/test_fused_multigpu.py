"""Fused engine over ALL visible H100s (2, 4 or 8 ranks): NVLink peer-scatter epilogues (R2 / R3) in both
layouts (direct, staged), device flag barrier, peer-memory gradient / loss
all-reduce, general partitions folded onto the pencil (BASELINE configs 3 and 4 in miniature) and the 2-D + time
plan -- each against the fp32 portable backend evaluated on the whole field.

One spawn runs every variant (process start + NCCL / IPC set-up dominate the cost on an 8-GPU box); the per-variant
numbers come back as a table and are asserted here.  ``DFNO_TEST_WORLD`` narrows the world (e.g. 2 on an 8-GPU box)."""
import gc
import os

import pytest
import torch

from dfno_b200.utils.testing import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

CFG = dict(in_shape=[1, 2, 16, 32, 16, 2], nt=8, width=8, modes=(4, 4, 4, 3), blocks=2)
CFG5 = dict(in_shape=[2, 1, 32, 32, 3], nt=8, width=12, modes=(4, 4, 3), blocks=2)       # 2-D + time
FWD_TOL, GRAD_TOL = 2e-2, 3e-2


def _world() -> int:
    have = torch.cuda.device_count()
    want = int(os.environ.get("DFNO_TEST_WORLD", "0")) or have
    return max(n for n in (1, 2, 4, 8) if n <= min(have, want))


def _variants(ws):
    folds = {2: [(1, 1, 2, 1, 1, 1), (1, 1, 1, 1, 1, 2)], 4: [(1, 1, 2, 1, 2, 1), (1, 1, 1, 2, 1, 2)],
             8: [(1, 1, 2, 2, 2, 1), (1, 1, 2, 2, 1, 2)]}[ws]
    grid5 = {2: (1, 1, 2, 1, 1), 4: (1, 1, 2, 2, 1), 8: (1, 1, 4, 2, 1)}[ws]
    out = [dict(name=f"pencil staged={st} p2p={p2p}", cfg=CFG, grid=None, staged=st, p2p=p2p)
           for st, p2p in (("0", True), ("0", False), ("1", True))]
    out += [dict(name=f"fold {g}", cfg=CFG, grid=g, staged="0", p2p=True) for g in folds]
    out += [dict(name="2d+time pencil", cfg=CFG5, grid=tuple([1, 1, ws, 1, 1]), staged="0", p2p=True),
            dict(name=f"2d+time fold {grid5}", cfg=CFG5, grid=grid5, staged="1", p2p=True)]
    return out


def _one(rank, ws, v):
    os.environ["DFNO_STAGED_SCATTER"] = v["staged"]
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam, FusedDistributedFNO
    from dfno_b200.parallel.decomposition import shard_bounds, assemble_slices
    cfg = v["cfg"]
    nd = len(cfg["in_shape"])
    dev = torch.device("cuda", torch.cuda.current_device())
    grid = v["grid"] or tuple([1] * (nd - 3) + [ws, 1, 1])
    _, P_x, P_0 = d.create_standard_partitions(tuple(grid))
    P_1 = d.Partition([rank], [1] * nd)
    torch.manual_seed(5)
    ref = d.DistributedFNO(P_1, cfg["in_shape"], cfg["nt"], cfg["width"], cfg["modes"], num_blocks=cfg["blocks"],
                           device=dev, dtype=torch.float32, backend="torch")
    state = d.gather_global_state(ref, to_all=True)
    net = FusedDistributedFNO(P_x, cfg["in_shape"], cfg["nt"], cfg["width"], cfg["modes"],
                              num_blocks=cfg["blocks"], device=dev, use_p2p=v["p2p"])
    want_staged = {"0": False, "1": True}[v["staged"]]
    assert net.plan.staged == want_staged, (net.plan.staged, want_staged)
    d.load_global_state(net, state, strict=False)
    g = torch.Generator().manual_seed(9)
    xg = torch.randn(*cfg["in_shape"], generator=g).to(dev)
    oshape = list(cfg["in_shape"]); oshape[1] = 1; oshape[-1] = cfg["nt"]
    tg = torch.randn(*oshape, generator=g).to(dev)
    lo, hi = shard_bounds(cfg["in_shape"], P_x.shape, P_x.index)
    lo_o, hi_o = shard_bounds(oshape, P_x.shape, P_x.index)
    xl, tl = xg[assemble_slices(lo, hi)].contiguous(), tg[assemble_slices(lo_o, hi_o)].contiguous()

    crit = d.DistributedMSELoss(P_x, engine=net if net.R_in is None else None)   # peer-memory reduction on the pencil
    y_ref = ref(xg)
    ((y_ref - tg) ** 2).mean().backward()
    res = {"name": v["name"]}
    for it in range(2):                      # twice: buffers / barrier epochs are reused across steps
        net.theta.grad = None
        y = net(xl)
        loss = crit(y, tl)
        loss.backward()
    want = y_ref.detach()[assemble_slices(lo_o, hi_o)]
    if net.R_in is None:
        la = d.DistributedRelativeLpLoss(P_x, engine=net)(y.detach(), tl)
        lb = d.DistributedRelativeLpLoss(P_x)(y.detach(), tl)
        if P_0.active:
            assert abs(float(la) - float(lb)) < 1e-5 * abs(float(lb)), (float(la), float(lb))
    res["fwd"] = float((y.detach() - want).norm() / want.norm())
    if P_0.active:
        res["loss"] = abs(float(loss) - float(((y_ref - tg) ** 2).mean())) / float(((y_ref - tg) ** 2).mean())
    for p in ref.parameters():               # gradients in canonical form
        p.data = p.grad if p.grad is not None else torch.zeros_like(p.data)
    G = d.gather_global_state(ref, to_all=True)
    net.theta.data.copy_(net.theta.grad)
    Gf = d.gather_global_state(net, to_all=True)
    worst = 0.0
    for k in G:
        if k.startswith(("linear", "blocks")) and not k.endswith("linear.b"):
            a, b = Gf[k], G[k]
            a = torch.view_as_real(a) if a.is_complex() else a
            b = torch.view_as_real(b) if b.is_complex() else b
            worst = max(worst, float((a.float().reshape(-1) - b.float().reshape(-1)).norm() / b.float().norm().clamp_min(1e-30)))
    res["grad"] = worst
    # one optimizer step keeps the replicated pointwise weights identical on all ranks
    d.load_global_state(net, state, strict=False)
    opt = FusedAdam(net, lr=1e-2)
    net.theta.grad = None
    crit(net(xl), tl).backward()
    opt.step()
    small = net.theta.data[:net.plan.n_small].clone()
    ref_small = small.clone()
    torch.distributed.broadcast(ref_small, src=0)
    res["replica_drift"] = float((small - ref_small).abs().max())
    torch.cuda.synchronize()
    del net, ref, opt
    gc.collect()
    torch.cuda.empty_cache()
    return res


def _all(rank, ws):
    out = []
    for v in _variants(ws):
        try:
            out.append(_one(rank, ws, v))
        except Exception as e:               # noqa: BLE001 - report per variant, keep the collectives of the others matched
            import traceback
            out.append({"name": v["name"], "error": f"{type(e).__name__}: {e}", "trace": traceback.format_exc()[-1500:]})
            raise
    return out


def test_every_rank_layout_matches_the_fp32_backend():
    n = _world()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    per_rank = run_distributed(_all, n, cuda=True, timeout=900)
    table = per_rank[0]
    print(f"\nworld = {n}")
    for i, row in enumerate(table):
        fwd = max(r[i]["fwd"] for r in per_rank)
        grad = max(r[i]["grad"] for r in per_rank)
        drift = max(r[i]["replica_drift"] for r in per_rank)
        print(f"  {row['name']:44s} fwd {fwd:.2e}  grad {grad:.2e}  loss {row.get('loss', 0):.1e}  replica drift {drift:.0e}")
    for i, row in enumerate(table):
        for r in per_rank:
            assert r[i]["fwd"] < FWD_TOL and r[i]["grad"] < GRAD_TOL, r[i]
            assert r[i].get("loss", 0) < 2e-2, r[i]
            assert r[i]["replica_drift"] == 0.0, r[i]
