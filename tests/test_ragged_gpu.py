"""Ragged pencils on one H100: every rank of a pencil whose GPU count does not divide the y extent or the kz mode
count, emulated in-process (the stand-ins of tests/test_pencil_ranks_gpu.py), against the float64 portable backend on
the whole field.

Each row checks the forward, both losses, dL/dx and the weight gradients as the even-pencil test does, and the
invariant that makes ragged storage exact: every saved activation and every gradient buffer is exactly zero at the
dead y rows, every saved spectrum and every spectral-weight gradient exactly zero at the dead kz modes.  A few
FusedAdam steps of the emulated ranks then track torch's Adam on the float64 backend, and the same model on one GPU
(nothing dead) gives the same forward, dx and gradients to within bf16 rounding."""
import pytest
import torch

from test_pencil_ranks_gpu import (DEV, FWD_TOL, GRAD_TOL, _canonical, _Case, _engines, _Peers, _real, _Reference,
                                   _rel, _shards)

pytestmark = pytest.mark.gpu

BLOCKS = 2
ADAM_STEPS, ADAM_LR, ADAM_TOL = 3, 1e-3, 2e-2
ONE_GPU_TOL = 1e-2             # ragged ranks against the same model on one GPU (no dead entries); 4e-3 measured

CASES = {
    # the reference's two-phase grid in y, z and t (60 x 64 x 30, modes 12, 12, 8) on a shorter x axis: 60 rows
    # over 8 GPUs are stored as 8 per rank
    "two_phase": _Case([1, 1, 16, 60, 64, 1], 30, 20, (4, 12, 12, 8)),
    # the headline's layout scaled down: ragged y (40 rows) and ragged kz (8 modes) over 3 and 6 GPUs
    "headline": _Case([1, 2, 16, 40, 32, 2], 8, 20, (4, 6, 4, 3)),
    # 2-D + time: 36 rows of the pencil axis (public X) and 8 kz modes over 5 GPUs
    "2d": _Case([2, 1, 36, 32, 10], 16, 20, (6, 4, 4)),
    # out_timesteps = 1: the chain without t stages, 32 rows and 8 kz modes over 7 GPUs (56 rows and 28 modes stored).
    # Not 30 rows: there the bf16 gradient of the one-element linear1.b misses float64 by 3.4e-2 on one GPU as well
    "steady": _Case([1, 1, 16, 32, 16, 1], 1, 20, (4, 4, 4, 1)),
}

MATRIX = [  # case, P, staged, frozen-weight backward too
    ("two_phase", 8, True, False), ("headline", 3, False, True), ("headline", 6, True, False),
    ("2d", 5, False, False), ("steady", 7, True, False),
]


@pytest.fixture
def pencil(monkeypatch):
    """``pencil(P, staged)`` -> a fresh :class:`_Peers` installed in place of the peer-memory runtime (as in
    tests/test_pencil_ranks_gpu.py)."""
    import threading
    from dfno_b200.ops import build
    from dfno_b200.runtime import symm
    mod = build.load()

    def no_device_barrier(*a, **k):
        raise AssertionError("p2p_barrier launched: with every peer on one GPU it would spin")

    monkeypatch.setattr(mod, "p2p_barrier", no_device_barrier)
    made = []

    def make(P, staged=False):
        peers = _Peers(P)
        monkeypatch.setattr(symm, "SymmetricBuffer", peers.Buffer)
        monkeypatch.setattr(symm, "PeerBarrier", peers.Barrier)
        monkeypatch.setenv("DFNO_STAGED_SCATTER", "1" if staged else "0")
        made.append(peers)
        return peers

    yield make
    torch.cuda.synchronize()
    assert not [t for t in threading.enumerate() if t.name.startswith("pencil-rank")]
    for peers in made:
        assert peers.damaged() == [], peers.damaged()


def _dead_rows(flat, pl, n_lead):
    """The dead y rows of an engine-layout buffer ``[n_lead, X, Yl, T, Z]``."""
    return flat[:n_lead * pl.S].view(n_lead, pl.X, pl.Yl, pl.T, pl.Z)[:, :, pl.Yli:]


def _dead_modes(flat, pl):
    """The dead kz modes of a spectral buffer ``[B or C, C, (kzl, mt, KY, KX), 2]``."""
    return flat.view(-1, pl.C, pl.kzl, pl.mt * pl.KY * pl.KX * 2)[:, :, pl.kzl_live:]


def _zero(t):
    return bool((t == 0).all())


@pytest.mark.parametrize("name,P,staged,frozen", MATRIX,
                         ids=[f"{n}-P{P}-{'staged' if s else 'direct'}" for n, P, s, _ in MATRIX])
def test_ragged_ranks_match_float64_backend(pencil, name, P, staged, frozen):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam
    from dfno_b200.models.loss import _EngineReducedLoss
    c = CASES[name]
    ref = _Reference(c)
    peers = pencil(P, staged)
    grids, nets = _engines(c, P, ref.state)
    pl0 = nets[0].plan
    assert nets[0].world == P and pl0.staged == staged and pl0.fused_pw
    assert pl0.Y != pl0.Yg or pl0.KZ != pl0.KZg, "not a ragged configuration"
    assert any(n.plan.padded for n in nets) == (pl0.Y != pl0.Yg)
    xs = _shards(ref.x, c.in_shape, grids)
    dys, ts = _shards(ref.dy, c.out_shape, grids), _shards(ref.t, c.out_shape, grids)
    BC = pl0.B * pl0.C

    def rank(r):
        net, out = nets[r], {}
        pl = net.plan
        out["y_eval"] = net._forward(xs[r], save=False)
        out["y"] = net._forward(xs[r], save=True)
        torch.cuda.current_stream().synchronize()
        out["dead_fwd"] = ([_zero(_dead_rows(h, pl, BC)) for h in net._saved["h"]]
                           + [_zero(_dead_rows(p, pl, BC)) for p in net._saved["pre"]]
                           + [_zero(_dead_modes(s, pl)) for s in net._saved["S3"]])
        with torch.no_grad():
            out["rel2"] = _EngineReducedLoss.apply(out["y"], ts[r], net, "rel2").clone()
            out["mse"] = _EngineReducedLoss.apply(out["y"], ts[r], net, "mse").clone()
        out["dx"] = net._backward(xs[r], dys[r].float(), input_grad=True, theta_grad=True)
        torch.cuda.current_stream().synchronize()
        # pre now holds dL/dpre of every block, g dL/dh of the lift's output
        out["dead_bwd"] = ([_zero(_dead_rows(p, pl, BC)) for p in net._saved["pre"]]
                           + [_zero(_dead_rows(net.ws["g"], pl, BC))]
                           + [_zero(_dead_modes(net._seg(f"blocks.{k}.spectral", net.grad_flat), pl))
                              for k in range(BLOCKS)])
        out["grad"] = net.grad_flat.clone()
        if frozen:                     # that backward used up the saved pre-activations: save them again
            grad = net.theta.grad
            net._forward(xs[r], save=True)
            out["dx_frozen"] = net._backward(xs[r], dys[r].float(), input_grad=True, theta_grad=False)
            out["grad_kept"] = net.theta.grad is grad and torch.equal(grad, out["grad"])
        return out

    res = peers.run(rank)
    print(f"\n{name} P={P} {'staged' if staged else 'direct'}: y {pl0.Yg} rows stored as {pl0.Y}, kz {pl0.KZg} modes "
          f"stored as {pl0.KZ}; spectral share of the output {ref.share:.2f}")
    for o in res:
        assert all(o["dead_fwd"]) and all(o["dead_bwd"]), (o["dead_fwd"], o["dead_bwd"])

    ys_ref, dx_ref = _shards(ref.y, c.out_shape, grids), _shards(ref.dx, c.in_shape, grids)
    for key in ("y", "y_eval"):
        for o, w in zip(res, ys_ref):
            assert o[key].shape == w.shape, (key, o[key].shape, w.shape)
        errs = [_rel(o[key], w) for o, w in zip(res, ys_ref)]
        whole = _rel(torch.cat([o[key] for o in res], dim=c.nd - 3), ref.y)
        print(f"  forward ({key}) rel err {whole:.2e}, per rank {['%.1e' % e for e in errs]}")
        assert whole < FWD_TOL and max(errs) < FWD_TOL, (key, whole, errs)

    y_all, t_all = torch.cat([o["y"] for o in res], dim=c.nd - 3).double(), ref.t.double()
    B = c.in_shape[0]
    want = {"rel2": float(((y_all - t_all).reshape(B, -1).norm(dim=1) / t_all.reshape(B, -1).norm(dim=1)).mean()),
            "mse": float(((y_all - t_all) ** 2).mean())}
    for kind in ("rel2", "mse"):
        vals = [o[kind] for o in res]
        assert all(torch.equal(v, vals[0]) for v in vals), (kind, [float(v) for v in vals])
        assert abs(float(vals[0]) - want[kind]) <= 1e-5 * abs(want[kind]), (kind, float(vals[0]), want[kind])

    errs = [_rel(o["dx"].view(w.shape), w) for o, w in zip(res, dx_ref)]
    whole = _rel(torch.cat([o["dx"].view(w.shape) for o, w in zip(res, dx_ref)], dim=c.nd - 3), ref.dx)
    print(f"  dx rel err {whole:.2e}, per rank {['%.1e' % e for e in errs]}")
    assert whole < GRAD_TOL and max(errs) < GRAD_TOL, (whole, errs)
    if frozen:
        for o in res:
            assert o["grad_kept"] and torch.equal(o["dx_frozen"], o["dx"])

    G = _canonical(nets, [o["grad"] for o in res])
    worst = 0.0
    for seg in pl0.segments:
        e = _rel(_real(G[seg]).reshape(-1), _real(ref.grads[seg]).reshape(-1))
        worst = max(worst, e)
        assert e < GRAD_TOL, (seg, e)
    print(f"  weight grads: worst segment rel err {worst:.2e}")

    # the same model on one GPU, where nothing is dead: the ragged layout adds no error of its own
    _, (one,) = _engines(c, 1, ref.state)
    y1 = one._forward(ref.x, save=True)
    dx1 = one._backward(ref.x, ref.dy.float(), input_grad=True, theta_grad=True).view(ref.dx.shape)
    G1 = _canonical([one], [one.grad_flat])
    e1 = {"y": _rel(torch.cat([o["y"] for o in res], dim=c.nd - 3), y1),
          "dx": _rel(torch.cat([o["dx"].view(w.shape) for o, w in zip(res, dx_ref)], dim=c.nd - 3), dx1),
          "grads": max(_rel(_real(G[k]).reshape(-1), _real(G1[k]).reshape(-1)) for k in pl0.segments)}
    print("  against one GPU: " + ", ".join(f"{k} {v:.1e}" for k, v in e1.items()))
    assert max(e1.values()) < ONE_GPU_TOL, e1
    del one

    # FusedAdam on the emulated ranks against torch's Adam on the float64 backend, from the same weights, on the
    # linear loss <y, dy> (its output gradient is dy: no reduction across ranks); dead-mode weights stay exactly zero
    for n in nets:
        n.engine_state_from_global(ref.state, strict=False)
    _, P1, _ = d.create_standard_partitions([1] * c.nd)
    fref = d.DistributedFNO(P1, c.in_shape, c.nt, c.width, c.modes, num_blocks=BLOCKS, device=DEV,
                            dtype=torch.float64, backend="torch")
    d.load_global_state(fref, ref.state, strict=False)
    ropt = torch.optim.Adam(fref.parameters(), lr=ADAM_LR)
    xr = ref.x.double()
    for _ in range(ADAM_STEPS):
        ropt.zero_grad()
        (fref(xr) * ref.dy).sum().backward()
        ropt.step()
    want_state = d.gather_global_state(fref, to_all=True)
    opts = [FusedAdam(n, lr=ADAM_LR) for n in nets]

    def train(r):
        net = nets[r]
        for _ in range(ADAM_STEPS):
            net._forward(xs[r], save=True)
            net._backward(xs[r], dys[r].float(), theta_grad=True)
            opts[r].step()
        torch.cuda.current_stream().synchronize()
        return [_zero(_dead_modes(net._seg(f"blocks.{k}.spectral"), net.plan)) for k in range(BLOCKS)]

    dead = peers.run(train)
    assert all(all(v) for v in dead), dead
    got = _canonical(nets, [n.theta.data for n in nets])
    worst_w, worst_u = 0.0, 0.0
    for seg in pl0.segments:
        a, w, s = (_real(t[seg]).reshape(-1).double().to(DEV) for t in (got, want_state, ref.state))
        ew, eu = _rel(a, w), _rel(a - s, w - s)      # the weights, and the update they took
        worst_u = max(worst_u, eu)
        # a missing update would give 1, a reversed one 2; early Adam steps are nearly sign(g), so entries whose
        # gradient is within bf16 rounding of 0 may step either way.  Zero-initialised biases are their update.
        assert eu < 0.5, (seg, eu)
        if bool(s.any()):
            worst_w = max(worst_w, ew)
            assert ew < ADAM_TOL, (seg, ew)
    print(f"  {ADAM_STEPS} Adam steps: worst segment rel err {worst_w:.2e} (of the update {worst_u:.2e})")


@pytest.mark.parametrize("name,P", [("headline", 3), ("headline", 6), ("two_phase", 8)])
def test_seeded_initialisation_is_partition_independent_on_ragged_pencils(pencil, name, P):
    """``_init_parameters(seed)`` on ragged storage: the live weights are those of one rank, the dead kz modes zero."""
    c = CASES[name]
    pencil(P, P >= 8)
    _, (one,) = _engines(c, 1, init_seed=7)
    _, nets = _engines(c, P, init_seed=7)
    mine, want = _canonical(nets, [n.theta.data for n in nets]), _canonical([one], [one.theta.data])
    assert sorted(mine) == sorted(want)
    for k in want:
        assert torch.equal(mine[k], want[k]), k
    for n in nets:
        for k in range(BLOCKS):
            assert _zero(_dead_modes(n._seg(f"blocks.{k}.spectral"), n.plan))
