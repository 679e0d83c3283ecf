"""FusedAdam's schedules, decoupled decay and global gradient-norm clipping on one H100.

* the sum-of-squares kernel against float64 ``torch``, and bitwise repeatable;
* ``FusedAdam`` against ``torch.optim.Adam`` after ``clip_grad_norm_`` on an fp32 copy of the parameters, fed the
  same gradients, under torch's schedulers;
* an engine trained by the CUDA-graph ``Trainer`` and by the eager one ends with the same ``theta`` under a schedule
  (replay reads the hyperparameters set before it), with no host synchronisation in the replayed step;
* the global norm over emulated pencil ranks (``test_pencil_ranks_gpu``'s stand-ins) equals the norm of the merged
  canonical gradient, and the same on two or more real GPUs;
* the default optimizer path keeps its single launch."""
import math
import os
import sys
import types
import warnings

import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_pencil_ranks_gpu import CASES, _canonical, _engines, _real, _shards, pencil  # noqa: E402,F401

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
STEPS = 32


def _C():
    from dfno_b200.ops import build
    return build.load()


def _sumsq(x):
    from dfno_b200.models.fused import SUMSQ_MAX_BLOCKS
    out = torch.full((1,), math.nan, device=DEV, dtype=torch.float64)
    partials = torch.zeros(SUMSQ_MAX_BLOCKS, device=DEV, dtype=torch.float64)
    ticket = torch.zeros(1, device=DEV, dtype=torch.int32)
    _C().sumsq(x, out, partials, ticket)
    assert int(ticket) == 0, "the kernel must leave its ticket at zero for the next call"
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 255, 1024, 4097, 1 << 20, (1 << 22) + 3, 50_000_001])
@pytest.mark.parametrize("offset", [0, 1, 3])
def test_sumsq_matches_float64(n, offset):
    g = torch.Generator(device=DEV).manual_seed(n + offset)
    base = torch.randn(n + offset, device=DEV, generator=g)
    x = base[offset:]                              # offsets 1 and 3: a body that starts off 16-byte alignment
    got = float(_sumsq(x))
    want = float((x.double() ** 2).sum())
    assert abs(got - want) <= 1e-12 * want, (got, want)
    again = [_sumsq(x) for _ in range(3)]
    assert all(torch.equal(a, again[0]) for a in again), "sum of squares differs between calls"


def test_sumsq_zeros_and_extremes():
    assert float(_sumsq(torch.zeros(12345, device=DEV))) == 0.0
    big = torch.full((1001,), 3.0e38, device=DEV)                   # squares far beyond the fp32 range
    big[::7] = -1.0e19
    tiny = torch.full((1001,), 1.0e-30, device=DEV)                 # squares below the fp32 range
    for x in (big, tiny, torch.cat([big, tiny])):
        got, want = float(_sumsq(x)), float((x.double() ** 2).sum())
        assert math.isfinite(got) and abs(got - want) <= 1e-12 * want, (got, want)
    x = torch.randn(1000, device=DEV)
    x[17] = math.inf
    assert float(_sumsq(x)) == math.inf
    x[18] = math.nan
    assert math.isnan(float(_sumsq(x)))


# ------------------------------------------------------------------ FusedAdam against torch.optim.Adam
def _stub(theta):
    """The optimizer needs only ``theta`` and the extension from the model."""
    return types.SimpleNamespace(theta=nn.Parameter(theta), _C=_C())


def _schedule(kind, opt):
    S = torch.optim.lr_scheduler
    if kind == "const":
        return None
    if kind == "step":
        return S.StepLR(opt, step_size=7, gamma=0.5)
    if kind == "cosine":
        return S.CosineAnnealingLR(opt, T_max=STEPS, eta_min=1e-4)
    if kind == "warmup_cosine":
        w = 5
        return S.LambdaLR(opt, lambda k: (k + 1) / w if k < w else 0.5 * (1 + math.cos(math.pi * (k - w) / (STEPS - w))))
    if kind == "onecycle":
        return S.OneCycleLR(opt, max_lr=1e-2, total_steps=STEPS, cycle_momentum=True)
    if kind == "onecycle_nomom":
        return S.OneCycleLR(opt, max_lr=1e-2, total_steps=STEPS, cycle_momentum=False)
    raise ValueError(kind)


@pytest.mark.parametrize("decoupled", [False, True], ids=["l2", "decoupled"])
@pytest.mark.parametrize("clip", [None, "active", "inactive"])
@pytest.mark.parametrize("sched", ["const", "step", "cosine", "warmup_cosine", "onecycle", "onecycle_nomom"])
def test_fused_adam_matches_torch_adam(sched, clip, decoupled):
    from dfno_b200.models.fused import FusedAdam
    n = 100_003                                     # a scalar tail
    gen = torch.Generator(device=DEV).manual_seed(11)
    theta0 = torch.randn(n, device=DEV, generator=gen)
    typical = math.sqrt(n) * 0.05                   # gradient norm of the sequence below
    max_norm = {None: None, "active": 0.3 * typical, "inactive": 20.0 * typical}[clip]
    kw = dict(lr=3e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=1e-2)
    model = _stub(theta0.clone())
    opt = FusedAdam(model, decoupled_weight_decay=decoupled, max_grad_norm=max_norm, **kw)
    ref_p = nn.Parameter(theta0.clone())
    ref = torch.optim.Adam([ref_p], decoupled_weight_decay=decoupled, **kw)
    s_f, s_r = _schedule(sched, opt), _schedule(sched, ref)
    assert opt.device_hparams() == (sched != "const" or clip is not None or decoupled)
    for k in range(STEPS):
        g = torch.randn(n, device=DEV, generator=gen) * 0.05 * (1 + 0.5 * math.sin(k))
        model.theta.grad = g.clone()
        ref_p.grad = g.clone()
        if max_norm is not None:
            want_norm = torch.nn.utils.clip_grad_norm_([ref_p], max_norm)
        opt.step()
        ref.step()
        if max_norm is not None:
            assert torch.allclose(opt.grad_norm, want_norm, rtol=1e-5, atol=0), (k, float(opt.grad_norm),
                                                                              float(want_norm))
        for s in (s_f, s_r):
            if s is not None:
                s.step()
        assert opt.lr == ref.param_groups[0]["lr"] and tuple(opt.betas) == tuple(ref.param_groups[0]["betas"])
    err = float((model.theta.data - ref_p.data).abs().max())
    moved = float((ref_p.data - theta0).abs().max())
    print(f"\n{sched} clip={clip} decoupled={decoupled}: max |theta - torch| {err:.2e} (update {moved:.2e})")
    torch.testing.assert_close(model.theta.data, ref_p.data, rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(opt.m, ref.state[ref_p]["exp_avg"], rtol=1e-4, atol=1e-7)
    torch.testing.assert_close(opt.v, ref.state[ref_p]["exp_avg_sq"], rtol=1e-4, atol=1e-9)


@pytest.mark.parametrize("bad", [math.inf, math.nan])
def test_nonfinite_gradient_norm_as_torch(bad):
    """An infinite norm scales the gradient by 0 (its infinite entries become NaN), a NaN norm spreads NaN: what
    clip_grad_norm_(error_if_nonfinite=False) does before torch's Adam.  No step is skipped."""
    from dfno_b200.models.fused import FusedAdam
    n = 4099
    gen = torch.Generator(device=DEV).manual_seed(5)
    theta0 = torch.randn(n, device=DEV, generator=gen)
    model = _stub(theta0.clone())
    opt = FusedAdam(model, lr=1e-2, max_grad_norm=1.0)
    ref_p = nn.Parameter(theta0.clone())
    ref = torch.optim.Adam([ref_p], lr=1e-2)
    for k in range(3):
        g = torch.randn(n, device=DEV, generator=gen)
        if k == 1:
            g[100] = bad
        model.theta.grad, ref_p.grad = g.clone(), g.clone()
        want = torch.nn.utils.clip_grad_norm_([ref_p], 1.0)
        opt.step()
        ref.step()
        torch.testing.assert_close(opt.grad_norm, want, equal_nan=True)
        torch.testing.assert_close(model.theta.data, ref_p.data, rtol=1e-5, atol=2e-6, equal_nan=True)
    assert opt.step_count == 3


# ------------------------------------------------------------------ the engine under the Trainer
SHAPE, NT = [1, 1, 16, 16, 16, 1], 8


def _net(seed=0):
    import dfno_b200 as d
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    net = d.DistributedFNO(P_x, SHAPE, NT, 8, (4, 4, 4, 3), num_blocks=2, device=DEV, dtype=torch.bfloat16,
                           init_seed=seed)
    assert isinstance(net, d.FusedDistributedFNO)
    return net, d.DistributedRelativeLpLoss(P_x, engine=net)


def _batches(k, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(*SHAPE, generator=g).pin_memory(),
             torch.randn(1, 1, 16, 16, 16, NT, generator=g).pin_memory()) for _ in range(k)]


def test_graph_trainer_follows_the_schedule_like_the_eager_one():
    """Fails where replay ignores lr changes.  StepLR halves lr every two steps; a third, eager run keeps lr constant,
    which is what a baked-in lr would do, and lands far from the scheduled one.  The graph and eager runs differ only
    by the engine's float atomics, amplified through its bf16 arithmetic and Adam's normalisation."""
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam
    batches = _batches(10)
    out = {}
    for name, graph, schedule in (("eager", False, True), ("graph", True, True), ("constant_lr", False, False)):
        net, crit = _net()
        theta0 = net.theta.detach().clone()
        opt = FusedAdam(net, lr=1e-2, weight_decay=1e-2, decoupled_weight_decay=True, max_grad_norm=0.01)
        sched = torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.5) if schedule else None
        tr = d.Trainer(net, crit, opt, device=DEV, cuda_graph=graph)
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            for x, y in batches:
                tr.step(x, y)
                if sched is not None:
                    sched.step()
        msgs = [str(w.message) for w in caught]
        assert not [m for m in msgs if "lr_scheduler.step()" in m or "capture" in m], msgs
        assert (tr._graph is not None) == graph and opt.step_count == len(batches)
        out[name] = (net.theta.detach().clone(), theta0, float(opt.grad_norm))
    te, t0, ne = out["eager"]
    tg, _, ng = out["graph"]
    tc = out["constant_lr"][0]
    rel = float((tg - te).norm() / (te - t0).norm())
    rel_const = float((tc - te).norm() / (te - t0).norm())
    print(f"\ngraph vs eager: theta rel diff {rel:.2e} of the update (constant lr: {rel_const:.2e}); "
          f"last grad norm {ne:.4f} / {ng:.4f} (clipped to 0.01)")
    assert rel < 1e-2, rel
    assert rel_const > 0.3, rel_const
    assert abs(ne - ng) <= 1e-2 * ne


def test_replayed_step_has_no_host_sync():
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam
    net, crit = _net()
    opt = FusedAdam(net, lr=1e-2, max_grad_norm=1.0)
    sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-2, total_steps=20)
    tr = d.Trainer(net, crit, opt, device=DEV, cuda_graph=True)
    (x, y), = _batches(1)
    tr.step(x, y)                                  # capture
    sched.step()
    assert tr._graph is not None
    xd, yd = x.to(DEV), y.to(DEV)
    torch.cuda.synchronize()
    lrs = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(4):
            tr.step_on_device(xd, yd)
            lrs.append(opt.lr)
            sched.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(set(lrs)) == 4 and math.isfinite(float(opt.grad_norm))
    assert float(opt.hparams[0]) == lrs[-1]        # the last replay read the last lr written


def _fwd_bwd_launches(net, crit, x, y):
    c0 = net._C.count
    loss = crit(net(x), y)
    loss.backward()
    torch.cuda.synchronize()
    return net._C.count - c0


@pytest.mark.parametrize("variant", ["default", "clipped"])
def test_launches_per_replayed_step(monkeypatch, variant):
    """The default optimizer path adds exactly one launch (adam_step) to the replayed step and never reaches the
    device-hyperparameter kernels; clipping adds the sum of squares, and one launch before each replay."""
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam
    net, crit = _net()
    (x, y), = _batches(1)
    fb = _fwd_bwd_launches(net, crit, x.to(DEV), y.to(DEV))
    net.theta.grad = None
    if variant == "default":
        opt = FusedAdam(net, lr=1e-2)
        mod = net._C._mod

        def refuse(*a, **k):
            raise AssertionError("the default path launched a device-hyperparameter kernel")
        for name in ("adam_step_dev", "adam_set_hparams", "sumsq"):
            monkeypatch.setattr(mod, name, refuse)
    else:
        opt = FusedAdam(net, lr=1e-2, max_grad_norm=1.0)
    tr = d.Trainer(net, crit, opt, device=DEV, cuda_graph=True)
    tr.step(x, y)
    assert tr._graph is not None
    want = fb + (1 if variant == "default" else 2)
    assert tr.graph_kernel_launches == want, (tr.graph_kernel_launches, fb)
    c0 = net._C.count
    tr.step(x, y)
    assert net._C.count - c0 == want + (0 if variant == "default" else 1)


def test_graph_recaptured_when_a_baked_in_hyperparameter_changes():
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam
    net, crit = _net()
    opt = FusedAdam(net, lr=1e-2)
    tr = d.Trainer(net, crit, opt, device=DEV, cuda_graph=True)
    (x, y), = _batches(1)
    tr.step(x, y)
    g0 = tr._graph
    tr.step(x, y)
    assert tr._graph is g0
    opt.lr = 5e-3                                  # default path: the graph holds lr as a kernel argument
    tr.step(x, y)
    g1 = tr._graph
    assert g1 is not g0 and tr._graph_key == opt.graph_key() == ("device", False)
    for lr in (4e-3, 3e-3):                        # now read from the device: no further capture
        opt.lr = lr
        tr.step(x, y)
        assert tr._graph is g1 and float(opt.hparams[0]) == lr
    assert opt.step_count == 5


# ------------------------------------------------------------------ the global norm across pencil ranks
@pytest.mark.parametrize("P,staged", [(2, False), (4, True)])
def test_emulated_ranks_global_norm(pencil, P, staged):
    from dfno_b200.models.fused import FusedAdam
    c = CASES["base"]
    peers = pencil(P, staged)
    grids, nets = _engines(c, P, init_seed=3)
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(*c.in_shape, device=DEV, generator=g)
    dy = torch.randn(*c.out_shape, device=DEV, generator=g)
    xs, dys = _shards(x, c.in_shape, grids), _shards(dy, c.out_shape, grids)
    opts = [FusedAdam(n, lr=1e-3, max_grad_norm=0.5 if P == 2 else math.inf) for n in nets]
    n_small = nets[0].plan.n_small

    def rank(r):
        net = nets[r]
        net._forward(xs[r], save=True)
        net._backward(xs[r], dys[r], input_grad=False, theta_grad=True)
        grad = net.grad_flat.clone()
        opts[r].step()
        return grad, opts[r].grad_norm.clone(), net.theta.data[:n_small].clone()

    res = peers.run(rank)
    G = _canonical(nets, [o[0] for o in res])
    want = math.sqrt(sum(float((_real(v).double() ** 2).sum()) for v in G.values()))
    got = [o[1] for o in res]
    print(f"\nP={P}: global grad norm {float(got[0]):.6e}, canonical float64 {want:.6e}")
    assert all(torch.equal(t, got[0]) for t in got), [float(t) for t in got]
    assert abs(float(got[0]) - want) <= 2e-6 * want, (float(got[0]), want)
    for o in res[1:]:                              # the same clip coefficient everywhere
        assert torch.equal(o[2], res[0][2])


def _mg_norm(rank, ws):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam, FusedDistributedFNO
    c = CASES["base"]
    dev = torch.device("cuda", torch.cuda.current_device())
    _, P_x, _ = d.create_standard_partitions(tuple([1] * (c.nd - 3) + [ws, 1, 1]))
    net = FusedDistributedFNO(P_x, c.in_shape, c.nt, c.width, c.modes, num_blocks=2, device=dev, init_seed=3)
    g = torch.Generator(device=dev).manual_seed(100 + rank)
    local = list(c.in_shape)
    local[c.nd - 3] //= ws
    y = net(torch.randn(*local, device=dev, generator=g))
    y.backward(torch.randn(y.shape, device=dev, generator=g))
    opt = FusedAdam(net, lr=1e-3, max_grad_norm=0.5)
    opt.step()
    torch.cuda.synchronize()
    return {"norm": float(opt.grad_norm), "grad": net.grad_flat.cpu(), "meta": net.engine_meta()}


@pytest.mark.multigpu
def test_multigpu_global_norm():
    from dfno_b200.models.fused import FusedDistributedFNO as F
    from dfno_b200.utils.testing import run_distributed
    ws = max(n for n in (2, 4, 8) if n <= torch.cuda.device_count())
    res = run_distributed(_mg_norm, ws, ws, cuda=True, timeout=600)
    parts = [F.theta_to_canonical(r["grad"], r["meta"], include_pointwise=i == 0) for i, r in enumerate(res)]
    G = F.merge_canonical(parts, res[0]["meta"])
    want = math.sqrt(sum(float((_real(v).double() ** 2).sum()) for v in G.values()))
    assert len({r["norm"] for r in res}) == 1, [r["norm"] for r in res]
    assert abs(res[0]["norm"] - want) <= 2e-6 * want, (res[0]["norm"], want)


# ------------------------------------------------------------------ out-of-bounds stores
@pytest.mark.parametrize("n", [1, 3, 4, 7, 1021, 100_003])
def test_new_kernels_write_only_their_outputs(n):
    """Every buffer the optimizer kernels get is a view between two guard bands of NaN; after sumsq, the
    hyperparameter write and both clipped and unclipped device-path Adam steps the guards are untouched, and sumsq
    writes no partial beyond its grid."""
    from dfno_b200.models.fused import SUMSQ_MAX_BLOCKS
    C_ = _C()
    G = 64

    def guarded(k, dtype=torch.float32, fill=0.0):
        buf = torch.full((k + 2 * G,), math.nan, device=DEV, dtype=dtype)
        buf[G:G + k] = fill
        return buf, buf[G:G + k]

    gen = torch.Generator(device=DEV).manual_seed(n)
    bufs = {k: guarded(n) for k in "pgmv"}
    bufs["g"][1].copy_(torch.randn(n, device=DEV, generator=gen))
    bufs["p"][1].copy_(torch.randn(n, device=DEV, generator=gen))
    hp_b, hp = guarded(8, torch.float64)
    sq_b, sq = guarded(1, torch.float64)
    part_b, part = guarded(SUMSQ_MAX_BLOCKS, torch.float64)
    tk_b = torch.full((3,), -7, device=DEV, dtype=torch.int32)
    tk_b[1] = 0
    nrm_b, nrm = guarded(1)
    step = torch.ones(1, device=DEV)
    C_.sumsq(bufs["g"][1], sq, part, tk_b[1:2])
    C_.adam_set_hparams(hp, 1e-3, 0.9, 0.999, 1e-8, 1e-2, True, 0.5)
    C_.adam_step_dev(bufs["p"][1], bufs["g"][1], bufs["m"][1], bufs["v"][1], hp, step, 1.0, sq, nrm.view(()))
    C_.adam_step_dev(bufs["p"][1], bufs["g"][1], bufs["m"][1], bufs["v"][1], hp, step, 1.0)
    torch.cuda.synchronize()
    for name, (b, _) in [*bufs.items(), ("hparams", (hp_b, None)), ("sumsq", (sq_b, None)), ("norm", (nrm_b, None)),
                         ("partials", (part_b, None))]:
        assert torch.isnan(b[:G]).all() and torch.isnan(b[-G:]).all(), f"{name}: a store outside the buffer"
    blocks = int((~torch.isnan(part)).sum())
    assert 1 <= blocks and torch.isnan(part[blocks:]).all(), "partials written beyond the grid"
    assert tk_b.tolist() == [-7, 0, -7]
    assert torch.isfinite(bufs["p"][1]).all() and math.isfinite(float(nrm))
