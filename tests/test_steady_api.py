"""``out_timesteps=1`` (steady problems, next-step prediction), CPU side: validation on both backends, float64
semantics against an explicit lift -> blocks of ``gelu(W h + Re(ifftn(R * trunc(fftn h))))`` -> head composition (1, 2
and 4 gloo ranks), a Taylor test, fused-engine eligibility, the T = 1 engine plan (no t stages, no Z1 / U) and its
chain replayed in float64 against torch.fft, forward and adjoint, on the direct and the staged peer layouts."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dfno_b200.models.fused import MAX_IN, EnginePlan, supports, wants
from dfno_b200.parallel.planner import validate_modes
from dfno_b200.utils.testing import run_distributed

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_engine_plan import _run_chain  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Grid:
    def __init__(self, shape):
        self.shape, self.dim = list(shape), len(shape)


def _net(d, P_x, cfg, seed=7):
    torch.manual_seed(seed)
    return d.DistributedFNO(P_x, cfg["in_shape"], 1, cfg["width"], cfg["modes"], num_blocks=cfg["blocks"],
                            dtype=torch.float64, backend="torch", out_channels=cfg.get("O", 1),
                            padding=cfg.get("padding"))


def _global_weight(blk):
    W = torch.zeros(blk.width, blk.width, *blk.fft_shape[2:], dtype=torch.complex128)
    for w, sl in zip(blk.weights, blk.slices):
        W[sl] = w.detach() if not torch.is_grad_enabled() else w
    return W


def _spectral(blk, h):
    """``Re(ifftn(R * trunc(fftn h)))`` over every transformed axis; the length-1 time axis keeps its one bin."""
    dims = list(range(2, h.dim()))
    H = torch.fft.fftn(h.to(torch.complex128), dim=dims)
    idx = []
    for a, m in enumerate(blk.modes):
        n = h.shape[2 + a]
        idx.append(torch.arange(m) if a == len(blk.modes) - 1 else torch.cat([torch.arange(m), torch.arange(n - m, n)]))
    sel = (slice(None), slice(None)) + tuple(torch.meshgrid(*idx, indexing="ij"))
    Y = torch.einsum("bi...,io...->bo...", H[sel], _global_weight(blk))
    full = torch.zeros_like(H)
    full[sel] = Y
    return torch.fft.ifftn(full, dim=dims).real


def _composition(net, x):
    """The T = 1 network written out: lift, (trailing spatial zeros,) blocks of gelu(W h + spectral(h)), crop, head."""
    h = F.gelu(net.linear2(F.gelu(net.linear1(x))))
    pad = net.padding or (0,) * (h.dim() - 2)
    h = F.pad(h, [v for p in reversed(pad) for v in (0, p)])
    for blk in net.blocks:
        h = F.gelu(torch.einsum("oi,bi...->bo...", blk.linear.W, h) + _spectral(blk, h))
    h = h[(slice(None), slice(None)) + tuple(slice(0, n - p) for n, p in zip(h.shape[2:], pad))]
    return net.linear4(F.gelu(net.linear3(h)))


CFG_3D = dict(in_shape=[2, 2, 8, 8, 8, 1], width=4, modes=(2, 2, 2, 1), blocks=2)
CFG_2D = dict(in_shape=[2, 1, 12, 10, 10], width=5, modes=(3, 2, 1), blocks=2, O=2)     # next step from 10 frames
CFG_3D_PAD = dict(CFG_3D, padding=(4, 2, 8, 0))
CFG_2D_PAD = dict(CFG_2D, in_shape=[2, 10, 12, 10, 1], padding=(4, 6, 0))                # frames as channels


def test_validation_accepts_a_single_time_step():
    import dfno_b200 as d
    validate_modes([2, 4, 8, 8, 1], (2, 2, 1))
    with pytest.raises(ValueError, match="rfft bins"):
        validate_modes([2, 4, 8, 8, 1], (2, 2, 2))
    with pytest.raises(ValueError, match="1 or even"):
        validate_modes([2, 4, 8, 8, 3], (2, 2, 1))
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    net = _net(d, P1, CFG_3D)
    assert net(torch.rand(*CFG_3D["in_shape"], dtype=torch.float64)).shape == (2, 1, 8, 8, 8, 1)
    with pytest.raises(ValueError, match="rfft bins"):
        _net(d, P1, dict(CFG_3D, modes=(2, 2, 2, 2)))
    # odd T > 1 stays refused on both backends
    with pytest.raises(ValueError, match="1 or even"):
        d.DistributedFNO(P1, [2, 2, 8, 8, 8, 1], 3, 4, (2, 2, 2, 1), dtype=torch.float64, backend="torch")
    ok, why = supports(_Grid([1] * 6), [1, 1, 16, 16, 16, 1], 3, 20, (4, 4, 4, 1))
    assert not ok and "T%2" in why and "1 or even" in why, why


@pytest.mark.parametrize("cfg", [CFG_3D, CFG_2D, CFG_3D_PAD, CFG_2D_PAD])
def test_forward_and_gradients_equal_explicit_composition(cfg):
    import dfno_b200 as d
    _, P1, _ = d.create_standard_partitions([1] * len(cfg["in_shape"]))
    net = _net(d, P1, cfg)
    x = torch.rand(*cfg["in_shape"], dtype=torch.float64, requires_grad=True)
    y = net(x)
    assert y.shape == (cfg["in_shape"][0], cfg.get("O", 1), *cfg["in_shape"][2:-1], 1)
    gy = torch.randn_like(y)
    (y * gy).sum().backward()
    got = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
    gx = x.grad.clone()
    net.zero_grad()
    x.grad = None
    want = _composition(net, x)
    (want * gy).sum().backward()
    assert torch.allclose(y, want, rtol=1e-12, atol=1e-14), float((y - want).abs().max())
    assert torch.allclose(gx, x.grad, rtol=1e-10, atol=1e-14)
    assert got and all(torch.allclose(got[n], p.grad, rtol=1e-10, atol=1e-14)
                       for n, p in net.named_parameters() if n in got)


def test_taylor_gradient_of_a_steady_model():
    import dfno_b200 as d
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1))
    net = _net(d, P1, dict(in_shape=[1, 2, 8, 8, 1], width=3, modes=(2, 2, 1), blocks=1))
    bad = [str(r) for r in d.gradient_test(net, [1, 2, 8, 8, 1]) if not r.ok]
    assert not bad, "\n".join(bad)


def _distributed_equals_serial(rank, ws, grid, cfg, tmp):
    import dfno_b200 as d
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    _, P_x, _ = d.create_standard_partitions(grid)
    serial = _net(d, d.Partition([rank], [1] * len(grid)), cfg)
    state = d.gather_global_state(serial, to_all=True)
    net = _net(d, P_x, cfg, seed=100 + rank)
    d.load_global_state(net, state)
    xg = torch.rand(*cfg["in_shape"], dtype=torch.float64, generator=torch.Generator().manual_seed(3)).requires_grad_()
    yg = serial(xg)
    yg.square().sum().backward()
    out = {"explicit": float((yg - _composition(serial, xg)).abs().max() / yg.abs().max())}
    lo, hi = shard_bounds(cfg["in_shape"], P_x.shape, P_x.index)
    xl = xg.detach()[assemble_slices(lo, hi)].clone().requires_grad_()
    yl = net(xl)
    oshape = list(cfg["in_shape"]); oshape[1] = cfg.get("O", 1); oshape[-1] = 1
    lo_o, hi_o = shard_bounds(oshape, P_x.shape, P_x.index)
    want = yg.detach()[assemble_slices(lo_o, hi_o)]
    out["fwd"] = float((yl.detach() - want).abs().max() / want.abs().max())
    yl.square().sum().backward()
    out["dx"] = float((xl.grad - xg.grad[assemble_slices(lo, hi)]).abs().max() / xg.grad.abs().max())
    for model in (net, serial):
        for p in model.parameters():
            p.data = p.grad.clone() if p.grad is not None else torch.zeros_like(p.data)
    gd = d.gather_global_state(net, to_all=True)
    gs = d.gather_global_state(serial, to_all=True)
    out["dparam"] = max(float((gd[k] - gs[k]).abs().max() / gs[k].abs().max().clamp_min(1e-30))
                        for k in gs if gs[k].is_floating_point() or gs[k].is_complex())
    return out


@pytest.mark.parametrize("ws,grid,cfg", [
    (2, (1, 1, 1, 2, 1, 1), CFG_3D),                    # the engine's y-pencil
    (4, (1, 1, 2, 2, 1, 1), CFG_3D),                    # a P_x the fused engine folds onto its pencil
    (2, (1, 1, 2, 1, 1), CFG_2D),
])
def test_distributed_steady_network_equals_serial(ws, grid, cfg):
    with tempfile.TemporaryDirectory() as tmp:
        res = run_distributed(_distributed_equals_serial, ws, grid, cfg, tmp)
    for r in res:
        assert r["explicit"] < 1e-12 and r["fwd"] < 1e-11 and r["dx"] < 1e-10 and r["dparam"] < 1e-9, r


def test_supports_accepts_every_composition_at_t1():
    g1, g4, g8, f1 = _Grid([1] * 6), _Grid([1, 1, 1, 4, 1, 1]), _Grid([1, 1, 1, 8, 1, 1]), _Grid([1] * 5)
    cases = [
        (f1, [16, 3, 128, 128, 1], 32, (12, 12, 1), dict(padding=(8, 8, 0))),        # 2-D Darcy-like, padded
        (f1, [20, 1, 64, 64, 10], 20, (8, 8, 1), {}),                                 # next step from 10 frames
        (f1, [20, 10, 64, 64, 1], 20, (8, 8, 1), {}),                                 # ... the frames as channels
        (g1, [4, 2, 128, 128, 128, 1], 20, (12, 12, 12, 1), {}),                      # 3-D steady
        (g1, [1, 1, 64, 64, 64, 1], 20, (8, 8, 8, 1), dict(out_channels=3)),
        (g1, [1, 1, 64, 64, 64, 1], 48, (8, 8, 8, 1), {}),
        (g1, [1, 1, 64, 64, 64, 1], 64, (8, 8, 8, 1), {}),
        (g1, [1, MAX_IN, 64, 64, 64, 1], 20, (8, 8, 8, 1), {}),
        (g1, [1, 1, 64, 64, 64, 64], 20, (8, 8, 8, 1), {}),                           # T_in = 64
        (g1, [1, 1, 64, 64, 64, 1], 20, (8, 8, 8, 1), dict(padding=(8, 4, 8, 0))),
        (g1, [1, 1, 64, 64, 96, 1], 20, (8, 8, 34, 1), {}),                           # round-1 route
        (g4, [1, 1, 64, 64, 96, 1], 20, (8, 8, 34, 1), {}),
        (g4, [2, 1, 64, 64, 64, 1], 20, (8, 8, 8, 1), dict(padding=(8, 0, 8, 0))),
        (g8, [4, 2, 128, 128, 128, 1], 20, (12, 12, 12, 1), {}),                      # staged peer layout
        (_Grid([1, 1, 2, 2, 2, 1]), [1, 1, 64, 64, 64, 1], 20, (8, 8, 8, 1), {}),    # folded onto the pencil
        (_Grid([1, 1, 2, 1, 1]), [4, 1, 64, 64, 1], 20, (8, 8, 1), {}),
    ]
    kw = dict(device=torch.device("cuda"), dtype=torch.bfloat16)
    for grid, in_shape, width, modes, extra in cases:
        got, why = supports(grid, in_shape, 1, width, modes, **extra)
        assert got, (in_shape, width, modes, extra, why)
        assert wants((grid, in_shape, 1, width, modes), dict(kw, **extra), "auto")
    # round-1 route: 2 * KZ = 136 > 128
    assert not EnginePlan(1, 1, 1, 20, 1, 64, 64, 96, (8, 8, 34, 1)).fused_pw


def test_supports_refusals_at_t1():
    g1 = _Grid([1] * 6)
    for T in (3, 15):                                   # odd T > 1: still refused, with the same reason
        got, why = supports(g1, [1, 1, 64, 64, 64, 1], T, 20, (8, 8, 8, 1))
        assert not got and "T%2" in why, why
    got, why = supports(g1, [1, 1, 64, 64, 64, 1], 1, 20, (8, 8, 8, 2))
    assert not got and "mode counts" in why, why
    # t padding of a single step cannot give an even (or unit) padded axis: the refusal names out_timesteps
    got, why = supports(g1, [1, 1, 64, 64, 64, 1], 1, 20, (8, 8, 8, 1), padding=(0, 0, 0, 2))
    assert not got and "out_timesteps" in why and "padding" in why, why
    got, why = supports(g1, [1, 1, 64, 64, 64, 1], 1, 20, (8, 8, 8, 1), padding=(0, 0, 0, 1))
    assert not got and "even" in why, why
    kw = dict(device=torch.device("cuda"), dtype=torch.bfloat16)
    assert not wants((g1, [1, 1, 64, 64, 64, 1], 3, 20, (8, 8, 8, 1)), kw, "auto")
    with pytest.raises(ValueError, match="T%2"):
        wants((g1, [1, 1, 64, 64, 64, 1], 3, 20, (8, 8, 8, 1)), kw, "fused")


def _plan(P=1, r=0, B=2, C=20, X=64, Y=64, Z=64, modes=(8, 8, 8, 1), **kw):
    pl = EnginePlan(B, 1, 1, C, 1, X, Y, Z, modes, world=P, rank=r, **kw)
    pl.finish(4)
    return pl


@pytest.mark.parametrize("staged", [False, True])
def test_engine_plan_at_t1_has_no_t_stages(staged):
    P = 8 if staged else 4
    pl = _plan(P, 3)
    assert not pl.has_t and pl.mtp == 1 and pl.mt == 1
    names = [st["name"] for st in pl.chain(staged=staged)]
    want = ["G1a"] + (["permS1"] if staged else []) + ["G2", "G3", "mix", "iG3", "iG2"] + \
        (["permT1"] if staged else []) + ["iG1a"]
    assert names == want, names
    st = {s["name"]: s for s in pl.chain(staged=staged)}
    assert st["G1a"]["dst"] == ("S1s" if staged else "S1") and st["G1a"]["peer_dst"] and st["G1a"]["barrier_after"]
    assert st["G1a"]["scatter"].peer == ("col", pl.kzl) and st["iG1a"]["src"] == "T1"
    ops = pl.operators()
    assert not any(k.startswith(("G1b", "iG1b")) for k in ops)
    assert sorted(ops) == sorted(["G1a", "G2", "G3", "iG3", "iG2", "iG1a"] +
                                 [k + "_adj" for k in ("G1a", "G2", "G3", "iG3", "iG2", "iG1a")])
    # T1 has U's layout and size; Z1 and U are not allocated
    assert pl.n_T1 == pl.BC * pl.X * pl.Yl * pl.KZ * 2 and pl.n_Z1 == pl.n_U == 0
    m = pl.memory_bytes()
    assert m["workspaces"] == (pl.n_S1 + pl.n_T1 + pl.n_S2 + 2 * pl.n_S3 + pl.n_T2) * 2
    # T = 2 keeps its t stages and the Z1 / U buffer
    p2 = EnginePlan(2, 1, 1, 20, 2, 64, 64, 64, (8, 8, 8, 2), world=P, rank=3)
    assert p2.has_t and p2.mtp == 4 and p2.n_Z1 > 0 and p2.n_U > 0
    assert [s["name"] for s in p2.chain(staged=staged)][1:2] == ["G1b"]


def test_cost_model_counts_what_runs_at_t1():
    for P in (1, 4):
        pl = _plan(P, 0)
        bf = 2
        act, S1, S2, S3, T2, T1 = (pl.n_act * bf, pl.n_S1 * bf, pl.n_S2 * bf, pl.n_S3 * bf, pl.n_T2 * bf,
                                   pl.n_T1 * bf)
        off = (P - 1) / P
        for front in (False, True):                      # spectral_in never runs at T = 1
            cm = pl.cost_model(front=front)
            st = {n: (c, b, l) for n, c, b, l in cm["stages"]}
            assert "G1b" not in st and "iG1b" not in st and "spectral_in" not in st
            assert st["G1a"] == (8, act + S1, S1 * off)
            assert st["iG2"] == (8, T2 + T1, T1 * off)
            assert st["G2"][1] == S1 + S2 and st["G3"][1] == S2 + S3
            assert st["spectral_out fwd"][1] == T1 + 3 * act and st["spectral_out adj"][1] == T1 + 2 * act
            assert cm["nvlink_bytes"] == pytest.approx(8 * (S1 + T1) * off)
    legacy = _plan(1, 0, Z=96, modes=(8, 8, 34, 1))
    st = {n: b for n, _, b, _ in legacy.cost_model()["stages"]}
    assert not legacy.fused_pw and st["iG1a"] == (legacy.n_T1 + legacy.n_act) * 2


@pytest.mark.parametrize("P,staged", [(1, False), (2, False), (4, False), (2, True), (4, True), (8, True)])
@pytest.mark.parametrize("five_d", [False, True])
def test_t1_chain_replays_the_spectral_convolution(P, staged, five_d):
    """The T = 1 chain replayed in float64 with the engine's operators and scatter tables equals torch.fft, and its
    adjoint chain satisfies <chain x, g> = <x, chain^T g>."""
    import dfno_b200 as d
    B, C = 2, 3
    X, Y, Z, modes = (1, 16, 8, (0, 2, 4, 1)) if five_d else (6, 16, 8, (2, 2, 4, 1))
    torch.manual_seed(0)
    if five_d:      # [B, C, X', Y', 1] runs as the 6-D plan with X = 1
        _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1))
        blk = d.DistributedFNOBlock(P1, [B, C, Y, Z, 1], modes[1:], dtype=torch.float64)
    else:
        _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
        blk = d.DistributedFNOBlock(P1, [B, C, X, Y, Z, 1], modes, dtype=torch.float64)
    Wg = torch.zeros(C, C, *blk.fft_shape[2:], dtype=torch.complex128)
    for w, sl in zip(blk.weights, blk.slices):
        Wg[sl] = w.detach()
    x = torch.randn(B, C, *blk.in_shape[2:], dtype=torch.float64)
    want = blk.spectral_forward(x).detach()
    with torch.no_grad():
        assert torch.allclose(want, _spectral(blk, x), atol=1e-12)
    if five_d:
        Wg, x, want = Wg.unsqueeze(2), x.unsqueeze(2), want.unsqueeze(2)
    plans = []
    for r in range(P):
        pl = EnginePlan(B, 1, 1, C, 1, X, Y, Z, modes, world=P, rank=r)
        pl.finish(1)
        plans.append(pl)
    assert not plans[0].has_t
    ops = plans[0].operators()
    h = x.permute(0, 1, 2, 3, 5, 4).contiguous().numpy()                  # engine layout [B, C, X, Y, T, Z]
    src, weights = [], []
    for pl in plans:
        src.append(h[:, :, :, pl.y_off:pl.y_off + pl.Yl].reshape(pl.BC, X, pl.Yl, 1, Z))
        wn = Wg[:, :, :, :, pl.kz_off:pl.kz_off + pl.kzl, :].permute(0, 1, 4, 5, 3, 2).contiguous()
        weights.append(wn.reshape(C, C, pl.Q).numpy())
    outs = _run_chain(plans, ops, src, weights, staged=staged)
    got = np.concatenate([o.reshape(B, C, X, pl.Yl, 1, Z) for o, pl in zip(outs, plans)], axis=3)
    got = torch.from_numpy(got).permute(0, 1, 2, 3, 5, 4)
    assert torch.allclose(got, want, atol=1e-10), float((got - want).abs().max())

    g = torch.randn(B, C, X, Y, Z, 1, dtype=torch.float64)
    gh = g.permute(0, 1, 2, 3, 5, 4).contiguous().numpy()
    gsrc = [gh[:, :, :, pl.y_off:pl.y_off + pl.Yl].reshape(pl.BC, X, pl.Yl, 1, Z) for pl in plans]
    wadj = [np.conj(np.transpose(w, (1, 0, 2))) for w in weights]
    gouts = _run_chain(plans, ops, gsrc, wadj, adj=True, staged=staged)
    gx = np.concatenate([o.reshape(B, C, X, pl.Yl, 1, Z) for o, pl in zip(gouts, plans)], axis=3)
    lhs = float((got * g).sum())
    rhs = float((torch.from_numpy(gx).permute(0, 1, 2, 3, 5, 4) * x).sum())
    assert abs(lhs - rhs) < 1e-9 * max(1.0, abs(lhs)), (lhs, rhs)


def test_plan_tool_prints_the_t1_chain():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "plan.py"), "--shape", "128", "128", "128", "1",
                        "--modes", "12", "12", "12", "1", "--batch", "4", "--in-channels", "2", "--gpus", "8"],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    out = r.stdout
    assert "fused engine: yes" in out and "T_out = 1" in out, out
    chain = out.split("stage chain")[1]
    assert "G1a" in chain and "S1s" in chain and "iG2" in chain and "iG1a" in chain
    assert "G1b" not in chain and "iG1b" not in chain and "spectral_in" not in out.split("stage chain")[0]
    assert "per-rank memory, training" in out
