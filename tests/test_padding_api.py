"""``padding=``: zeros appended to the lifted field on non-periodic axes, CPU side -- argument checks, float64
semantics against an explicit lift -> F.pad -> blocks -> crop -> head composition (1, 2 and 4 gloo ranks), gradients,
state dicts across paddings, fused-engine eligibility and the padded engine plan replayed against torch.fft."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dfno_b200.models.fused import EnginePlan, supports
from dfno_b200.utils.testing import run_distributed

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_engine_plan import _run_chain  # noqa: E402


class _Grid:
    def __init__(self, shape):
        self.shape, self.dim = list(shape), len(shape)


def _net(d, P_x, cfg, padding="omit", seed=7):
    torch.manual_seed(seed)
    kw = {} if isinstance(padding, str) and padding == "omit" else dict(padding=padding)
    return d.DistributedFNO(P_x, cfg["in_shape"], cfg["nt"], cfg["width"], cfg["modes"], num_blocks=cfg["blocks"],
                            dtype=torch.float64, backend="torch", out_channels=cfg.get("O", 1), **kw)


def _composition(net, x, padding):
    """The padded network written out: lift, trailing zeros, the same blocks, crop, head."""
    h = F.gelu(net.linear2(F.gelu(net.linear1(x))))
    pads = []
    for p in reversed(padding):
        pads += [0, p]
    h = F.pad(h, pads)
    for blk in net.blocks:
        h = blk(h)
    idx = (slice(None), slice(None)) + tuple(slice(0, n - p) for n, p in zip(h.shape[2:], padding))
    h = h[idx]
    return net.linear4(F.gelu(net.linear3(h)))


CFG_3D = dict(in_shape=[2, 2, 8, 8, 8, 2], nt=6, width=4, modes=(2, 2, 2, 3), blocks=2)
CFG_2D = dict(in_shape=[2, 1, 12, 10, 3], nt=8, width=5, modes=(3, 2, 3), blocks=2, O=2)


def test_padding_argument_validation():
    import dfno_b200 as d
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    for bad in [(1, 2, 3), (0, 0, 0, 0, 2), (0, -1, 0, 2), (0, 0, 0, 2.0), (0, 0, 0, True), "0002", 2]:
        with pytest.raises(ValueError, match="padding"):
            _net(d, P1, CFG_3D, padding=bad)
    # np integers are ints
    assert _net(d, P1, CFG_3D, padding=np.array([0, 0, 8, 2])).padding == (0, 0, 8, 2)


def test_none_and_zeros_are_the_periodic_network():
    import dfno_b200 as d
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    x = torch.rand(*CFG_3D["in_shape"], dtype=torch.float64)
    nets = [_net(d, P1, CFG_3D), _net(d, P1, CFG_3D, padding=None), _net(d, P1, CFG_3D, padding=[0, 0, 0, 0])]
    ys = [n(x) for n in nets]
    for n, y in zip(nets[1:], ys[1:]):
        assert n.padding is None and n.block_in_shape == nets[0].block_in_shape
        assert torch.equal(y, ys[0])
        sd0, sd = nets[0].state_dict(), n.state_dict()
        assert list(sd) == list(sd0) and all(torch.equal(sd[k], sd0[k]) for k in sd0)


@pytest.mark.parametrize("cfg,padding", [(CFG_3D, (0, 0, 8, 2)), (CFG_3D, (4, 2, 0, 0)), (CFG_3D, (4, 4, 8, 4)),
                                         (CFG_2D, (0, 0, 2)), (CFG_2D, (4, 6, 4))])
def test_padded_forward_and_gradients_equal_explicit_composition(cfg, padding):
    import dfno_b200 as d
    _, P1, _ = d.create_standard_partitions([1] * len(cfg["in_shape"]))
    net = _net(d, P1, cfg, padding=padding)
    assert net.block_in_shape[2:] == [n + p for n, p in zip(cfg["in_shape"][2:-1] + [cfg["nt"]], padding)]
    x = torch.rand(*cfg["in_shape"], dtype=torch.float64, requires_grad=True)
    y = net(x)
    assert y.shape[2:-1] == tuple(cfg["in_shape"][2:-1]) and y.shape[-1] == cfg["nt"]
    gy = torch.randn_like(y)
    (y * gy).sum().backward()
    got = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}     # bn1 / bn2 are unused
    gx = x.grad.clone()
    net.zero_grad()
    x.grad = None
    want = _composition(net, x, padding)
    (want * gy).sum().backward()
    assert torch.equal(y, want)
    assert torch.allclose(gx, x.grad, rtol=1e-12, atol=0)
    assert got and all(torch.allclose(got[n], p.grad, rtol=1e-12, atol=0) for n, p in net.named_parameters() if n in got)
    # padding changes the function
    other = _net(d, P1, cfg, padding=None)
    other.load_state_dict(net.state_dict())
    assert not torch.allclose(other(x), y)


def _distributed_equals_serial(rank, ws, grid, cfg, padding, tmp):
    import dfno_b200 as d
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    _, P_x, _ = d.create_standard_partitions(grid)
    P_1 = d.Partition([rank], [1] * len(grid))
    serial = _net(d, P_1, cfg, padding=padding)
    state = d.gather_global_state(serial, to_all=True)
    net = _net(d, P_x, cfg, padding=padding, seed=100 + rank)
    d.load_global_state(net, state)
    xg = torch.rand(*cfg["in_shape"], dtype=torch.float64, generator=torch.Generator().manual_seed(3)).requires_grad_()
    yg = _composition(serial, xg, padding)
    yg.square().sum().backward()
    out = {}
    lo, hi = shard_bounds(cfg["in_shape"], P_x.shape, P_x.index)
    xl = xg.detach()[assemble_slices(lo, hi)].clone().requires_grad_()
    yl = net(xl)
    oshape = list(cfg["in_shape"]); oshape[1] = cfg.get("O", 1); oshape[-1] = cfg["nt"]
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
    # checkpoint round trip records the padding
    d.load_global_state(net, state)
    d.save_checkpoint(net, tmp, epoch=1)
    torch.distributed.barrier()
    net2 = _net(d, P_x, cfg, padding=padding, seed=5)
    info = d.load_checkpoint(net2, tmp, epoch=1)
    out["ckpt_padding"] = info["padding"]
    out["ckpt_equal"] = all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), net2.state_dict().values()))
    return out


@pytest.mark.parametrize("ws,grid,cfg,padding", [
    (1, (1, 1, 1, 1, 1, 1), CFG_3D, (4, 4, 8, 4)),
    (2, (1, 1, 2, 1, 1, 1), CFG_3D, (0, 2, 8, 2)),       # x split: pad y, z, t
    (4, (1, 1, 1, 4, 1, 1), CFG_3D, (4, 0, 8, 4)),       # y split: pad x, z, t
    (4, (1, 1, 2, 2, 1, 1), CFG_3D, (0, 0, 8, 2)),
    (2, (1, 1, 1, 1, 1, 2), CFG_3D, (0, 0, 0, 4)),       # time partition, folded onto a spatial axis: pad t
    (2, (1, 1, 2, 1, 1), CFG_2D, (0, 6, 4)),
])
def test_distributed_padded_network_equals_serial_composition(ws, grid, cfg, padding):
    with tempfile.TemporaryDirectory() as tmp:
        res = run_distributed(_distributed_equals_serial, ws, grid, cfg, padding, tmp)
    for r in res:
        assert r["fwd"] < 1e-11 and r["dx"] < 1e-10 and r["dparam"] < 1e-9, r
        assert r["ckpt_padding"] == list(padding) and r["ckpt_equal"], r


def _split_axis(rank, ws):
    import dfno_b200 as d
    _, P_x, _ = d.create_standard_partitions((1, 1, 2, 1, 1, 1))
    try:
        _net(d, P_x, CFG_3D, padding=(4, 0, 0, 0))
    except ValueError as e:
        return str(e)
    return ""


def test_padding_a_split_axis_raises():
    for msg in run_distributed(_split_axis, 2):
        assert "padding" in msg and "splits" in msg, msg


def test_taylor_gradient_of_a_padded_model():
    import dfno_b200 as d
    cfg = dict(in_shape=[1, 1, 8, 8, 2], nt=4, width=3, modes=(2, 2, 2), blocks=1)
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1))
    net = _net(d, P1, cfg, padding=(4, 0, 2))
    bad = [str(r) for r in d.gradient_test(net, cfg["in_shape"]) if not r.ok]
    assert not bad, "\n".join(bad)


def test_state_dicts_load_across_paddings():
    import dfno_b200 as d
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    x = torch.rand(*CFG_3D["in_shape"], dtype=torch.float64)
    a = _net(d, P1, CFG_3D, padding=(0, 0, 8, 4), seed=1)
    b = _net(d, P1, CFG_3D, padding=(4, 4, 0, 2), seed=2)
    c = _net(d, P1, CFG_3D, seed=3)
    sa = a.state_dict()
    assert list(b.state_dict()) == list(sa) and list(c.state_dict()) == list(sa)
    for n in (b, c):
        assert all(n.state_dict()[k].shape == v.shape for k, v in sa.items())
        n.load_state_dict(sa)
    b.padding, b.blocks = a.padding, a.blocks        # same padding, same modules: same function
    assert torch.equal(b(x), a(x))


def test_supports_accepts_and_refuses_padding():
    g1 = _Grid([1, 1, 1, 1, 1, 1])
    g4 = _Grid([1, 1, 1, 4, 1, 1])
    ok = lambda *a, **k: supports(*a, **k)[0]                                     # noqa: E731
    # Navier-Stokes: 2-D + time, padded in time
    assert ok(_Grid([1, 1, 1, 1, 1]), [10, 1, 64, 64, 10], 40, 20, (8, 8, 8), padding=(0, 0, 8))
    assert ok(g1, [1, 1, 64, 64, 64, 1], 30, 20, (8, 8, 8, 8), padding=(8, 4, 8, 2))
    assert ok(g4, [1, 1, 64, 64, 64, 1], 30, 20, (8, 8, 8, 8), padding=(8, 0, 8, 2))
    assert ok(g1, [1, 1, 64, 64, 64, 1], 20, 64, (8, 8, 8, 8), padding=(0, 0, 0, 4))
    for args, pad, why in [
        ((g1, [1, 1, 64, 64, 64, 1], 20, 20, (12, 12, 40, 8)), (0, 0, 16, 4), "round-2"),   # 2 * KZ > 128
        ((g4, [1, 1, 64, 64, 64, 1], 20, 20, (8, 8, 8, 8)), (0, 4, 0, 0), "splits"),
        ((g1, [1, 1, 64, 64, 64, 1], 20, 20, (8, 8, 8, 8)), (0, 0, 4, 0), "multiple of 8"),
        ((g1, [1, 1, 64, 64, 64, 1], 20, 20, (8, 8, 8, 8)), (0, 0, 0, 3), "even"),
    ]:
        got, reason = supports(*args, padding=pad)
        assert not got and "padding" in reason and why in reason, reason
    # the limits apply to the padded extents: T = 120 + 16 > 128
    got, reason = supports(g1, [1, 1, 32, 32, 32, 1], 120, 20, (4, 4, 4, 4), padding=(0, 0, 0, 16))
    assert not got and "T <= 128" in reason, reason
    # modes refer to the padded grid
    assert ok(g1, [1, 1, 32, 32, 32, 1], 10, 20, (4, 4, 4, 8), padding=(0, 0, 0, 4))
    assert not ok(g1, [1, 1, 32, 32, 32, 1], 10, 20, (4, 4, 4, 8))
    with pytest.raises(ValueError, match="padding"):
        supports(g1, [1, 1, 32, 32, 32, 1], 10, 20, (4, 4, 4, 4), padding=(0, 0, 8))


def test_auto_backend_serves_refused_padding_on_the_portable_backend():
    import dfno_b200 as d
    from dfno_b200.models.fused import wants
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    kw = dict(device=torch.device("cuda"), dtype=torch.bfloat16)
    args = (P1, [1, 1, 64, 64, 64, 1], 20, 20, (8, 8, 8, 8))
    assert wants(args, dict(kw, padding=(0, 0, 8, 2)), "auto")
    assert not wants(args, dict(kw, padding=(0, 0, 4, 2)), "auto")
    with pytest.raises(ValueError, match="padding"):
        wants(args, dict(kw, padding=(0, 0, 4, 2)), "fused")


def test_engine_plan_extents_and_memory_grow_with_the_padded_volume():
    base = EnginePlan(2, 1, 1, 20, 30, 64, 64, 64, (8, 8, 8, 8))
    pad = EnginePlan(2, 1, 1, 20, 30, 64, 64, 64, (8, 8, 8, 8), pad=(8, 4, 8, 2))
    for pl in (base, pad):
        pl.finish(4)
    assert (pad.X, pad.Y, pad.Z, pad.T) == (72, 68, 72, 32) and (pad.Xi, pad.Yi, pad.Zi, pad.Ti) == (64, 64, 64, 30)
    assert pad.S == 72 * 68 * 72 * 32 and pad.Si == base.S == base.Si
    assert pad.segments == base.segments and pad.n_theta == base.n_theta             # the weights do not change
    mb, mp = base.memory_bytes(), pad.memory_bytes()
    assert mp["input_output"] == mb["input_output"]
    ratio = pad.S / base.S
    assert mp["saved_activations"] > mb["saved_activations"] * (ratio - 0.01)
    assert mp["workspaces"] > mb["workspaces"] and mp["total"] > mb["total"]
    cb, cp = base.cost_model(), pad.cost_model()
    assert cb["hbm_bytes"] < cp["hbm_bytes"] < cb["hbm_bytes"] * ratio * 1.01


@pytest.mark.parametrize("P,staged,pad", [(1, False, (4, 4, 8, 2)), (2, False, (4, 0, 8, 2)), (4, True, (0, 0, 8, 4)),
                                          (1, False, (0, 0, 0, 2))])
def test_padded_engine_plan_replays_the_spectral_convolution(P, staged, pad):
    """The chain of a padded plan is the chain of the padded grid: replayed in float64 it equals torch.fft there."""
    import dfno_b200 as d
    B, C, X, Y, Z, T = 2, 3, 8, 8, 8, 4
    modes = (2, 2, 2, 3)
    Xp, Yp, Zp, Tp = X + pad[0], Y + pad[1], Z + pad[2], T + pad[3]
    torch.manual_seed(0)
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    blk = d.DistributedFNOBlock(P1, [B, C, Xp, Yp, Zp, Tp], modes, dtype=torch.float64)
    Wg = torch.zeros(C, C, *blk.fft_shape[2:], dtype=torch.complex128)
    for w, sl in zip(blk.weights, blk.slices):
        Wg[sl] = w.detach()
    x = F.pad(torch.randn(B, C, X, Y, Z, T, dtype=torch.float64), [0, pad[3], 0, pad[2], 0, pad[1], 0, pad[0]])
    want = blk.spectral_forward(x).detach()
    plans = []
    for r in range(P):
        pl = EnginePlan(B, 1, 1, C, T, X, Y, Z, modes, world=P, rank=r, pad=pad)
        pl.finish(1)
        assert (pl.X, pl.Y, pl.Z, pl.T) == (Xp, Yp, Zp, Tp)
        plans.append(pl)
    ops = plans[0].operators()
    h = x.permute(0, 1, 2, 3, 5, 4).contiguous().numpy()
    src, weights = [], []
    for pl in plans:
        src.append(h[:, :, :, pl.y_off:pl.y_off + pl.Yl].reshape(pl.BC, Xp, pl.Yl, Tp, Zp))
        wn = Wg[:, :, :, :, pl.kz_off:pl.kz_off + pl.kzl, :].permute(0, 1, 4, 5, 3, 2).contiguous()
        weights.append(wn.reshape(C, C, pl.Q).numpy())
    outs = _run_chain(plans, ops, src, weights, staged=staged)
    got = np.concatenate([o.reshape(B, C, Xp, pl.Yl, Tp, Zp) for o, pl in zip(outs, plans)], axis=3)
    got = torch.from_numpy(got).permute(0, 1, 2, 3, 5, 4)
    assert torch.allclose(got, want, atol=1e-10), float((got - want).abs().max())
