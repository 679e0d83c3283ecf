"""``out_channels``: one network predicting several fields (CPU only).  The portable backend is the semantic reference;
the fused engine's plan, eligibility and dispatch are checked without a GPU."""
import os
import subprocess
import sys

import pytest
import torch

import dfno_b200 as d
from dfno_b200.models import fused
from dfno_b200.utils.testing import run_distributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(grid):
    return d.create_standard_partitions(grid)[1]


@pytest.mark.parametrize("O", [2, 3])
@pytest.mark.parametrize("grid,shape,modes", [
    ((1, 1, 1, 1, 1, 1), [2, 1, 8, 8, 8, 1], (2, 2, 2, 2)),      # 3-D + time
    ((1, 1, 1, 1, 1), [2, 3, 8, 8, 4], (2, 2, 2)),               # 2-D + time, C_in > 1, T_in > 1
])
def test_portable_forward_shape(O, grid, shape, modes):
    torch.manual_seed(0)
    net = d.DistributedFNO(_p(grid), shape, 6, 4, modes, num_blocks=1, backend="torch", out_channels=O)
    y = net(torch.randn(*shape))
    assert list(y.shape) == [shape[0], O, *shape[2:-1], 6]


def test_state_dict_keys_and_linear4_shapes():
    P_x = _p((1, 1, 1, 1, 1, 1))
    args = (P_x, [1, 1, 8, 8, 8, 1], 4, 4, (2, 2, 2, 2))
    one = d.DistributedFNO(*args, num_blocks=1, backend="torch")
    three = d.DistributedFNO(*args, num_blocks=1, backend="torch", out_channels=3)
    s1, s3 = one.state_dict(), three.state_dict()
    assert list(s1) == list(s3)
    assert tuple(s3["linear4.W"].shape) == (3, 128) and tuple(s3["linear4.b"].shape) == (1, 3, 1, 1, 1, 1)
    assert all(s1[k].shape == s3[k].shape for k in s1 if not k.startswith("linear4"))


def test_out_channels_one_is_the_default_bitwise():
    P_x = _p((1, 1, 1, 1, 1))
    shape = [2, 1, 8, 8, 3]
    nets = []
    for kw in ({}, {"out_channels": 1}):
        torch.manual_seed(5)
        nets.append(d.DistributedFNO(P_x, shape, 4, 4, (2, 2, 2), num_blocks=2, backend="torch", **kw))
    for (k, a), (k2, b) in zip(nets[0].state_dict().items(), nets[1].state_dict().items()):
        assert k == k2 and torch.equal(a, b), k
    x = torch.randn(*shape)
    assert torch.equal(nets[0](x), nets[1](x))


@pytest.mark.parametrize("bad", [0, -1, 1.5, "2", True])
def test_out_channels_validation(bad):
    P_x = _p((1, 1, 1, 1, 1, 1))
    with pytest.raises(ValueError, match="out_channels"):
        d.DistributedFNO(P_x, [1, 1, 8, 8, 8, 1], 4, 4, (2, 2, 2, 2), num_blocks=1, backend="torch", out_channels=bad)
    with pytest.raises(ValueError, match="out_channels"):
        fused.supports(P_x, [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), out_channels=bad)


def test_taylor_gradient_three_outputs():
    P_x = _p((1, 1, 1, 1, 1))
    torch.manual_seed(3)
    net = d.DistributedFNO(P_x, [1, 1, 8, 8, 2], 4, 3, (2, 2, 2), num_blocks=1, dtype=torch.float64,
                           backend="torch", out_channels=3)
    res = d.gradient_test(net, (1, 1, 8, 8, 2), names=["linear3.W", "linear3.b", "linear4.W", "linear4.b",
                                                        "blocks.0.linear.W", "linear1.W"])
    bad = [str(r) for r in res if not r.ok]
    assert res and not bad, "\n".join(bad)


def _fold(rank, ws, O):
    """4 ranks with a time-partitioned P_x (folded onto the spatial axes) against a private 1-rank network"""
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    grid = (1, 1, 1, 2, 1, 2)
    shape = [1, 1, 8, 8, 8, 4]
    _, P_x, _ = d.create_standard_partitions(grid)
    P_1 = d.Partition([rank], [1] * len(grid))
    kw = dict(num_blocks=1, dtype=torch.float64, backend="torch", out_channels=O)
    torch.manual_seed(7)
    serial = d.DistributedFNO(P_1, shape, 4, 4, (2, 2, 2, 2), **kw)
    state = d.gather_global_state(serial, to_all=True)
    net = d.DistributedFNO(P_x, shape, 4, 4, (2, 2, 2, 2), **kw)
    d.load_global_state(net, state)
    xg = torch.rand(*shape, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    yg = serial(xg)
    lo, hi = shard_bounds(shape, P_x.shape, P_x.index)
    yl = net(xg[assemble_slices(lo, hi)])
    oshape = [1, O, 8, 8, 8, 4]
    lo_o, hi_o = shard_bounds(oshape, P_x.shape, P_x.index)
    want = yg.detach()[assemble_slices(lo_o, hi_o)]
    assert yl.shape == want.shape, (yl.shape, want.shape)
    return float((yl.detach() - want).abs().max() / want.abs().max())


def test_folded_time_partition_two_outputs_matches_one_rank():
    res = run_distributed(_fold, 4, 2)
    assert all(r < 1e-11 for r in res), res


def _plan(O, B=2, mz=4):
    pl = fused.EnginePlan(B, 1, 1, 20, 8, 16, 16, 16, (4, 4, mz, 3), out_channels=O)
    pl.finish(4)
    return pl


def test_engine_plan_layout_and_figures():
    one, three = _plan(1), _plan(3)
    H = 128
    off_w, shape_w = three.segments["linear4.W"]
    off_b, shape_b = three.segments["linear4.b"]
    assert shape_w == (3, H) and shape_b == (3,) and off_b == off_w + 3 * H
    # segments before linear4 are unchanged; the replicated segment grows by the new head entries
    for k, v in one.segments.items():
        if not k.startswith(("linear4", "blocks.")) or k.endswith(".linear.W"):
            assert three.segments[k] == v, k
    assert three.n_small == (off_b + 3 + 63) // 64 * 64
    m1, m3 = one.memory_bytes(train=True), three.memory_bytes(train=True)
    out_bytes = one.B * one.S * 4
    assert m3["input_output"] - m1["input_output"] == 2 * out_bytes
    assert m3["parameters"] - m1["parameters"] == (three.n_theta - one.n_theta) * 4
    c1, c3 = dict((n, b) for n, _, b, _ in one.cost_model()["stages"]), \
        dict((n, b) for n, _, b, _ in three.cost_model()["stages"])
    assert c3["head fwd"] - c1["head fwd"] == 2 * one.npos * 4
    assert c3["head bwd"] - c1["head bwd"] == 2 * 2 * one.npos * 4
    assert all(c3[k] == c1[k] for k in c1 if not k.startswith(("head", "adam")))


def test_engine_plan_default_is_one_output():
    a = fused.EnginePlan(2, 1, 1, 20, 8, 16, 16, 16, (4, 4, 4, 3))
    a.finish(4)
    b = _plan(1)
    assert a.segments == b.segments and (a.n_small, a.n_theta) == (b.n_small, b.n_theta)
    assert a.memory_bytes() == b.memory_bytes() and a.memory_bytes(train=False) == b.memory_bytes(train=False)
    assert a.cost_model() == b.cost_model()
    assert a.segments["linear4.W"][1] == (1, 128) and a.segments["linear4.b"][1] == (1,)


def test_supports_out_channels():
    P_x = _p((1, 1, 1, 1, 1, 1))
    args = (P_x, [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3))
    for O in (1, 2, 3, 4):
        ok, why = fused.supports(*args, out_channels=O)
        assert ok, (O, why)
    ok, why = fused.supports(*args, out_channels=5)
    assert not ok and "out_channels" in why and "4" in why
    # 2 * KZ > 128 selects the round-1 route, whose head is single-output
    wide = (P_x, [1, 1, 16, 16, 80, 1], 8, 8, (4, 4, 34, 4))
    ok1, why1 = fused.supports(*wide)
    assert ok1, why1
    ok, why = fused.supports(*wide, out_channels=2)
    assert not ok and "round-2" in why
    # width 32: the multi-output backward does not fit the register budget
    w32 = (P_x, [1, 1, 16, 16, 16, 1], 8, 32, (4, 4, 4, 3))
    assert fused.supports(*w32)[0] and not fused.supports(*w32, out_channels=2)[0]
    assert "width" in fused.supports(*w32, out_channels=2)[1]


def test_dispatch_passes_out_channels_to_the_fused_engine(monkeypatch):
    P_x = _p((1, 1, 1, 1, 1, 1))
    args = (P_x, [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3))
    kw = dict(device=torch.device("cuda"), dtype=torch.bfloat16)
    assert fused.wants(args, dict(kw, out_channels=3), "auto") is True
    assert fused.wants(args, dict(kw, out_channels=5), "auto") is False
    with pytest.raises(ValueError, match="out_channels"):
        fused.wants(args, dict(kw, out_channels=5), "fused")
    seen = {}

    class Engine(fused.FusedDistributedFNO):
        def __init__(self, *a, **k):          # records what the dispatch hands over (no GPU needed)
            torch.nn.Module.__init__(self)
            seen.update(k)

    monkeypatch.setattr(fused, "FusedDistributedFNO", Engine)
    net = d.DistributedFNO(*args, out_channels=3, **kw)
    assert isinstance(net, Engine) and seen.get("out_channels") == 3


def test_out_channels_is_a_keyword_of_every_entry_point():
    import inspect
    for fn in (d.DistributedFNO.__init__, fused.FusedDistributedFNO.__init__, fused.supports, fused.fold_onto_pencil,
               fused.EnginePlan.__init__):
        assert inspect.signature(fn).parameters["out_channels"].default == 1, fn


def test_plan_tool_out_channels():
    cmd = [sys.executable, os.path.join(ROOT, "tools", "plan.py"), "--shape", "16", "16", "16", "8", "--modes", "4",
           "4", "4", "3", "--width", "8"]
    r1 = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    r3 = subprocess.run(cmd + ["--out-channels", "3"], capture_output=True, text=True, cwd=ROOT)
    assert r1.returncode == 0 and r3.returncode == 0, r1.stderr + r3.stderr
    assert "out_channels = 3" in r3.stdout and "fused engine: yes" in r3.stdout
    r5 = subprocess.run(cmd + ["--out-channels", "5"], capture_output=True, text=True, cwd=ROOT)
    assert "fused engine: no" in r5.stdout and "out_channels" in r5.stdout
