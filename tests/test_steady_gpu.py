"""``out_timesteps=1`` on the fused engine (one H100): G1a's scatter into S1 / S1s on the T = 1 route, the lift and
projection-head kernels at T = 1 against float64, the engine against the float64 portable backend (output, loss, theta
gradients, dx and frozen dx), and the T = 1 network under a CUDA-graph Trainer, InferenceSession, a fused -> portable
-> fused state round trip and a checkpoint.  Engine tolerances are those of test_padding_gpu.py."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_engine_plan import _addresses  # noqa: E402

DEV = "cuda"


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def C_():
    from dfno_b200.ops import build
    return build.load()


# ------------------------------------------------------------------ G1a into S1 / S1s
@pytest.mark.parametrize("P,staged", [(1, False), (2, False), (4, False), (8, True)])
def test_g1a_scatters_into_s1_of_every_owner(P, staged):
    """The T = 1 chain's first stage with P destination buffers on one GPU: every owner of kz receives its slab of this
    rank's z-spectrum at this rank's y (direct) or in this rank's block (staged); nothing else is written."""
    from dfno_b200.models.fused import EnginePlan
    from dfno_b200.ops.gemm import pad_operator
    B, C, X, Y, Z, modes = 2, 4, 6, 8 * P, 64, (2, 2, 12, 1)
    r = P - 1
    pl = EnginePlan(B, 1, 1, C, 1, X, Y, Z, modes, world=P, rank=r)
    pl.finish(1)
    st = pl.chain(staged=staged)[0]
    assert st["name"] == "G1a" and st["dst"] == ("S1s" if staged else "S1")
    g = torch.Generator(device=DEV).manual_seed(P)
    A = torch.randn(st["M"], Z, device=DEV, generator=g).to(torch.bfloat16)
    op = pad_operator(pl.operators()["G1a"], device=DEV)
    guard, sentinel = 4096, -1024.0
    bufs = [torch.full((pl.n_S1 + 2 * guard,), sentinel, device=DEV, dtype=torch.bfloat16) for _ in range(P)]
    ptrs = [b[guard:].data_ptr() for b in bufs]
    (j0, n, spec, p0, pn), = pl.parts(st)
    C_().dft_gemm(A, st["M"], st["K"], st["lda"], op, 2 * n, spec.epi(), ptrs, None, 0, 0)
    torch.cuda.synchronize()
    want = (A.double() @ op[:st["N"], :Z].double().t()).cpu().numpy()                # [M, 2 KZ]
    peer, off = _addresses(spec, st["M"], n)
    for p in range(P):
        got = bufs[p].float().cpu().numpy()
        sel = peer == p
        o = off[sel] + guard
        np.testing.assert_allclose(got[o], want[:, 0::2][sel], rtol=2e-2, atol=2e-2 * np.abs(want).max())
        np.testing.assert_allclose(got[o + 1], want[:, 1::2][sel], rtol=2e-2, atol=2e-2 * np.abs(want).max())
        written = np.zeros(got.shape, dtype=bool)
        written[o] = written[o + 1] = True
        assert sel.sum() == st["M"] * pl.kzl                     # this owner's kz slab of every row
        assert (got[~written] == sentinel).all()                 # guard bands and other ranks' slots untouched


# ------------------------------------------------------------------ lift and head at T = 1
def _lift_case(Cin, Tin, pad, seed):
    B, C, X, Y, Z = 2, 20, 4, 8, 16
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, Cin, X, Y, Z, Tin, device=DEV, generator=g)
    W1 = torch.randn(1, Tin, device=DEV, generator=g) / math.sqrt(Tin)
    b1 = torch.randn(1, device=DEV, generator=g) * 0.3
    W2 = torch.randn(C, Cin, device=DEV, generator=g) / math.sqrt(Cin)
    b2 = torch.randn(C, device=DEV, generator=g) * 0.3
    Xp, Yp, Zp = X + pad[0], Y + pad[1], Z + pad[2]
    dims = [B, Cin, Tin, C, 1, X, Y, Z] + ([Xp, Yp, Zp, 1] if any(pad) else [])
    return x, (W1, b1, W2, b2), dims, (Xp, Yp, Zp)


@pytest.mark.parametrize("pad", [(0, 0, 0), (4, 4, 8)], ids=["unpadded", "padded"])
@pytest.mark.parametrize("with_dx", [False, True], ids=["no_dx", "dx"])
@pytest.mark.parametrize("Tin", [1, 10])
@pytest.mark.parametrize("Cin", [1, 4, 10, 16])
def test_lift_at_t1(Cin, Tin, with_dx, pad):
    x, (W1, b1, W2, b2), dims, (Xp, Yp, Zp) = _lift_case(Cin, Tin, pad, seed=100 * Cin + Tin)
    B, C, X, Y, Z = dims[0], dims[3], dims[5], dims[6], dims[7]
    h = torch.full((B * C * Xp * Yp * Zp,), 9.0, device=DEV, dtype=torch.bfloat16)
    C_().lift_fwd(x, W1, b1, W2, b2, h, dims)
    xr = x.double().requires_grad_()
    ps = [p.double().requires_grad_() for p in (W1, b1, W2, b2)]
    z1 = torch.einsum("ti,bcxyzi->bcxyzt", ps[0], xr) + ps[1]
    z1.retain_grad()
    ref = F.gelu(torch.einsum("oc,bcxyzt->boxyzt", ps[2], F.gelu(z1)) + ps[3].view(1, C, 1, 1, 1, 1))[..., 0]
    got = h.view(B, C, Xp, Yp, Zp)
    assert _rel(got[:, :, :X, :Y, :Z], ref) < 6e-3
    inner = torch.zeros_like(got, dtype=torch.bool)
    inner[:, :, :X, :Y, :Z] = True
    assert (got[~inner] == 0).all()                                     # exact zeros on pad positions
    g = torch.Generator(device=DEV).manual_seed(7)
    dh = torch.randn(B, C, Xp, Yp, Zp, device=DEV, generator=g).to(torch.bfloat16)
    ref.backward(dh[:, :, :X, :Y, :Z].double())
    grads = [torch.zeros_like(p) for p in (W1, b1, W2, b2)]
    dx = torch.full(x.shape, float("nan"), device=DEV) if with_dx else None
    C_().lift_bwd(x, W1, b1, W2, b2, dh.view(-1), *grads, dims, dx)
    err = {name: _rel(gr, p.grad) for name, gr, p in zip(("W2", "b2"), grads[2:], ps[2:])}
    err.update(_sum_errors(grads[0], grads[1], ps[0].grad, ps[1].grad, z1.grad, xr))
    if with_dx:
        assert torch.isfinite(dx).all()
        err["dx"] = _rel(dx, xr.grad)
    print({k: round(v, 6) for k, v in err.items()})
    assert all(v < 1e-2 for v in err.values()), err


def _sum_errors(gW1, gb1, want_W1, want_b1, dz1, x):
    """Errors of the linear1 gradients relative to the sums of their terms' magnitudes.  At T = 1 (and T_in = 1) each
    is ONE sum over every position, b1 of dz1 = dL/d(W1 x + b1) and W1 of dz1 * x, which cancels to a small fraction of
    its terms: a norm-relative error would measure that cancellation, not the arithmetic.  dz1: [..., T], x: [..., Tin]"""
    f64 = lambda t: t.detach().double().cpu()                        # noqa: E731
    dz1, xx = f64(dz1).flatten(0, -2), f64(x).flatten(0, -2)         # [positions, T], [positions, Tin]
    scale_W = torch.einsum("pt,pi->ti", dz1.abs(), xx.abs())
    scale_b = dz1.abs().sum(0)
    eW = ((f64(gW1).view(scale_W.shape) - f64(want_W1).view(scale_W.shape)).abs() / scale_W).max()
    eb = ((f64(gb1).view(scale_b.shape) - f64(want_b1).view(scale_b.shape)).abs() / scale_b).max()
    return {"W1/terms": float(eW), "b1/terms": float(eb)}


def _head_engine(O, pad):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    return FusedDistributedFNO(P_x, [2, 1, 8, 12, 16, 1], 1, 20, (2, 2, 4, 1), num_blocks=1, device=torch.device(DEV),
                               out_channels=O, init_seed=1, padding=pad)


@pytest.mark.parametrize("pad", [None, (4, 4, 8, 0)], ids=["unpadded", "padded"])
@pytest.mark.parametrize("O", [1, 3])
def test_head_at_t1(O, pad):
    f = _head_engine(O, pad)
    pl = f.plan
    assert pl.T == 1 and pl.padded == (pad is not None)
    g = torch.Generator(device=DEV).manual_seed(O)
    h = torch.randn(pl.BC, pl.X, pl.Yl, 1, pl.Z, device=DEV, generator=g).to(torch.bfloat16)
    w3a, w3t = f._head_operators_cm()
    R, SR, *lim = f._head_row_digits()
    out = torch.empty(pl.B, O, pl.Xi, pl.Yli, pl.Zi, 1, device=DEV)
    if O == 1:
        f._C.head_fwd(h.view(-1), w3a, f._w4b4(), out, pl.B, pl.C, pl.S, R, SR, *lim)
    else:
        f._C.head_fwd_multi(h.view(-1), w3a, f._w4b4(), out, pl.B, pl.C, pl.S, O, pl.Si, R, SR, *lim)
    W3, b3, W4, b4 = (f._seg(n).double().requires_grad_() for n in ("linear3.W", "linear3.b", "linear4.W", "linear4.b"))
    hr = h.view(pl.B, pl.C, pl.X, pl.Yl, pl.Z)[:, :, :pl.Xi, :pl.Yli, :pl.Zi].double().requires_grad_()
    a = F.gelu(torch.einsum("hc,bcxyz->bhxyz", W3, hr) + b3.view(1, -1, 1, 1, 1))
    ref = (torch.einsum("oh,bhxyz->boxyz", W4, a) + b4.view(1, -1, 1, 1, 1)).unsqueeze(-1)
    assert _rel(out, ref) < 1e-2, _rel(out, ref)
    dy = torch.randn(ref.shape, device=DEV, generator=g)
    ref.backward(dy.double())
    gb = torch.full((pl.BC * pl.S,), float("nan"), device=DEV, dtype=torch.bfloat16)
    grads = [torch.zeros(pl.H, pl.C, device=DEV), torch.zeros(pl.H, device=DEV), torch.zeros(O * pl.H, device=DEV),
             torch.zeros(O, device=DEV)]
    amax = torch.zeros(1, device=DEV, dtype=torch.int32)
    if O == 1:
        f._C.head_bwd2(h.view(-1), w3a, w3t, W4.detach().float().view(-1), dy.view(-1), amax, gb, *grads, pl.B,
                       pl.C, pl.S, R, SR, *lim)
    else:
        f._C.head_bwd_multi(h.view(-1), w3a, w3t, W4.detach().float().view(-1), dy.view(-1), amax, gb, *grads, pl.B,
                            pl.C, pl.S, O, pl.Si, R, SR, *lim)
    gv = gb.view(pl.B, pl.C, pl.X, pl.Yl, pl.Z).float()
    inner = torch.zeros_like(gv, dtype=torch.bool)
    inner[:, :, :pl.Xi, :pl.Yli, :pl.Zi] = True
    assert (gv[~inner] == 0).all()
    assert _rel(gv[:, :, :pl.Xi, :pl.Yli, :pl.Zi], hr.grad) < 2e-2, _rel(gv[:, :, :pl.Xi, :pl.Yli, :pl.Zi], hr.grad)
    for name, got, p in zip(("W3", "b3", "W4", "b4"), grads, (W3, b3, W4, b4)):
        assert _rel(got.view(p.shape), p.grad) < 2e-2, (name, _rel(got.view(p.shape), p.grad))


# ------------------------------------------------------------------ engine against the float64 portable backend
def _pair(in_shape, width, modes, padding=None, O=1, blocks=2, seed=0):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    torch.manual_seed(seed)
    dev = torch.device(DEV)
    ref = d.DistributedFNO(P_x, in_shape, 1, width, modes, num_blocks=blocks, device=dev, dtype=torch.float64,
                           backend="torch", out_channels=O, padding=padding)
    fused = FusedDistributedFNO(P_x, in_shape, 1, width, modes, num_blocks=blocks, device=dev, input_grad=True,
                                out_channels=O, padding=padding)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    return d, ref, fused


ENGINE = {
    "3d_w20": ([1, 1, 16, 16, 16, 1], 20, (4, 4, 4, 1), None, 1),
    "2d_w20": ([4, 1, 32, 32, 1], 20, (8, 8, 1), None, 1),
    "3d_w32": ([1, 2, 16, 16, 16, 1], 32, (4, 4, 4, 1), None, 1),
    "3d_w64": ([1, 1, 16, 16, 16, 1], 64, (4, 4, 4, 1), None, 1),
    "2d_w64": ([2, 1, 32, 32, 1], 64, (8, 8, 1), None, 1),
    "3d_o3": ([1, 1, 16, 16, 16, 1], 20, (4, 4, 4, 1), None, 3),
    "2d_cin10": ([2, 10, 32, 32, 1], 20, (8, 8, 1), None, 1),         # frames as channels
    "2d_tin10": ([2, 1, 32, 32, 10], 20, (8, 8, 1), None, 1),         # next step from 10 frames
    "3d_pad": ([1, 1, 16, 16, 16, 1], 20, (4, 4, 4, 1), (4, 4, 8, 0), 1),
    "2d_pad_o3": ([2, 3, 24, 24, 1], 20, (8, 8, 1), (8, 8, 0), 3),    # Darcy-like: padded, several fields
    "3d_round1": ([1, 1, 8, 8, 72, 1], 20, (2, 2, 34, 1), None, 1),  # 2 * KZ = 136 > 128
}


def _engine_errors(d, ref, fused, x):
    xr = x.double().requires_grad_()
    xf = x.clone().requires_grad_()
    z1 = []                                                   # linear1's output, for the linear1 gradient scales

    def keep(module, inputs, out):
        out.retain_grad()
        z1.append(out)
    hook = ref.linear1.register_forward_hook(keep)
    y_ref = ref(xr)
    hook.remove()
    y = fused(xf)
    assert y.shape == y_ref.shape
    err = {"fwd": _rel(y, y_ref)}
    # a target correlated with the output, so that the weight-gradient sums do not cancel to a small fraction of
    # their terms (which a norm-relative check would then measure instead of the arithmetic)
    t = 0.5 * y_ref.detach() + 0.1 * torch.randn_like(y_ref)
    loss_ref = ((y_ref - t) ** 2).mean()
    loss = ((y - t.float()) ** 2).mean()
    err["loss"] = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    loss_ref.backward()
    loss.backward()
    err["dx"] = _rel(xf.grad, xr.grad)
    for p in ref.parameters():
        p.data = p.grad if p.grad is not None else torch.zeros_like(p.data)
    G = d.gather_global_state(ref, to_all=True)
    got = {}
    for name, (off, shape) in fused.plan.segments.items():
        got[name] = fused.theta.grad[off:off + int(np.prod(shape))].view(shape).cpu()
        if name.endswith(".spectral"):
            Gs = G[name] if G[name].dim() == 6 else G[name].unsqueeze(2)
            want = torch.view_as_real(Gs.permute(0, 1, 4, 5, 3, 2).contiguous()).reshape(shape)
        else:
            want = G[name].reshape(shape)
        if not name.startswith("linear1."):        # one sum per entry at T = 1: checked against its terms below
            err[name] = _rel(got[name], want)
    err.update({"linear1." + k: v for k, v in _sum_errors(got["linear1.W"], got["linear1.b"], G["linear1.W"],
                                                         G["linear1.b"], z1[0].grad, xr).items()})
    # frozen weights: dx alone, theta.grad left as it was
    before = fused.theta.grad.clone()
    fused.theta.requires_grad_(False)
    xz = x.clone().requires_grad_()
    ((fused(xz) - t.float()) ** 2).mean().backward()
    fused.theta.requires_grad_(True)
    err["frozen_dx"] = _rel(xz.grad, xr.grad)
    err["frozen_theta_grad_kept"] = bool(torch.equal(fused.theta.grad, before))
    return err


def _within(err):
    bad = [k for k in ("fwd", "loss") if not err[k] < 2e-2]
    bad += [k for k in err if k in ("dx", "frozen_dx") or "." in k if not err[k] < 3e-2]
    return bad + ([] if err["frozen_theta_grad_kept"] else ["frozen_theta_grad_kept"])


@pytest.mark.parametrize("name", list(ENGINE))
def test_t1_engine_matches_float64_portable_backend(name):
    in_shape, width, modes, padding, O = ENGINE[name]
    d, ref, fused = _pair(in_shape, width, modes, padding, O)
    pl = fused.plan
    assert not pl.has_t and fused.front is None and "Z1U" not in fused.ws
    assert [s["name"] for s in fused.chain_desc if s["name"] in ("G1b", "iG1b")] == []
    assert pl.fused_pw == (name != "3d_round1")
    x = torch.randn(*in_shape, device=DEV)
    err = _engine_errors(d, ref, fused, x)
    print(name, {k: (round(v, 5) if isinstance(v, float) else v) for k, v in err.items()})
    assert not _within(err), (_within(err), err)


def test_t1_check_rejects_swapped_g2_rows():
    """Sensitivity: the same check fails when two rows of the G2 operator (the y-DFT of modes 0 and 1) are swapped."""
    in_shape, width, modes, padding, O = ENGINE["3d_w20"]
    d, ref, fused = _pair(in_shape, width, modes, padding, O)
    G2 = fused.ops["G2"]
    G2[[0, 2]] = G2[[2, 0]]
    x = torch.randn(*in_shape, device=DEV)
    with torch.no_grad():
        e = _rel(fused(x), ref(x.double()))
    print("swapped G2 rows: forward rel err", e)
    assert not e < 2e-2, e


# ------------------------------------------------------------------ end to end
def test_t1_trainer_inference_round_trip_and_checkpoint(tmp_path):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    dev = torch.device(DEV)
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1))
    in_shape, modes = [4, 3, 32, 32, 1], (8, 8, 1)
    net = d.DistributedFNO(P_x, in_shape, 1, 20, modes, num_blocks=2, device=dev, dtype=torch.bfloat16,
                           padding=(8, 8, 0), init_seed=0)
    assert isinstance(net, FusedDistributedFNO) and not net.plan.has_t
    opt = d.FusedAdam(net, lr=1e-2)
    crit = d.DistributedRelativeLpLoss(P_x, engine=net)
    tr = d.Trainer(net, crit, opt, device=dev, cuda_graph=True)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(*in_shape, generator=g).pin_memory()
    y = (0.5 * x[:, :1] + 0.2 * x[:, 1:2] * x[:, 2:3]).contiguous().pin_memory()       # a steady map of the inputs
    losses = [tr.step(x, y, next_batch=(x, y)) for _ in range(30)]
    print("losses", losses[0], losses[-1])
    assert tr._graph is not None
    assert all(math.isfinite(v) for v in losses) and losses[-1] < 0.95 * losses[0], losses
    # the step runs the engine's kernels: no FFT library on the T = 1 route
    from torch.profiler import ProfilerActivity, profile
    xd, yd = x.to(dev), y.to(dev)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        crit(net(xd), yd).backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("dft_gemm" in n for n in names), names
    assert not [n for n in names if "fft" in n.lower()], names
    sess = d.InferenceSession(net, device=dev, cuda_graph=True)
    xs = [torch.randn(*in_shape, generator=g).pin_memory() for _ in range(2)]
    outs = [sess.run(v).clone() for v in xs]
    with torch.no_grad():
        for v, o in zip(xs, outs):
            want = net(v.to(dev)).cpu()
            assert torch.allclose(o, want, atol=1e-5, rtol=1e-4), float((o - want).abs().max())
    # fused -> canonical state -> portable -> canonical state -> fused: the same outputs
    port = d.DistributedFNO(P_x, in_shape, 1, 20, modes, num_blocks=2, device=dev, dtype=torch.float32,
                            backend="torch", padding=(8, 8, 0))
    d.load_global_state(port, d.gather_global_state(net, to_all=True), strict=False)
    back = FusedDistributedFNO(P_x, in_shape, 1, 20, modes, num_blocks=2, device=dev, padding=(8, 8, 0), init_seed=6)
    d.load_global_state(back, d.gather_global_state(port, to_all=True), strict=False)
    xd = xs[0].to(dev)
    with torch.no_grad():
        ya, yb, yp = net(xd), back(xd), port(xd)
    assert torch.equal(ya, yb)
    assert _rel(ya, yp) < 2e-2, _rel(ya, yp)
    # checkpoint at T = 1
    d.save_checkpoint(net, str(tmp_path), epoch=1)
    other = FusedDistributedFNO(P_x, in_shape, 1, 20, modes, num_blocks=2, device=dev, padding=(8, 8, 0), init_seed=9)
    assert not torch.equal(other.theta, net.theta)
    d.load_checkpoint(other, str(tmp_path), epoch=1)
    assert torch.equal(other.theta, net.theta)
    with torch.no_grad():
        assert torch.equal(other(xd), ya)
