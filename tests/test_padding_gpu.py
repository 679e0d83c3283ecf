"""``padding=`` on the fused engine (one H100): the padded network against the float64 portable backend with the same
weights, the padded-layout lift and head kernels on their own, and a padded network training under a CUDA graph."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _pair(in_shape, nt, width, modes, padding, out_channels=1, blocks=2, seed=0):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    torch.manual_seed(seed)
    dev = torch.device("cuda")
    ref = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev, dtype=torch.float64,
                           backend="torch", out_channels=out_channels, padding=padding)
    fused = FusedDistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev, input_grad=True,
                                out_channels=out_channels, padding=padding)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    return d, ref, fused


@pytest.mark.parametrize("in_shape,nt,width,modes,padding,O", [
    ([10, 1, 64, 64, 10], 40, 20, (8, 8, 8), (0, 0, 8), 1),           # Navier-Stokes: time only
    ([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), (0, 0, 8, 0), 1),     # z only
    ([1, 2, 12, 8, 24, 3], 12, 20, (2, 4, 6, 7), (4, 0, 8, 4), 1),    # x, z and t together
    ([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), (0, 4, 0, 0), 1),     # y (the pencil axis) at one rank
    ([1, 1, 16, 16, 16, 1], 30, 20, (4, 4, 4, 8), (0, 0, 0, 2), 1),   # two-phase T = 30, T % 4 != 0
    ([1, 8, 16, 16, 16, 2], 8, 20, (4, 4, 4, 3), (0, 0, 8, 2), 1),    # 8 input channels (many-channel lift)
    ([1, 1, 16, 16, 16, 1], 8, 20, (4, 4, 4, 3), (4, 0, 8, 2), 3),    # 3 output fields
    ([1, 1, 16, 16, 16, 1], 8, 64, (4, 4, 4, 3), (0, 0, 8, 2), 1),    # width 64
])
def test_padded_engine_matches_float64_portable_backend(in_shape, nt, width, modes, padding, O):
    d, ref, fused = _pair(in_shape, nt, width, modes, padding, out_channels=O)
    assert fused.plan.padded
    x = torch.randn(*in_shape, device="cuda")
    xr = x.double().requires_grad_()
    xf = x.clone().requires_grad_()
    y_ref = ref(xr)
    y = fused(xf)
    assert y.shape == y_ref.shape
    print("forward rel err", _rel(y, y_ref))
    assert _rel(y, y_ref) < 2e-2, _rel(y, y_ref)
    t = torch.randn_like(y_ref)
    loss_ref = ((y_ref - t) ** 2).mean()
    loss = ((y - t.float()) ** 2).mean()
    assert abs(float(loss.detach()) - float(loss_ref.detach())) < 2e-2 * float(loss_ref.detach())
    loss_ref.backward()
    loss.backward()
    print("dx rel err", _rel(xf.grad, xr.grad))
    assert _rel(xf.grad, xr.grad) < 3e-2, _rel(xf.grad, xr.grad)
    for p in ref.parameters():
        p.data = p.grad if p.grad is not None else torch.zeros_like(p.data)
    G = d.gather_global_state(ref, to_all=True)
    gflat = fused.theta.grad
    for name, (off, shape) in fused.plan.segments.items():
        got = gflat[off:off + int(torch.tensor(shape).prod())].view(shape).cpu()
        if name.endswith(".spectral"):
            Gs = G[name] if G[name].dim() == 6 else G[name].unsqueeze(2)
            want = torch.view_as_real(Gs.permute(0, 1, 4, 5, 3, 2).contiguous()).reshape(shape)
        else:
            want = G[name].reshape(shape)
        print(name, "grad rel err", _rel(got, want))
        assert _rel(got, want) < 3e-2, (name, _rel(got, want))


def test_lift_writes_exact_zeros_at_pad_positions():
    _, _, fused = _pair([1, 3, 16, 8, 16, 2], 6, 20, (4, 4, 4, 3), (4, 4, 8, 2))
    for cin in (3, 8):                                       # lift_fwd_kernel and lift_fwd_many_kernel
        if cin == 8:
            _, _, fused = _pair([1, 8, 16, 8, 16, 2], 6, 20, (4, 4, 4, 3), (4, 4, 8, 2))
        pl = fused.plan
        fused._ensure_train_buffers()
        fused._saved["h"][0].fill_(float("nan"))
        x = torch.randn(*fused.in_shape, device="cuda")
        fused(x)
        h = fused._saved["h"][0].view(pl.BC, pl.X, pl.Yl, pl.T, pl.Z).float()
        assert not torch.isnan(h).any()
        inner = torch.zeros_like(h, dtype=torch.bool)
        inner[:, :pl.Xi, :pl.Yli, :pl.Ti, :pl.Zi] = True
        assert (h[~inner] == 0).all()
        assert (h[inner] != 0).float().mean() > 0.5


def _head_case(O):
    """A padded engine and an unpadded one with the same weights, h in the padded layout (with garbage in the pad
    region: the head must not depend on it) and its interior."""
    from dfno_b200.models.fused import FusedDistributedFNO
    import dfno_b200 as d
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    kw = dict(num_blocks=1, device=torch.device("cuda"), out_channels=O, init_seed=1)
    fp = FusedDistributedFNO(P_x, [2, 1, 8, 12, 16, 1], 6, 20, (2, 2, 4, 3), padding=(4, 4, 8, 2), **kw)
    fu = FusedDistributedFNO(P_x, [2, 1, 8, 12, 16, 1], 6, 20, (2, 2, 4, 3), **kw)
    fu.theta.data.copy_(fp.theta.data)
    pp, pu = fp.plan, fu.plan
    h = torch.randn(pp.BC, pp.X, pp.Yl, pp.T, pp.Z, device="cuda").to(torch.bfloat16)
    hc = h[:, :pp.Xi, :pp.Yli, :pp.Ti, :pp.Zi].contiguous()
    return fp, fu, pp, pu, h.view(-1), hc.view(-1)


@pytest.mark.parametrize("O", [1, 3])
def test_head_forward_stores_interior_rows_only(O):
    fp, fu, pp, pu, h, hc = _head_case(O)
    w3a, _ = fp._head_operators_cm()
    n = pp.B * O * pp.Si
    sentinel = -12345.0
    out_p = torch.full((n + 4096,), sentinel, device="cuda")
    out_u = torch.full((n,), sentinel, device="cuda")
    R, SR, lim = fp._head_row_digits()
    Ru, SRu = fu._head_row_digits()
    if O == 1:
        fp._C.head_fwd(h, w3a, fp._w4b4(), out_p, pp.B, pp.C, pp.S, R, SR, lim)
        fu._C.head_fwd(hc, w3a, fu._w4b4(), out_u, pu.B, pu.C, pu.S, Ru, SRu)
    else:
        fp._C.head_fwd_multi(h, w3a, fp._w4b4(), out_p, pp.B, pp.C, pp.S, O, pp.Si, R, SR, lim)
        fu._C.head_fwd_multi(hc, w3a, fu._w4b4(), out_u, pu.B, pu.C, pu.S, O, pu.S, Ru, SRu)
    torch.cuda.synchronize()
    assert (out_u != sentinel).all()
    assert torch.equal(out_p[:n], out_u)                       # each row is computed alone: bitwise the same
    assert (out_p[n:] == sentinel).all()                       # nothing beyond the interior output


@pytest.mark.parametrize("O", [1, 3])
def test_head_backward_is_zero_on_pad_rows(O):
    fp, fu, pp, pu, h, hc = _head_case(O)
    w3a, w3t = fp._head_operators_cm()
    dy = torch.randn(pp.B * O * pp.Si, device="cuda")
    W4 = fp._seg("linear4.W").view(-1)
    res = []
    for f, pl, hh, padded in ((fp, pp, h, True), (fu, pu, hc, False)):
        g = torch.full((pl.BC * pl.S,), float("nan"), device="cuda", dtype=torch.bfloat16)
        grads = [torch.zeros(pl.H, pl.C, device="cuda"), torch.zeros(pl.H, device="cuda"),
                 torch.zeros(O * pl.H, device="cuda"), torch.zeros(O, device="cuda")]
        amax = torch.zeros(1, device="cuda", dtype=torch.int32)
        R, SR, *lim = f._head_row_digits()
        if O == 1:
            f._C.head_bwd2(hh, w3a, w3t, W4, dy, amax, g, *grads, pl.B, pl.C, pl.S, R, SR, *lim)
        else:
            f._C.head_bwd_multi(hh, w3a, w3t, W4, dy, amax, g, *grads, pl.B, pl.C, pl.S, O, pl.Si, R, SR, *lim)
        res.append((g, grads))
    torch.cuda.synchronize()
    (gp, grads_p), (gu, grads_u) = res
    gp = gp.view(pp.BC, pp.X, pp.Yl, pp.T, pp.Z).float()
    inner = torch.zeros_like(gp, dtype=torch.bool)
    inner[:, :pp.Xi, :pp.Yli, :pp.Ti, :pp.Zi] = True
    assert (gp[~inner] == 0).all()                              # exact zeros, and every pad row written
    assert torch.equal(gp[inner].view(-1), gu.float().view(-1))
    for a, b in zip(grads_p, grads_u):                          # atomics reorder the sums
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6 * float(b.abs().max())), float((a - b).abs().max())


def test_padded_network_trains_under_a_cuda_graph():
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam, FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    dev = torch.device("cuda")
    nt = 30
    net = d.DistributedFNO(P_x, [1, 1, 32, 32, 32, 1], nt, 20, (4, 4, 4, 8), num_blocks=2, device=dev,
                           dtype=torch.bfloat16, padding=(0, 0, 8, 2), init_seed=0)
    assert isinstance(net, FusedDistributedFNO) and net.plan.padded
    opt = FusedAdam(net, lr=1e-2)
    crit = d.DistributedRelativeLpLoss(P_x)
    tr = d.Trainer(net, crit, opt, device=dev, cuda_graph=True)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(1, 1, 32, 32, 32, 1, device=dev, generator=g)
    t = 0.5 * x * torch.cos(0.3 * torch.arange(nt, device=dev, dtype=torch.float32))
    with torch.no_grad():
        l0 = float(crit(net(x), t))
    for _ in range(30):
        tr.step_on_device(x, t)
    torch.cuda.synchronize()
    assert tr._graph is not None
    with torch.no_grad():
        l1 = float(crit(net(x), t))
    assert l1 == l1 and l1 < 0.95 * l0, (l0, l1)
