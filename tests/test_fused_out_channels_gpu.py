"""The fused engine with several output channels against the portable backend on one H100: outputs, every parameter
gradient, dL/dx, the frozen-weight backward, the CUDA-graph trainer, the inference session and checkpoints."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _pair(in_shape, nt, width, modes, O, blocks=2, seed=0, dtype=torch.float32, input_grad=False):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    torch.manual_seed(seed)
    dev = torch.device("cuda")
    ref = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev, dtype=dtype,
                           backend="torch", out_channels=O)
    fused = FusedDistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev, out_channels=O,
                                input_grad=input_grad)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    return d, P_x, ref, fused


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


SHAPES = [
    ([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3)),            # small 3-D + time
    ([2, 3, 32, 32, 4], 10, 20, (4, 4, 3)),                 # 2-D + time (Navier-Stokes-like), C_in > 1, T_in > 1
    ([1, 2, 8, 8, 16, 1], 8, 24, (2, 2, 4, 4)),             # widest multi-output width (KR = 32 kernels)
    ([2, 1, 12, 8, 24, 3], 10, 16, (2, 4, 6, 5)),           # B = 2, T_in = 3
]


@pytest.mark.parametrize("O", [2, 3, 4])
@pytest.mark.parametrize("in_shape,nt,width,modes", SHAPES)
def test_forward_backward_match_portable_backend(in_shape, nt, width, modes, O):
    d, _, ref, fused = _pair(in_shape, nt, width, modes, O)
    x = torch.randn(*in_shape, device="cuda")
    y_ref, y = ref(x), fused(x)
    assert y.shape == y_ref.shape and y.shape[1] == O
    # every plane is checked on its own, against the scale of the whole output: a random-init head can give one
    # channel a small norm (cancellation in its 128-term sum), so a per-plane relative error would measure that
    plane = [float((y[:, o] - y_ref[:, o]).norm() / y_ref.norm() * O ** 0.5) for o in range(O)]
    print("forward rel err", _rel(y, y_ref), "per plane", plane)
    assert _rel(y, y_ref) < 2e-2
    assert all(e < 2e-2 for e in plane), plane
    t = torch.randn_like(y_ref)
    ((y_ref - t) ** 2).mean().backward()
    ((y - t) ** 2).mean().backward()
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


def test_shape_with_partial_head_tile():
    """2-D + time with S = 12 * 24 * 6 = 1728 positions per slab: the last head tile is partial"""
    in_shape, nt = [2, 1, 12, 24, 1], 6
    assert (12 * 24 * nt) % 128 != 0
    d, _, ref, fused = _pair(in_shape, nt, 8, (2, 2, 2), 3)
    x = torch.randn(*in_shape, device="cuda")
    y_ref, y = ref(x), fused(x)
    assert _rel(y, y_ref) < 2e-2
    t = torch.randn_like(y_ref)
    ((y - t) ** 2).mean().backward()
    ((y_ref - t) ** 2).mean().backward()
    off, shape = fused.plan.segments["linear4.W"]
    got = fused.theta.grad[off:off + shape[0] * shape[1]].view(shape)
    assert _rel(got, ref.linear4.W.grad) < 3e-2


def test_input_gradient_and_frozen_backward():
    in_shape, nt, width, modes = [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3)
    d, _, ref, fused = _pair(in_shape, nt, width, modes, 3, dtype=torch.float64, input_grad=True)
    x = torch.randn(*in_shape, device="cuda")
    t = torch.randn(1, 3, 16, 16, 16, nt, device="cuda")
    xr = x.double().requires_grad_()
    ((ref(xr) - t.double()) ** 2).mean().backward()
    xf = x.clone().requires_grad_()
    ((fused(xf) - t) ** 2).mean().backward()
    print("dx rel err", _rel(xf.grad, xr.grad))
    assert xf.grad.shape == x.shape and _rel(xf.grad, xr.grad) < 5e-2
    # frozen weights: dx only, theta.grad untouched
    before = fused.theta.grad.clone()
    fused.theta.requires_grad_(False)
    xg = x.clone().requires_grad_()
    ((fused(xg) - t) ** 2).mean().backward()
    assert torch.equal(fused.theta.grad, before)
    assert _rel(xg.grad, xr.grad) < 5e-2


def test_cuda_graph_trainer_and_inference_session():
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam, FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    shape = [1, 1, 16, 16, 16, 1]
    x, t = torch.randn(*shape, device="cuda"), torch.randn(1, 2, 16, 16, 16, 8, device="cuda")
    thetas, losses = [], []
    for graph in (False, True):
        net = FusedDistributedFNO(P_x, shape, 8, 8, (4, 4, 4, 3), num_blocks=1, device=torch.device("cuda"),
                                  init_seed=3, out_channels=2)
        opt = FusedAdam(net, lr=1e-2)
        tr = d.Trainer(net, d.DistributedRelativeLpLoss(P_x, engine=net), opt, device=torch.device("cuda"),
                       cuda_graph=graph)
        for _ in range(4):
            tr.step_on_device(x, t)
        torch.cuda.synchronize()
        assert (tr._graph is not None) == graph
        thetas.append(net.theta.detach().clone())
        with torch.no_grad():
            losses.append(float(d.DistributedRelativeLpLoss(P_x)(net(x), t)))
    assert float((thetas[0] - thetas[1]).norm() / thetas[0].norm()) < 2e-3
    sess = d.InferenceSession(net)
    y = sess.run(x.cpu())
    with torch.no_grad():
        want = net(x).cpu()
    assert y.shape == (1, 2, 16, 16, 16, 8) and _rel(y, want) < 1e-5


def test_checkpoint_round_trip_fused_portable(tmp_path):
    import dfno_b200 as d
    in_shape, nt, width, modes = [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3)
    d_, P_x, ref, fused = _pair(in_shape, nt, width, modes, 3)
    with torch.no_grad():
        fused.theta.add_(0.01 * torch.randn_like(fused.theta))
    state = d.gather_global_state(fused, to_all=True)
    assert tuple(state["linear4.W"].shape) == (3, 128)
    torch.manual_seed(9)
    port = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=2, device=torch.device("cuda"),
                            backend="torch", out_channels=3)
    d.load_global_state(port, state, strict=False)         # the engine has no batch-norm entries
    x = torch.randn(*in_shape, device="cuda")
    assert _rel(fused(x), port(x)) < 2e-2
    back = d.gather_global_state(port, to_all=True)
    fused2 = _pair(in_shape, nt, width, modes, 3, seed=1)[3]
    d.load_global_state(fused2, back)
    v1, v2 = fused.named_views(), fused2.named_views()
    assert all(torch.equal(v1[k], v2[k]) for k in v1)
    # across different out_channels the load fails and names the shapes
    one = _pair(in_shape, nt, width, modes, 1)[3]
    with pytest.raises(ValueError, match=r"linear4.*\[3, 128\].*\[1, 128\]"):
        d.load_global_state(one, state)
    port1 = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=2, device=torch.device("cuda"),
                             backend="torch")
    with pytest.raises(ValueError, match=r"linear4.*\[3, 128\]"):
        d.load_global_state(port1, state, strict=False)


def test_round1_shape_with_two_outputs_runs_on_the_portable_backend():
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    args = (P_x, [1, 1, 8, 8, 80, 1], 4, 8, (2, 2, 34, 2))
    kw = dict(num_blocks=1, device=torch.device("cuda"), dtype=torch.bfloat16)
    assert isinstance(d.DistributedFNO(*args, **kw), FusedDistributedFNO)
    net = d.DistributedFNO(*args, out_channels=2, **kw)
    assert not isinstance(net, FusedDistributedFNO)
    y = net(torch.randn(1, 1, 8, 8, 80, 1, device="cuda", dtype=torch.bfloat16))
    assert y.shape == (1, 2, 8, 8, 80, 4)
    with pytest.raises(ValueError, match="round-2"):
        d.DistributedFNO(*args, out_channels=2, backend="fused", **kw)
