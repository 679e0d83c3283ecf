"""Fused sm_90a engine vs the portable fp32 backend on one H100."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _pair(in_shape, nt, width, modes, blocks=2, seed=0):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    torch.manual_seed(seed)
    dev = torch.device("cuda")
    ref = d.DistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev,
                           dtype=torch.float32, backend="torch")
    fused = FusedDistributedFNO(P_x, in_shape, nt, width, modes, num_blocks=blocks, device=dev)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    return d, ref, fused


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


@pytest.mark.parametrize("in_shape,nt,width,modes", [
    ([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3)),
    ([2, 2, 12, 8, 24, 3], 12, 20, (2, 4, 6, 7)),
    ([1, 1, 256, 256, 8, 1], 4, 8, (4, 6, 2, 2)),          # axes > 128: K = 512 stages, column-part inverse stages
    ([1, 2, 12, 12, 16, 1], 30, 20, (4, 4, 4, 8)),         # T = 30 (reference two-phase run / demo): padded t pitch
    ([2, 1, 32, 32, 10], 16, 20, (4, 4, 4)),               # 2-D + time (reference Navier-Stokes trainer): singleton-x plan
    ([1, 3, 16, 8, 16, 2], 8, 32, (2, 2, 4, 4)),           # widest supported channel count, 3 input channels
])
def test_forward_backward_match_portable_backend(in_shape, nt, width, modes):
    d, ref, fused = _pair(in_shape, nt, width, modes)
    x = torch.randn(*in_shape, device="cuda")
    y_ref = ref(x)
    y = fused(x)
    assert y.shape == y_ref.shape
    # bf16 storage of every activation (2^-9 relative) through 2 blocks + the 128-term output sum of a random-init
    # head (heavy cancellation): the achieved error is printed; it is a few 1e-3 .. 1e-2
    print("forward rel err", _rel(y, y_ref))
    assert _rel(y, y_ref) < 2e-2, _rel(y, y_ref)
    t = torch.randn_like(y_ref)
    ((y_ref - t) ** 2).mean().backward()
    ((y - t) ** 2).mean().backward()
    g_ref = {n: p.grad for n, p in ref.named_parameters() if p.grad is not None}
    for p in ref.parameters():          # canonical form of the reference gradients
        p.data = p.grad if p.grad is not None else torch.zeros_like(p.data)
    G = d.gather_global_state(ref, to_all=True)
    views = {n: v for n, v in fused.named_views().items()}
    gflat = fused.theta.grad
    for name, (off, shape) in fused.plan.segments.items():
        got = gflat[off:off + int(torch.tensor(shape).prod())].view(shape).cpu()
        if name.endswith(".spectral"):
            pl = fused.plan
            Gs = G[name] if G[name].dim() == 6 else G[name].unsqueeze(2)      # 2-D + time: singleton kx
            want = torch.view_as_real(Gs.permute(0, 1, 4, 5, 3, 2).contiguous()).reshape(shape)
        else:
            want = G[name].reshape(shape)
        print(name, "grad rel err", _rel(got, want))
        assert _rel(got, want) < 3e-2, (name, _rel(got, want))


def test_device_gelu_matches_erf_gelu():
    from dfno_b200.ops import build
    x = torch.linspace(-9, 9, 400001, device="cuda")
    y, dy = build.load().gelu_probe(x)
    xd = x.double().requires_grad_()
    ref = torch.nn.functional.gelu(xd)
    ref.sum().backward()
    assert float((y.double() - ref).abs().max()) < 2e-6
    assert float((dy.double() - xd.grad).abs().max()) < 2e-6


def test_eval_mode_and_state_round_trip():
    d, ref, fused = _pair([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3))
    x = torch.randn(1, 1, 16, 16, 16, 1, device="cuda")
    with torch.no_grad():
        y0 = fused(x)
    y1 = fused(x)
    assert torch.allclose(y0, y1.detach())
    state = d.gather_global_state(fused, to_all=True)
    want = d.gather_global_state(ref, to_all=True)
    for k in want:
        if k.startswith(("linear", "blocks")):
            assert torch.allclose(state[k].float() if not state[k].is_complex() else torch.view_as_real(state[k]),
                                  want[k].float() if not want[k].is_complex() else torch.view_as_real(want[k]),
                                  atol=1e-6), k


def test_fused_adam_matches_torch_adam():
    from dfno_b200.models.fused import FusedAdam
    d, ref, fused = _pair([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), blocks=1)
    opt = FusedAdam(fused, lr=1e-2, weight_decay=1e-3)
    p0 = fused.theta.detach().clone()
    pt = torch.nn.Parameter(p0.clone())
    topt = torch.optim.Adam([pt], lr=1e-2, weight_decay=1e-3)
    for i in range(3):
        g = torch.randn_like(p0)
        fused.theta.grad = g.clone()
        pt.grad = g.clone()
        opt.step()
        topt.step()
    assert torch.allclose(fused.theta, pt, atol=1e-6, rtol=1e-5)


def test_stale_backward_and_input_gradients_are_refused():
    """ADVICE r1: the engine keeps ONE set of saved activations.  A backward after a second saving forward must
    raise instead of using the wrong activations; a no-grad forward in between is harmless; dL/dx is refused."""
    d, ref, fused = _pair([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3))
    x = torch.randn(1, 1, 16, 16, 16, 1, device="cuda")
    y1 = fused(x)
    with torch.no_grad():
        fused(x * 2)                              # evaluation in between: separate buffers
    y1.square().mean().backward()                 # still valid
    g1 = fused.theta.grad.clone()
    y2 = fused(x)
    y2.square().mean().backward()
    assert torch.allclose(g1, fused.theta.grad, rtol=1e-3, atol=1e-6 * float(g1.abs().max()))
    ya = fused(x)
    yb = fused(x * 0.5)
    with pytest.raises(RuntimeError, match="overwritten"):
        ya.sum().backward()
    yb.sum().backward()
    with pytest.raises(RuntimeError, match="input gradients"):
        fused(x.clone().requires_grad_())


def test_fused_checkpoint_files_reassemble_offline(tmp_path):
    """ADVICE r1: per-rank files of the fused engine hold one flat `theta`; with the segment table stored next
    to them they are re-assembled into the canonical state without the module (and no longer load 'nothing')."""
    from dfno_b200.utils.checkpoint import assemble_global_from_files, reshard_checkpoint
    d, ref, fused = _pair([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3))
    d.save_checkpoint(fused, str(tmp_path), epoch=None)
    want = d.gather_global_state(fused, to_all=True)
    got = assemble_global_from_files(str(tmp_path), (1, 1, 1, 1, 1, 1), fused.block_in_shape, fused.modes)
    assert sorted(got) == sorted(want)
    for k in want:
        assert torch.equal(torch.view_as_real(got[k]) if got[k].is_complex() else got[k],
                           torch.view_as_real(want[k]) if want[k].is_complex() else want[k]), k
    d2, ref2, fused2 = _pair([1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3), seed=5)
    assert not torch.equal(fused2.theta, fused.theta)
    reshard_checkpoint(str(tmp_path), fused2)                        # fused files -> another engine instance
    assert torch.equal(fused2.theta, fused.theta)
    reshard_checkpoint(str(tmp_path), ref2)                          # ... and into the portable backend
    y0, y1 = ref2(torch.ones(1, 1, 16, 16, 16, 1, device="cuda")), ref(torch.ones(1, 1, 16, 16, 16, 1, device="cuda"))
    assert torch.allclose(y0, y1, atol=1e-5)
    with pytest.raises(KeyError):
        d.load_global_state(fused2, {"unrelated": torch.zeros(3)}, strict=False)


def test_cuda_graph_trainer_applies_exactly_one_update_per_step():
    """ADVICE r1: warm-up + capture must not train.  Graph-replayed steps == the same number of eager steps."""
    from dfno_b200.models.fused import FusedAdam, FusedDistributedFNO
    import dfno_b200 as d
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    shape = [1, 1, 16, 16, 16, 1]
    x, t = torch.randn(*shape, device="cuda"), torch.randn(1, 1, 16, 16, 16, 8, device="cuda")
    thetas, counts = [], []
    for graph in (False, True):
        net = FusedDistributedFNO(P_x, shape, 8, 8, (4, 4, 4, 3), num_blocks=1, device=torch.device("cuda"), init_seed=3)
        opt = FusedAdam(net, lr=1e-2)
        tr = d.Trainer(net, d.DistributedRelativeLpLoss(P_x), opt, device=torch.device("cuda"), cuda_graph=graph)
        for _ in range(3):
            tr.step_on_device(x, t)
        torch.cuda.synchronize()
        assert (tr._graph is not None) == graph
        thetas.append(net.theta.detach().clone())
        counts.append((opt.step_count, float(opt.step_dev)))
    assert counts[0] == counts[1] == (3, 3.0), counts
    assert float((thetas[0] - thetas[1]).norm() / thetas[0].norm()) < 2e-3     # same trajectory (atomics reorder sums)


def test_fused_engine_learns_and_tracks_the_fp32_backend():
    """VERDICT r1: show that the engine LEARNS.  A learnable target (a smoothed copy of the input field, growing in
    time), 300 Adam steps: the loss of the bf16 fused engine must drop >= 5x and track the fp32 portable backend
    started from the same weights within 10 %."""
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam
    dd, ref, fused = _pair([2, 1, 16, 16, 16, 1], 8, 12, (4, 4, 4, 3), blocks=2, seed=11)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(2, 1, 16, 16, 16, 1, device="cuda", generator=g)
    k = torch.ones(1, 1, 3, 3, 3, device="cuda") / 27
    sm = torch.nn.functional.conv3d(torch.nn.functional.pad(x[..., 0], (1, 1, 1, 1, 1, 1), mode="circular"), k)
    tgt = torch.stack([sm * (1 + 0.1 * s) for s in range(8)], dim=-1)                            # [B,1,X,Y,Z,T]
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    crit = d.DistributedRelativeLpLoss(P_x)
    opt_f, opt_r = FusedAdam(fused, lr=1e-2), torch.optim.Adam([p for p in ref.parameters() if p.numel()], lr=1e-2)
    lf, lr_ = [], []
    for _ in range(300):
        opt_f.zero_grad(); l = crit(fused(x), tgt); l.backward(); opt_f.step(); lf.append(float(l))
        opt_r.zero_grad(); l = crit(ref(x), tgt); l.backward(); opt_r.step(); lr_.append(float(l))
    print("fused", lf[0], lf[-1], "fp32", lr_[0], lr_[-1])
    assert lf[-1] < lf[0] / 5, (lf[0], lf[-1])
    assert abs(lf[-1] - lr_[-1]) < 0.1 * lr_[-1] + 5e-3, (lf[-1], lr_[-1])
    mid = len(lf) // 2
    assert abs(lf[mid] - lr_[mid]) < 0.1 * lr_[mid] + 5e-3, (lf[mid], lr_[mid])
