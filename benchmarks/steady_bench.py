"""``out_timesteps=1`` (steady problems, next-step prediction): training step on both backends, the T = 1 chain's
kernels against their traffic, and the two calls the chain with t stages would have made instead.

(a) One training step (forward, relative L2 loss, backward, Adam) through the CUDA-graph ``Trainer``, the fused
    engine against the portable fp32 backend (``torch.optim.Adam(capturable=True)``), 4 blocks, on
      2d_darcy   [16, 3, 128, 128, 1] -> 1, width 32, modes (12, 12, 1), padding (8, 8, 0)
      next_step  [20, 1, 64, 64, 10] -> 1, width 20, modes (8, 8, 1)
      3d_steady  [4, 2, 128, 128, 128, 1] -> 1, width 20, modes (12, 12, 12, 1)
    and, fused only, next_step with the 10 frames given as channels ([20, 10, 64, 64, 1]) with the many-channel
    lift's share of that step.
(b) Every kernel of the 3d_steady step alone (CUDA events over many calls) against the bytes EnginePlan.cost_model()
    counts for it, as a share of H100_COPY_GBS.
(c) The two calls the unchanged chain would make at 3d_steady: spectral_in with T = 1 (4-row tiles, K = 2 second
    GEMM) and iG1b as a K = 2 dft_gemm over T1 with the kt pitch of 4.

    python benchmarks/steady_bench.py [--iters 10] [--rounds 3]

Prints one line per measurement and one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from many_inputs_bench import gpu_state, time_ms  # noqa: E402
from dfno_b200.models.fused import H100_COPY_GBS  # noqa: E402

SHAPES = {
    "2d_darcy": dict(in_shape=[16, 3, 128, 128, 1], width=32, modes=(12, 12, 1), padding=(8, 8, 0)),
    "next_step": dict(in_shape=[20, 1, 64, 64, 10], width=20, modes=(8, 8, 1)),
    "3d_steady": dict(in_shape=[4, 2, 128, 128, 128, 1], width=20, modes=(12, 12, 12, 1)),
    "next_step_channels": dict(in_shape=[20, 10, 64, 64, 1], width=20, modes=(8, 8, 1), fused_only=True),
}


def build_trainer(cfg, backend):
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    _, P_x, _ = d.create_standard_partitions([1] * len(cfg["in_shape"]))
    fused = backend == "fused"
    net = d.DistributedFNO(P_x, cfg["in_shape"], 1, cfg["width"], cfg["modes"], num_blocks=4, device=dev,
                           dtype=torch.bfloat16 if fused else torch.float32, backend="auto" if fused else "torch",
                           padding=cfg.get("padding"), init_seed=0)
    assert isinstance(net, d.FusedDistributedFNO) == fused
    opt = d.FusedAdam(net, lr=1e-4) if fused else torch.optim.Adam(net.parameters(), lr=1e-4, capturable=True)
    crit = d.DistributedRelativeLpLoss(P_x, engine=net) if fused else d.DistributedRelativeLpLoss(P_x)
    tr = d.Trainer(net, crit, opt, device=dev, cuda_graph=True)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(*cfg["in_shape"], device=dev, generator=g)
    y = torch.randn(*cfg["in_shape"][:1], 1, *cfg["in_shape"][2:-1], 1, device=dev, generator=g)
    return net, tr, (lambda: tr.step_on_device(x, y))


def steps(name, cfg, a, res):
    backends = ("fused",) if cfg.get("fused_only") else ("fused", "torch")
    fns, keep = {}, {}
    for b in backends:
        net, tr, fn = build_trainer(cfg, b)
        time_ms(fn, 1, a.warmup)
        keep[b] = (net, tr)
        fns[b] = fn
        res["graph_captured"][f"{name} {b}"] = tr._graph is not None
    per = {b: [] for b in backends}
    for _ in range(a.rounds):
        for b, fn in fns.items():
            per[b].append(time_ms(fn, a.iters, 1))
    for b, v in per.items():
        res["step_ms"][f"{name} {b}"] = round(statistics.median(v), 3)
        print(f"{name:18s} {b:5s} step: median {statistics.median(v):8.3f} ms over {len(v)} windows "
              f"({min(v):.3f} .. {max(v):.3f}), CUDA graph {'yes' if keep[b][1]._graph is not None else 'no'}")
    if "torch" in per:
        sp = statistics.median(per["torch"]) / statistics.median(per["fused"])
        res["step_ms"][f"{name} speedup"] = round(sp, 2)
        print(f"{name:18s} portable fp32 / fused: {sp:.2f}x")
    if cfg.get("fused_only"):          # the many-channel lift's share of the step
        net = keep["fused"][0]
        lift = lift_ms(net, a)
        share = (lift["lift fwd"] + lift["lift bwd"]) / statistics.median(per["fused"])
        res["lift_share"][name] = dict(lift, share=round(share, 3))
        print(f"{name:18s} lift fwd {lift['lift fwd']:.3f} ms + bwd {lift['lift bwd']:.3f} ms = {100 * share:.1f} % "
              f"of the step")
    del keep, fns
    torch.cuda.empty_cache()


def lift_ms(net, a):
    pl, C_ = net.plan, net._C
    dev = torch.device("cuda", 0)
    x = torch.randn(pl.B, pl.Cin, pl.Xi, pl.Yli, pl.Zi, pl.Tin, device=dev)
    h = torch.empty(pl.n_act, device=dev, dtype=torch.bfloat16)
    gf = torch.zeros(pl.n_theta, device=dev)
    seg = net._seg
    lw = [seg("linear1.W"), seg("linear1.b"), seg("linear2.W"), seg("linear2.b")]
    lg = [seg("linear1.W", gf), seg("linear1.b", gf), seg("linear2.W", gf), seg("linear2.b", gf)]
    g = (torch.randn(pl.n_act, device=dev) * 1e-3).to(torch.bfloat16)
    calls = {"lift fwd": lambda: C_.lift_fwd(x, *lw, h, net._lift_dims()),
             "lift bwd": lambda: C_.lift_bwd(x, *lw, g, *lg, net._lift_dims(), None)}
    return {k: round(statistics.median([time_ms(fn, 2 * a.iters, 2) for _ in range(a.rounds)]), 4)
            for k, fn in calls.items()}


def kernels(a, res):
    """(b) and (c) on the 3d_steady engine's own buffers"""
    from dfno_b200.ops.gemm import ScatterSpec, pad_operator
    from dfno_b200.ops import operators as OPS
    dev = torch.device("cuda", 0)
    net, _, _ = build_trainer(SHAPES["3d_steady"], "fused")
    pl, C_ = net.plan, net._C
    assert not pl.has_t and net.front is None
    net._ensure_train_buffers()
    cm = {n: b for n, _, b, _ in pl.cost_model()["stages"]}
    rnd = lambda n: (torch.randn(n, device=dev) * 0.1).to(torch.bfloat16)  # noqa: E731
    h, pre, g = rnd(pl.n_act), rnd(pl.n_act), rnd(pl.n_act)
    for k in ("S1", "S2", "S3w", "S4", "T2", "T1"):
        net.ws[k].copy_(rnd(net.ws[k].numel()))
    bufs = {"src": h, "S1": net.ws["S1"], "S2": net.ws["S2"], "S3": net.ws["S3w"], "S4": net.ws["S4"],
            "T2": net.ws["T2"], "T1": net.ws["T1"], "dst": g}
    calls = {}
    for st in net.chain_desc:
        if "N" in st and st["name"] != "iG1a":
            calls[st["name"]] = (lambda st=st: net._gemm(st, bufs, adj=False), cm[st["name"]])
    R = net._seg("blocks.0.spectral")
    Wb = net._seg("blocks.0.linear.W")
    gR = torch.zeros_like(R)
    gW = torch.zeros_like(Wb)
    op = net.ops["iG1a"]
    L, K1 = pl.X * pl.Yl * pl.T, 2 * pl.KZ
    calls.update({
        "spectral_mix fwd": (lambda: C_.spectral_mix_fwd(bufs["S3"], R, bufs["S4"], pl.B, pl.C, pl.Q),
                             cm["spectral_mix fwd"]),
        "spectral_mix bwd": (lambda: C_.spectral_mix_bwd(bufs["S3"], R, bufs["S3"], bufs["S4"], gR, False, pl.B, pl.C,
                                                         pl.Q), cm["spectral_mix bwd"]),
        "spectral_out fwd": (lambda: C_.spectral_out(bufs["T1"], h, op, Wb, False, pre, g, pl.B, pl.C, L, pl.Z, K1,
                                                     True, True), cm["spectral_out fwd"]),
        "spectral_out adj": (lambda: C_.spectral_out(bufs["T1"], pre, net.ops["iG1a_adj"], Wb, True, None, g, pl.B,
                                                     pl.C, L, pl.Z, K1, False, False), cm["spectral_out adj"]),
        "dpre_dw": (lambda: C_.dpre_dw(g, pre, h, gW, pl.B, pl.C, L, pl.Z), cm["dpre_dw"]),
    })
    lift = lift_ms(net, a)
    res["kernels"] = {}
    for k, (fn, nbytes) in calls.items():
        ms = statistics.median([time_ms(fn, a.iters, 2) for _ in range(a.rounds)])
        res["kernels"][k] = dict(ms=round(ms, 4), gb=round(nbytes / 1e9, 4),
                                 copy_rate_share=round(nbytes / (ms * 1e-3) / 1e9 / H100_COPY_GBS, 3))
        print(f"3d_steady {k:17s} {ms:8.4f} ms  {nbytes / 1e9:7.3f} GB  "
              f"{100 * res['kernels'][k]['copy_rate_share']:5.1f} % of the copy rate")
    for k, ms in lift.items():
        res["kernels"][k] = dict(ms=ms, gb=round(cm[k] / 1e9, 4),
                                 copy_rate_share=round(cm[k] / (ms * 1e-3) / 1e9 / H100_COPY_GBS, 3))
        print(f"3d_steady {k:17s} {ms:8.4f} ms  {cm[k] / 1e9:7.3f} GB  "
              f"{100 * res['kernels'][k]['copy_rate_share']:5.1f} % of the copy rate")

    # (c) the unchanged chain's two extra calls
    X, Y, Yl, KZ, kzl, BC = pl.X, pl.Y, pl.Yl, pl.KZ, pl.kzl, pl.BC
    o1 = net.ops["G1a"]
    o2 = pad_operator(OPS.fwd_complex(1, 1, False), device=dev)
    dstr = [Y * 2, X * Y * 2, X * Y * 2, kzl * X * Y * 2]
    why = C_.spectral_in_check(o1.shape[0], o1.shape[1], o2.shape[0], o2.shape[1], 1, 0, dstr, BC, X, Yl, 1, pl.Z,
                               KZ, 1)
    res["unchanged_chain"] = {}
    if why:
        print(f"spectral_in refuses T = 1 here: {why}")
        res["unchanged_chain"]["spectral_in"] = why
    else:
        fn = lambda: C_.spectral_in(h, o1, o2, [net.ws["S1"].data_ptr()], 0, dstr, BC, X, Yl, 1, pl.Z, KZ, 1)  # noqa
        ms = statistics.median([time_ms(fn, a.iters, 2) for _ in range(a.rounds)])
        nbytes = cm["G1a"]
        res["unchanged_chain"]["spectral_in"] = dict(ms=round(ms, 4), gb=round(nbytes / 1e9, 4))
        print(f"unchanged chain: spectral_in (T = 1) {ms:8.4f} ms for {nbytes / 1e9:.3f} GB "
              f"(G1a on this route: {res['kernels']['G1a']['ms']:.4f} ms)")
    mtp4 = 4                                               # the kt pitch the chain with t stages gives T1
    T1p = torch.zeros(pl.n_T1 * mtp4, device=dev, dtype=torch.bfloat16)
    U = torch.empty(pl.n_T1, device=dev, dtype=torch.bfloat16)
    M = BC * X * Yl * KZ
    spec = ScatterSpec(rows=[(KZ, 2), (BC * X * Yl, KZ * 2)], cols=(1, KZ * 2, 0))
    opb = pad_operator(OPS.inv_complex_hermitian(1, 1), device=dev)
    fn = lambda: C_.dft_gemm(T1p, M, 2, 2 * mtp4, opb, 2, spec.epi(), [U.data_ptr()], None, 0, 0)  # noqa: E731
    ms = statistics.median([time_ms(fn, a.iters, 2) for _ in range(a.rounds)])
    nbytes = 2 * pl.n_T1 * 2                               # T1 (valid part) + U, as the t-stage cost model counts
    res["unchanged_chain"]["iG1b"] = dict(ms=round(ms, 4), gb=round(nbytes / 1e9, 4), M=M)
    print(f"unchanged chain: iG1b as a K = 2 dft_gemm, M = {M:,d}: {ms:8.4f} ms for {nbytes / 1e9:.3f} GB")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the fused and portable steps")
    ap.add_argument("--skip-steps", action="store_true", help="only (b) and (c)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("steady_bench.py needs a GPU")
    res = {**gpu_state(), "step_ms": {}, "graph_captured": {}, "lift_share": {}}
    if not a.skip_steps:
        for name, cfg in SHAPES.items():
            steps(name, cfg, a, res)
    kernels(a, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
