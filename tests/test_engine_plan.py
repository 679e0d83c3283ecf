"""CPU emulation of the fused engine's stage plan: every GEMM stage is replayed in float64
with the engine's operator matrices and *its own scatter address tables* (including the
peer-selecting digits), for 1, 2 and 4 simulated ranks, and compared with torch.fft.
This validates the multi-GPU addressing (Repartition R2/R3 fused into epilogues) without a GPU."""
import numpy as np
import pytest
import torch

from dfno_b200.models.fused import EnginePlan


def _addresses(spec, M, npairs):
    """Vectorised ScatterSpec.address for all (row, pair)."""
    rows = np.arange(M, dtype=np.int64)
    off = np.full(M, spec.base_off, dtype=np.int64)
    rpeer = np.zeros(M, dtype=np.int64)
    r = rows.copy()
    for l, (radix, stride) in enumerate(spec.rows):
        last = l == len(spec.rows) - 1
        d = r if last else r % radix
        r = r if last else r // radix
        if spec.peer is not None and spec.peer[0] == "row" and spec.peer[1] == l:
            rpeer, d = d // spec.peer[2], d % spec.peer[2]
        off = off + d * stride
    j = np.arange(npairs, dtype=np.int64)
    cpeer = np.zeros(npairs, dtype=np.int64)
    if spec.peer is not None and spec.peer[0] == "col":
        cpeer, j = j // spec.peer[1], j % spec.peer[1]
    J0, SJ0, SJ1 = spec.cols
    coff = (j % J0) * SJ0 + (j // J0) * SJ1
    peer = rpeer[:, None] + cpeer[None, :]
    return peer, off[:, None] + coff[None, :]


def _run_chain(plans, ops, src, weights, adj=False, staged=False):
    """src: list (per rank) of engine-layout arrays; returns list of outputs."""
    P = len(plans)
    pl0 = plans[0]
    bufs = [dict(src=src[r].reshape(-1).copy(),
                 Z1=np.zeros(max(pl0.n_Z1, pl0.n_U)), S1=np.zeros(pl0.n_S1), S2=np.zeros(pl0.n_S2),
                 S3=np.zeros(pl0.n_S3), S4=np.zeros(pl0.n_S3), T2=np.zeros(pl0.n_T2), T1=np.zeros(pl0.n_T1),
                 S1s=np.full(pl0.n_S1, np.nan), T1s=np.full(pl0.n_T1, np.nan),
                 dst=np.zeros(pl0.n_act)) for r in range(P)]
    for b in bufs:
        b["U"] = b["Z1"]
    chains = [pl.chain(staged=staged) for pl in plans]
    for si in range(len(chains[0])):
        for r in range(P):
            st = chains[r][si]
            pl = plans[r]
            if st["name"].startswith("perm"):
                # strided permutation of 32-bit words (= complex pairs): dst walked innermost digit first
                src_w = bufs[r][st["src"]].reshape(-1, 2)
                dst_w = bufs[r][st["dst"]].reshape(-1, 2)
                idx = np.indices(st["size"][::-1]).reshape(len(st["size"]), -1)[::-1]      # digit l of every word
                so = sum(idx[l] * st["sstr"][l] for l in range(len(st["size"])))
                do = sum(idx[l] * st["dstr"][l] for l in range(len(st["size"])))
                dst_w[do] = src_w[so]
                continue
            if st["name"] == "mix":
                x = bufs[r]["S3"].reshape(pl.B, pl.C, pl.Q, 2)
                xc = x[..., 0] + 1j * x[..., 1]
                w = weights[r]                                  # [C, C, Q] complex
                y = np.einsum("biq,ioq->boq", xc, w)
                bufs[r]["S4"][:] = np.stack([y.real, y.imag], -1).reshape(-1)
                continue
            op = ops[st["op"] + ("_adj" if adj else "")].numpy()
            A = bufs[r][st["src"]][: st["M"] * st["lda"]].reshape(st["M"], st["lda"])[:, : st["K"]]
            if "scatter" in st:
                for j0, n, spec, p0, pn in pl.parts(st):         # column parts: one launch each on the GPU
                    Cm = A @ op[2 * j0:2 * (j0 + n)].T           # [M, 2n]
                    peer, off = _addresses(spec, st["M"], n)
                    peer = peer + p0
                    assert pn is None or (peer < p0 + pn).all()
                    for p in range(P):
                        sel = peer == p
                        if not sel.any():
                            continue
                        tgt = bufs[p if st.get("peer_dst") else r][st["dst"]]
                        tgt[off[sel]] = Cm[:, 0::2][sel]
                        tgt[off[sel] + 1] = Cm[:, 1::2][sel]
                    assert st.get("peer_dst") or (peer == 0).all()
            else:
                assert st["N"] <= pl.max_n
                Cm = A @ op.T                                    # [M, N]
                bufs[r][st["dst"]][: st["M"] * st["ldc"]].reshape(st["M"], st["ldc"])[:, : st["N"]] = Cm
    return [b["dst"] for b in bufs]


@pytest.mark.parametrize("P,staged,max_n", [(1, False, 256), (2, False, 256), (4, False, 256), (2, True, 256),
                                             (4, True, 256), (1, False, 8), (2, False, 8), (4, False, 8),
                                             (4, True, 8), (2, True, 8), (1, False, 6), (2, True, 6), (4, False, 6)])
def test_stage_plan_reproduces_spectral_convolution(P, staged, max_n):
    """``max_n`` below the real limit forces the column-part path (used on the GPU for axes > 128)."""
    Y, T = (8 if max_n == 256 else 16), 4
    if max_n == 6:                      # T = 6 is not a multiple of 4: Z1 carries a padded t pitch (Tp = 8)
        Y, T, max_n = 8, 6, 256
    _check_stage_plan(P, staged, 8, Y, 8, T, (2, 2, 2, 3), max_n=max_n)


@pytest.mark.parametrize("P,staged,T,pad", [(1, False, 1, None), (2, False, 1, None), (4, False, 1, None),
                                            (2, True, 1, None), (4, True, 1, None),
                                            (2, False, 4, (4, 0, 8, 2)), (4, True, 4, (4, 0, 8, 2))])
def test_stage_plan_reproduces_steady_and_padded_convolution(P, staged, T, pad):
    """The out_timesteps = 1 chain (no t stages: G1a scatters into the owners' S1 and iG2's T1 feeds the last stage)
    and a plan padded in x, z and t (the chain runs on the padded extents)."""
    _check_stage_plan(P, staged, 8, 8, 8, T, (2, 2, 2, 1 if T == 1 else 2), pad=pad)


def _check_stage_plan(P, staged, X, Y, Z, T, modes, max_n=256, pad=None):
    """The stage plan of P ranks replayed in float64 against the portable block's spectral convolution on the
    (padded) field, and the adjoint chain against it through <chain(x), g> = <x, chain_adj(g)>."""
    import dfno_b200 as d
    B, C = 2, 3
    if pad is not None:
        X, Y, Z, T = X + pad[0], Y + pad[1], Z + pad[2], T + pad[3]
    torch.manual_seed(0)
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    blk = d.DistributedFNOBlock(P1, [B, C, X, Y, Z, T], modes, dtype=torch.float64)
    # global spectral weight [C, C, KX, KY, KZ, mt] from the block's corner parameters
    Wg = torch.zeros(C, C, *blk.fft_shape[2:], dtype=torch.complex128)
    for w, sl in zip(blk.weights, blk.slices):
        Wg[sl] = w.detach()
    x = torch.randn(B, C, X, Y, Z, T, dtype=torch.float64)
    want = blk.spectral_forward(x).detach()                      # [B, C, X, Y, Z, T]

    plans = []
    for r in range(P):
        if pad is None:
            pl = EnginePlan(B, 1, 1, C, T, X, Y, Z, modes, world=P, rank=r)
        else:                           # interior extents + padding: the plan's X, Y, Z, T are the padded ones
            pl = EnginePlan(B, 1, 1, C, T - pad[3], X - pad[0], Y - pad[1], Z - pad[2], modes, world=P, rank=r,
                            pad=pad)
            assert (pl.X, pl.Y, pl.Z, pl.T) == (X, Y, Z, T)
        pl.finish(1)
        pl.max_n = max_n
        plans.append(pl)
    if max_n != 256:
        assert sum(len(plans[0].parts(st)) > 1 for st in plans[0].chain(staged=staged) if "N" in st) == 2
    if T == 1:
        assert [st["name"] for st in plans[0].chain(staged=staged) if st["name"] in ("G1b", "iG1b")] == []
    ops = plans[0].operators()
    h = x.permute(0, 1, 2, 3, 5, 4).contiguous().numpy()         # engine layout [B, C, X, Y, T, Z]
    src, weights = [], []
    for pl in plans:
        src.append(h[:, :, :, pl.y_off:pl.y_off + pl.Yl].reshape(pl.BC, X, pl.Yl, T, Z))
        wn = Wg[:, :, :, :, pl.kz_off:pl.kz_off + pl.kzl, :].permute(0, 1, 4, 5, 3, 2).contiguous()
        weights.append(wn.reshape(C, C, pl.Q).numpy())           # native [i, o, (kzl, mt, KY, KX)]
    outs = _run_chain(plans, ops, src, weights, staged=staged)
    got = np.concatenate([o.reshape(B, C, X, pl.Yl, T, Z) for o, pl in zip(outs, plans)], axis=3)
    got = torch.from_numpy(got).permute(0, 1, 2, 3, 5, 4)
    assert torch.allclose(got, want, atol=1e-10), float((got - want).abs().max())

    # adjoint chain: <chain(x), g> == <x, chain_adj(g)> with conjugated-transposed mixing
    g = torch.randn(B, C, X, Y, Z, T, dtype=torch.float64)
    gh = g.permute(0, 1, 2, 3, 5, 4).contiguous().numpy()
    gsrc = [gh[:, :, :, pl.y_off:pl.y_off + pl.Yl].reshape(pl.BC, X, pl.Yl, T, Z) for pl in plans]
    wadj = [np.conj(np.transpose(w, (1, 0, 2))) for w in weights]
    gouts = _run_chain(plans, ops, gsrc, wadj, adj=True, staged=staged)
    gx = np.concatenate([o.reshape(B, C, X, pl.Yl, T, Z) for o, pl in zip(gouts, plans)], axis=3)
    lhs = float((got * g).sum())
    rhs = float((torch.from_numpy(gx).permute(0, 1, 2, 3, 5, 4) * x).sum())
    assert abs(lhs - rhs) < 1e-9 * max(1.0, abs(lhs)), (lhs, rhs)


@pytest.mark.parametrize("P,staged", [(1, False), (2, False), (4, True), (2, True)])
def test_stage_plan_2d_plus_time_runs_as_singleton_x(P, staged):
    """A 5-D problem [B, C, X', Y', T] is the 6-D engine plan with X = 1: the x stages vanish and G2 / iG2 talk to
    the mix directly.  Oracle: the portable 5-D block (reference semantics, dfno.py:82-97 with n = 3)."""
    import dfno_b200 as d
    B, C, Xp, Yp, T = 2, 3, 8, 8, 6
    modes3 = (2, 2, 3)
    torch.manual_seed(1)
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1))
    blk = d.DistributedFNOBlock(P1, [B, C, Xp, Yp, T], modes3, dtype=torch.float64)
    Wg = torch.zeros(C, C, *blk.fft_shape[2:], dtype=torch.complex128)
    for w, sl in zip(blk.weights, blk.slices):
        Wg[sl] = w.detach()
    x = torch.randn(B, C, Xp, Yp, T, dtype=torch.float64)
    want = blk.spectral_forward(x).detach()
    plans = []
    for r in range(P):
        pl = EnginePlan(B, 1, 1, C, T, 1, Xp, Yp, (0, *modes3), world=P, rank=r)
        pl.finish(1)
        plans.append(pl)
    assert not plans[0].has_x and plans[0].KX == 1
    assert [st["name"] for st in plans[0].chain() if st["name"] in ("G3", "iG3")] == []
    ops = plans[0].operators()
    h = x.unsqueeze(2).permute(0, 1, 2, 3, 5, 4).contiguous().numpy()          # [B, C, 1, Y=X', T, Z=Y']
    src, weights = [], []
    W6 = Wg.unsqueeze(2)                                                       # [C, C, KX=1, KY, KZ, mt]
    for pl in plans:
        src.append(h[:, :, :, pl.y_off:pl.y_off + pl.Yl].reshape(pl.BC, 1, pl.Yl, T, Yp))
        wn = W6[:, :, :, :, pl.kz_off:pl.kz_off + pl.kzl, :].permute(0, 1, 4, 5, 3, 2).contiguous()
        weights.append(wn.reshape(C, C, pl.Q).numpy())
    outs = _run_chain(plans, ops, src, weights, staged=staged)
    got = np.concatenate([o.reshape(B, C, 1, pl.Yl, T, Yp) for o, pl in zip(outs, plans)], axis=3)
    got = torch.from_numpy(got).permute(0, 1, 2, 3, 5, 4).squeeze(2)
    assert torch.allclose(got, want, atol=1e-10), float((got - want).abs().max())


class _Grid:
    """Stand-in for a Partition: ``supports`` only looks at ``dim`` and ``shape``."""

    def __init__(self, *shape):
        self.shape, self.dim = list(shape), len(shape)


def test_supports_covers_the_baseline_configs():
    from dfno_b200.models.fused import supports
    # config 2: 128^3 x 20, width 20, 1 x 8 pencil
    assert supports(_Grid(1, 1, 1, 8, 1, 1), [1, 1, 128, 128, 128, 1], 20, 20, (12, 12, 12, 10))[0]
    # config 3: 256^3, width 32, 2 x 2 x 2 (folded onto the pencil; axes of 256 samples)
    assert supports(_Grid(1, 1, 2, 2, 2, 1), [1, 2, 256, 256, 256, 1], 16, 32, (12, 12, 12, 8))[0]
    # config 4: 64^3 x 32, width 24, 8 modes, 8-way time partition
    assert supports(_Grid(1, 1, 1, 1, 1, 8), [1, 1, 64, 64, 64, 1], 32, 24, (8, 8, 8, 8))[0]
    # reference two-phase trainer: 60 x 60 x 64 x 30 on 4 ranks (T % 4 != 0: padded t pitch), and the in-module
    # demo (dfno.py:359-366): 64^3 x 30 on (1,1,2,2,1,1)
    assert supports(_Grid(1, 1, 1, 4, 1, 1), [1, 2, 60, 60, 64, 1], 30, 20, (12, 12, 12, 8))[0]
    assert supports(_Grid(1, 1, 2, 2, 1, 1), [1, 1, 64, 64, 64, 1], 30, 20, (4, 4, 4, 8))[0]
    ok, why = supports(_Grid(1, 1, 1, 4, 1, 1), [1, 2, 60, 60, 64, 1], 15, 20, (12, 12, 12, 8))
    assert not ok and "T%2" in why
    assert not supports(_Grid(2, 1, 1, 4, 1, 1), [2, 1, 64, 64, 64, 1], 16, 20, (8, 8, 8, 8))[0]      # data parallel
    assert not supports(_Grid(1, 1, 1, 16, 1, 1), [1, 1, 64, 64, 64, 1], 16, 20, (8, 8, 8, 8))[0]     # > one NVSwitch box
    # 2-D + time (the reference's Navier-Stokes trainer, experiment_navier_stokes.py:22-35): singleton-x plan
    assert supports(_Grid(1, 1, 2, 2, 1), [10, 1, 64, 64, 10], 40, 20, (4, 4, 4))[0]
    assert supports(_Grid(1, 1, 1, 1, 1), [1, 1, 64, 64, 1], 16, 20, (8, 8, 8))[0]
    assert not supports(_Grid(1, 1, 2, 2), [1, 1, 64, 64], 16, 20, (8, 8))[0]                        # 1-D + time
    assert not supports(_Grid(1, 1, 1, 1, 1, 1), [1, 1, 512, 64, 64, 1], 16, 20, (8, 8, 8, 8))[0]     # X > 256


def test_supports_refuses_lift_weights_over_the_kernel_budget():
    """The lift kernel keeps W1, b1 and the packed W2, b2 in 4096 floats of shared memory (kLiftMaxW)."""
    from dfno_b200.models.fused import LIFT_MAX_W, supports, wants
    g = _Grid(1, 1, 1, 1, 1, 1)
    assert 62 * 64 + 62 + 2 * (8 + 8) <= LIFT_MAX_W < 64 * 64 + 64 + 2 * (8 + 8)
    assert supports(g, [1, 1, 8, 8, 16, 64], 62, 8, (2, 2, 4, 4))[0]
    ok, why = supports(g, [1, 1, 8, 8, 16, 64], 64, 8, (2, 2, 4, 4))
    assert not ok and "4192" in why and "kLiftMaxW" in why, why
    kw = dict(device=torch.device("cuda"), dtype=torch.bfloat16)
    assert not wants((g, [1, 1, 8, 8, 16, 64], 64, 8, (2, 2, 4, 4)), kw, "auto")
    assert wants((g, [1, 1, 8, 8, 16, 64], 62, 8, (2, 2, 4, 4)), kw, "auto")
    with pytest.raises(ValueError, match="kLiftMaxW"):
        wants((g, [1, 1, 8, 8, 16, 64], 64, 8, (2, 2, 4, 4)), kw, "fused")


def test_dft_gemm_sizing_mirrors_the_launcher():
    """dft_gemm_min_smem: operator + 5 KB fixed + 8.5 KB row scratch of one warpgroup + two A stages of one K block
    (8 KB each with 64-row tiles, n_pad > 128; 16 KB with 128-row tiles), within 227 KB."""
    from dfno_b200.ops.gemm import DFT_GEMM_SMEM, dft_gemm_fits, dft_gemm_min_smem
    assert DFT_GEMM_SMEM == 227 * 1024
    assert dft_gemm_min_smem(192, 512) == 192 * 512 * 2 + 5120 + 8704 + 2 * 8192
    assert dft_gemm_min_smem(128, 512) == 128 * 512 * 2 + 5120 + 8704 + 2 * 16384
    assert dft_gemm_min_smem(190, 500) == dft_gemm_min_smem(192, 512)          # padded to [ceil16, ceil64]
    assert dft_gemm_fits(192, 512) and not dft_gemm_fits(200, 512) and not dft_gemm_fits(208, 512)
    assert dft_gemm_fits(256, 256) and not dft_gemm_fits(256, 400)
    assert not dft_gemm_fits(272, 64) and not dft_gemm_fits(16, 576)           # the launcher's n_pad / k_pad limits
    # the stage shapes the check uses are those of the operators the engine pads
    pl = EnginePlan(1, 1, 1, 8, 20, 256, 256, 64, (8, 40, 12, 10))
    pl.finish(1)
    ops = pl.operators()
    for st in pl.chain():
        if "N" in st:
            assert tuple(ops[st["op"]].shape) == (st["N"], st["K"]) == tuple(ops[st["op"] + "_adj"].shape), st["name"]


@pytest.mark.parametrize("in_shape,modes,accept,stage", [
    ([1, 1, 4, 256, 8, 1], (2, 48, 2, 2), True, None),      # G2 / G2_adj: 192 x 512 bf16 (n_pad 192) fits
    ([1, 1, 4, 256, 8, 1], (2, 50, 2, 2), False, "G2"),     # n_pad 208: 237 KiB
    ([1, 1, 4, 256, 8, 1], (2, 64, 2, 2), False, "G2"),     # 256 x 512 bf16 = 256 KB
    ([1, 1, 256, 4, 8, 1], (48, 2, 2, 2), True, None),      # the same on the x axis (G3)
    ([1, 1, 256, 4, 8, 1], (52, 2, 2, 2), False, "G3"),
    ([1, 1, 8, 8, 256, 1], (2, 2, 100, 2), False, "iG1a"),  # legacy pointwise route: iG1a is 256 x 400
])
def test_supports_refuses_operators_too_large_for_shared_memory(in_shape, modes, accept, stage):
    from dfno_b200.models.fused import supports, wants
    g = _Grid(1, 1, 1, 1, 1, 1)
    ok, why = supports(g, in_shape, 4, 4, modes)
    assert ok == accept, why
    if not accept:
        assert f"stage {stage}:" in why and "shared memory" in why, why
    kw = dict(device=torch.device("cuda"), dtype=torch.bfloat16)
    assert wants((g, in_shape, 4, 4, modes), kw, "auto") == accept


def test_memory_plan_sizes_shards_for_a_b200():
    from dfno_b200.models.fused import HBM_BUDGET, supports
    pl = EnginePlan(1, 1, 1, 20, 20, 128, 128, 128, (12, 12, 12, 10), world=1, rank=0)
    pl.finish(4)
    m = pl.memory_bytes(train=True)
    act = 20 * 128 ** 3 * 20 * 2                                        # one bf16 activation, 1.68 GB
    assert m["saved_activations"] >= 8 * act and m["adam_moments"] == 2 * m["parameters"] == 2 * m["gradients"]
    assert 20 * 2 ** 30 < m["total"] < 40 * 2 ** 30 and m["total"] == sum(v for k, v in m.items() if k != "total")
    assert pl.memory_bytes(train=False)["total"] < m["total"] / 2
    # batch 8 of the same field does not fit one GPU; spread over 8 it does
    ok, why = supports(_Grid(1, 1, 1, 1, 1, 1), [8, 1, 128, 128, 128, 1], 20, 20, (12, 12, 12, 10))
    assert not ok and ("GiB" in why or "2^31" in why)
    assert supports(_Grid(1, 1, 1, 8, 1, 1), [8, 1, 128, 128, 128, 1], 20, 20, (12, 12, 12, 10))[0]
    assert HBM_BUDGET < 80 * 2 ** 30                                    # an H100 holds 80 GB


def test_plan_routes_follow_the_shape_and_size_the_memory_check():
    """The plan's route flags for every shape of the GPU route matrix, and supports() checking the memory of the route
    that runs: at modes_z = 34 (2*KZ = 136 > 128) the round-1 dataflow also holds the channels-last head buffers and
    dhb, which take this problem over the budget; at modes_z = 32 the fused pointwise dataflow fits."""
    from dfno_b200.models.fused import HBM_BUDGET, _as_6d, supports
    from test_spectral_conv_gpu import ROUTES
    for name, in_shape, T, C, modes, routes in ROUTES:
        _, (B, Cin, X, Y, Z, Tin), modes6, _ = _as_6d([1] * len(in_shape), in_shape, modes)
        pl = EnginePlan(B, Cin, Tin, C, T, X, Y, Z, modes6)
        assert (pl.fused_pw, pl.tc_bypass) == (routes["fused_pw"], routes["tc"]), name
    g = _Grid(1, 1, 1, 1, 1, 1)
    ok, why = supports(g, [1, 1, 256, 256, 72, 1], 20, 20, (12, 12, 34, 10))
    assert not ok and "GiB per GPU" in why, why
    pl = EnginePlan(1, 1, 1, 20, 20, 256, 256, 72, (12, 12, 34, 10))
    pl.finish(4)
    assert not pl.fused_pw and pl.memory_bytes()["total"] > HBM_BUDGET                  # 77.4 GiB
    pl.fused_pw = True
    assert pl.memory_bytes()["total"] < HBM_BUDGET                                      # 68.9 GiB
    assert supports(g, [1, 1, 256, 256, 72, 1], 20, 20, (12, 12, 32, 10))[0]           # fused route, 67.0 GiB


def test_column_parts_address_the_same_elements():
    """``ScatterSpec.column_part``: pair ``j`` of a part lands exactly where pair ``j0 + j`` of the whole
    stage does (same peer after slicing the peer table, same element offset), for row-, column- and
    un-peered specs and for both ways a part can relate to the column radix."""
    from dfno_b200.ops.gemm import ScatterSpec
    rng = np.random.default_rng(0)
    specs = [
        (ScatterSpec(rows=[(5, 2), (3, 40)], cols=(16, 10, 0), peer=("col", 4), base_off=7), 16),      # 4 peers x 4 cols
        (ScatterSpec(rows=[(5, 2), (3, 40)], cols=(16, 10, 0), peer=("col", 16), base_off=0), 16),     # one peer
        (ScatterSpec(rows=[(4, 2), (6, 64), (2, 1000)], cols=(8, 8, 0), peer=("row", 1, 3), base_off=3), 8),
        (ScatterSpec(rows=[(7, 2)], cols=(4, 14, 200), peer=None, base_off=1), 12),                     # two-level columns
    ]
    for spec, npairs in specs:
        M = int(np.prod([r for r, _ in spec.rows]))
        for n in (1, 2, 4, 8):
            if npairs % n:
                continue
            try:
                parts = [(j0, n) + spec.column_part(j0, n) for j0 in range(0, npairs, n)]
            except ValueError:
                continue                                   # this split is not expressible; parts() tries the next size
            for j0, n_, part, p0, pn in parts:
                for row in rng.integers(0, M, size=6):
                    for j in range(n_):
                        peer, off = part.address(int(row), j)
                        assert (peer + p0, off) == spec.address(int(row), j0 + j), (spec.cols, spec.peer, j0, n_, row, j)
                        assert pn is None or peer < pn
    # a split that cannot be expressed is refused, not silently wrong
    with pytest.raises(ValueError):
        ScatterSpec(rows=[(4, 2)], cols=(6, 2, 0), peer=("col", 3)).column_part(0, 2)


def test_cost_model_reproduces_measured_dram_traffic():
    """The per-kernel byte counts of the traffic model against the DRAM bytes Nsight Compute recorded for the
    headline configuration on a B200 (126 MB L2), not re-recorded on an H100: the bytes a kernel must move belong
    to the dataflow; the tolerance (8 %, 12 % for spectral_out) covers that device's L2 hits."""
    pl = EnginePlan(1, 1, 1, 20, 20, 128, 128, 128, (12, 12, 12, 10), world=1, rank=0)
    pl.finish(4)
    pl.fused_pw = False                                    # round-1 dataflow, which these counts were recorded on
    cm = pl.cost_model()
    got = {n: b / 1e9 for n, _, b, _ in cm["stages"]}
    measured_gb = {"G1a": 2.27, "G1b": 0.91, "G2": 0.35, "iG1b": 0.96, "bypass fwd": 6.66, "bypass bwd": 8.35,
                   "spectral_mix fwd": 0.46, "spectral_mix bwd": 0.87, "adam": 12.3, "head fwd": 2.2, "head bwd": 4.2}
    for k, v in measured_gb.items():
        assert abs(got[k] - v) / v < 0.08, (k, got[k], v)
    assert 130e9 < cm["hbm_bytes"] < 175e9 and cm["nvlink_bytes"] == 0
    pl.fused_pw = True
    cm = pl.cost_model()                                   # round-2 dataflow: fused pointwise kernels
    got = {n: b / 1e9 for n, _, b, _ in cm["stages"]}
    measured_gb = {"G1a": 2.274, "G1b": 0.910, "G2": 0.354, "iG1b": 0.952, "spectral_out fwd": 5.624, "dpre_dw": 6.852,
                   "head fwd": 1.835, "head bwd": 3.483 + 0.168, "adam": 12.33, "lift fwd": 1.622, "lift bwd": 1.686}
    for k, v in measured_gb.items():
        assert abs(got[k] - v) / v < (0.12 if k == "spectral_out fwd" else 0.08), (k, got[k], v)
    assert 97.4e9 < cm["hbm_bytes"] < 136e9 and cm["nvlink_bytes"] == 0
    cf = pl.cost_model(front=True)                         # + spectral_in: Z1 (0.63 GB written and re-read) is gone
    assert abs((cm["hbm_bytes"] - cf["hbm_bytes"]) - 8 * 2 * pl.n_Z1 * 2) < 1e6
    assert cf["hbm_bytes"] < cm["hbm_bytes"] - 9.1e9
    p8 = EnginePlan(1, 1, 1, 20, 20, 128, 128, 128, (12, 12, 12, 10), world=8, rank=0)
    p8.finish(4)
    assert p8.cost_model(front=True)["nvlink_bytes"] == p8.cost_model()["nvlink_bytes"]
    c8 = p8.cost_model()
    per_chain = c8["nvlink_bytes"] / (2 * 4)
    assert abs(per_chain - 68.8e6) / 68.8e6 < 0.01        # bytes leaving a rank per spectral convolution


def test_fused_front_stage_plan_and_eligibility():
    """Host-side tile planner of csrc/spectral_in_sm90.cu (no GPU needed): the configurations the engine relies
    on are accepted with the expected tile shape, and the documented limits are refused with a reason (the engine
    then keeps the two separate GEMMs)."""
    from dfno_b200.ops import build
    C_ = build.load()

    def cfg(P, off, dstr, BC, X, Yl, T, Z, KZ, mt, n1=None, k1=None, n2=None, k2=None):
        c16 = lambda v: (v + 15) // 16 * 16
        c64 = lambda v: (v + 63) // 64 * 64
        a = (n1 or c16(2 * KZ), k1 or c64(Z), n2 or c16(2 * mt), k2 or c64(2 * T), P, off, dstr, BC, X, Yl, T, Z, KZ, mt)
        why = C_.spectral_in_check(*a)
        return why, (C_.spectral_in_config(*a) if not why else None)

    # headline, one rank: S1[bc, kz, kt, x, y, ri]; 4 positions per tile, 32-position store chunks, 2 consumer
    # warpgroups
    Y = 128
    why, c = cfg(1, 0, [Y * 2, 128 * Y * 2, 10 * 128 * Y * 2, 24 * 10 * 128 * Y * 2], 20, 128, 128, 20, 128, 24, 10)
    assert why == "" and c[:3] == [4, 32, 2] and c[3] >= 4
    # headline, rank 5 of 8, staged layout S1s[bc, kz', kt, r_src, x, y_loc, ri]: 16 local y -> 16-position chunks
    P, Yl, X = 8, 16, 128
    dstr = [Yl * 2, P * X * Yl * 2, 10 * P * X * Yl * 2, 3 * 10 * P * X * Yl * 2]
    why, c = cfg(P, 5 * X * Yl * 2, dstr, 20, X, Yl, 20, 128, 24, 10)
    assert why == "" and c[:2] == [4, 16]
    # BASELINE config 3 (256^3 x 16 t, width 32, 12 modes, 8 ranks): four K blocks per tile still fit
    why, c = cfg(8, 0, [32 * 2, 8 * 256 * 32 * 2, 8 * 8 * 256 * 32 * 2, 3 * 8 * 8 * 256 * 32 * 2], 64, 256, 32, 16, 256, 24, 8)
    assert why == "" and c[0] >= 1 and c[3] >= 2
    # two-phase default (60 x 60 x 64 x 30) on 4 ranks: 15 local y is not a multiple of 4 -> separate GEMMs
    why, _ = cfg(4, 0, [15 * 2 + 2, 8, 8, 8], 20, 60, 15, 30, 64, 24, 8)
    assert "multiple of 4" in why or "multiples of 8" in why
    # ... and on one rank (60 local y) it is accepted
    why, c = cfg(1, 0, [60 * 2, 60 * 60 * 2, 8 * 60 * 60 * 2, 24 * 8 * 60 * 60 * 2], 20, 60, 60, 30, 64, 24, 8)
    assert why == "" and c[0] == 4
    # documented limits
    assert "T <= 64" in cfg(1, 0, [256, 256, 256, 256], 4, 4, 32, 80, 64, 8, 4, k2=192)[0]
    assert "alignment" in cfg(2, 4, [256, 256, 256, 256], 4, 4, 32, 20, 64, 8, 4)[0]           # y offset not 16-byte aligned
    assert cfg(3, 0, [256, 256, 256, 256], 4, 4, 32, 20, 64, 8, 4)[0] != ""                    # KZ not divisible by the ranks


def _emulate_spectral_in(h, o1, o2, dst, dst_off, dstr, BC, X, Yl, T, Z, KZ, mt, P, Rp, Yc):
    """Float64 replay of csrc/spectral_in_sm90.cu with the kernel's own index arithmetic: tiles of Rp positions,
    D1 -> A2 transposition, D2 -> staging[kz][kt][y], one clipped box store per destination rank and chunk."""
    kzl, tpc, ncy = KZ // P, Yc // Rp, (Yl + Yc - 1) // Yc
    lines = h.reshape(BC * X, Yl * T, Z)
    for row in range(BC * X):
        bc, x = divmod(row, X)
        for cy in range(ncy):
            stg = torch.zeros(KZ * mt * Yc, 2, dtype=torch.float64)
            for tt in range(tpc):
                line0 = (cy * Yc + tt * Rp) * T
                tile = torch.zeros(Rp * T, Z, dtype=torch.float64)          # TMA box: rows past the tensor are zero
                n = max(0, min(Rp * T, Yl * T - line0))
                tile[:n] = lines[row, line0:line0 + n]
                D1 = tile @ o1.t()                                          # [m1 = p*T + t, 2 kz + ri]
                A2 = torch.zeros(KZ * Rp, 2 * T, dtype=torch.float64)
                for m1 in range(Rp * T):
                    p1, t1 = divmod(m1, T)
                    for kz in range(KZ):
                        A2[kz * Rp + p1, 2 * t1:2 * t1 + 2] = D1[m1, 2 * kz:2 * kz + 2]
                D2 = A2 @ o2.t()                                            # [m2 = kz*Rp + p, 2 kt + ri]
                for m2 in range(KZ * Rp):
                    kz2, p2 = divmod(m2, Rp)
                    for kt in range(mt):
                        stg[(kz2 * mt + kt) * Yc + tt * Rp + p2] = D2[m2, 2 * kt:2 * kt + 2]
            box = stg.view(KZ, mt, Yc, 2)
            ny = max(0, min(Yc, Yl - cy * Yc))                              # the store is clipped at the row end
            for j in range(P):
                for kzp in range(kzl):
                    for kt in range(mt):
                        base = dst_off + bc * dstr[3] + kzp * dstr[2] + kt * dstr[1] + x * dstr[0] + cy * Yc * 2
                        dst[j][base:base + 2 * ny] = box[j * kzl + kzp, kt, :ny].reshape(-1)


@pytest.mark.parametrize("P,staged,Yl,Rp,Yc", [(1, False, 8, 4, 8), (2, False, 8, 2, 4), (4, True, 12, 4, 8)])
def test_fused_front_stage_dataflow_emulated(P, staged, Yl, Rp, Yc):
    from dfno_b200.ops import operators as OPS
    torch.manual_seed(0)
    BC, X, T, Z, mz, mt, r = 2, 3, 6, 8, 2, 2, P - 1
    KZ, kzl, Y = 2 * mz, 2 * mz // P, Yl * P
    o1, o2 = OPS.fwd_real_to_complex(Z, mz), OPS.fwd_complex(T, mt, False)
    h = torch.randn(BC, X, Yl, T, Z, dtype=torch.float64)
    if staged:      # S1s[bc, kz', kt, r_src, x, y_loc, ri] on the owner of kz
        dstr, off, n = [Yl * 2, P * X * Yl * 2, mt * P * X * Yl * 2, kzl * mt * P * X * Yl * 2], r * X * Yl * 2, BC * kzl * mt * P * X * Yl * 2
    else:           # S1[bc, kz', kt, x, y, ri]
        dstr, off, n = [Y * 2, X * Y * 2, mt * X * Y * 2, kzl * mt * X * Y * 2], r * Yl * 2, BC * kzl * mt * X * Y * 2
    dst = [torch.full((n,), float("nan"), dtype=torch.float64) for _ in range(P)]
    _emulate_spectral_in(h, o1, o2, dst, off, dstr, BC, X, Yl, T, Z, KZ, mt, P, Rp, Yc)
    z1 = (h.reshape(-1, Z) @ o1.t()).view(BC * X * Yl, T, KZ, 2).permute(0, 2, 1, 3).reshape(-1, 2 * T)
    ref = (z1 @ o2.t()).view(BC, X, Yl, KZ, mt, 2).permute(0, 3, 4, 1, 2, 5)       # [bc, kz, kt, x, y, ri]
    for j in range(P):
        if staged:
            got = dst[j].view(BC, kzl, mt, P, X, Yl, 2)
            mine, rest = got[:, :, :, r], torch.cat([got[:, :, :, :r], got[:, :, :, r + 1:]], 3)
        else:
            got = dst[j].view(BC, kzl, mt, X, Y, 2)
            mine, rest = got[..., r * Yl:(r + 1) * Yl, :], torch.cat([got[..., :r * Yl, :], got[..., (r + 1) * Yl:, :]], -2)
        assert torch.allclose(mine, ref[:, j * kzl:(j + 1) * kzl], atol=1e-12)
        assert torch.isnan(rest).all()                  # nothing outside this rank's slice of the destination is written
