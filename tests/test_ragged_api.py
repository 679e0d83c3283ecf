"""Ragged pencils on the fused engine, without a GPU: grids and kz mode counts that the pencil's GPU count does not
divide run on uniform per-rank storage whose entries past each rank's balanced share are dead.

Checked here: which configurations ``supports()`` takes, that the live rows and modes of the plan partition the global
axes exactly once, that the storage operators are the float64 DFT at the live entries' true indices and zero at the
dead ones, a float64 replay of the ragged chains (with the engine's own scatter tables) against the portable block,
the canonical round trip of weights and optimizer moments between ragged and even partitions, and ``tools/plan.py``."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dfno_b200.models.fused import EnginePlan, FusedDistributedFNO, pencil_storage, supports
from dfno_b200.ops import operators as OPS
from dfno_b200.parallel.decomposition import balanced_bounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWO_PHASE = dict(in_shape=[1, 1, 60, 60, 64, 1], nt=30, width=20, modes=(12, 12, 12, 8))
HEADLINE = dict(in_shape=[1, 1, 128, 128, 128, 1], nt=20, width=20, modes=(12, 12, 12, 10))


class _Grid:
    def __init__(self, shape):
        self.shape, self.dim = list(shape), len(shape)


def _pencil(P, nd=6):
    g = [1] * nd
    g[nd - 3] = P
    return _Grid(g)


def _supports(cfg, grid, **kw):
    return supports(grid, cfg["in_shape"], cfg["nt"], cfg["width"], cfg["modes"], **kw)


def _plans(cfg, P, blocks=1):
    B, Cin, X, Y, Z, Tin = cfg["in_shape"]
    out = []
    for r in range(P):
        pl = EnginePlan(B, Cin, Tin, cfg["width"], cfg["nt"], X, Y, Z, cfg["modes"], world=P, rank=r)
        pl.finish(blocks)
        out.append(pl)
    return out


# ------------------------------------------------------------------ eligibility
def test_supports_takes_the_two_phase_shape_on_eight_gpus():
    ok, why = _supports(TWO_PHASE, _pencil(8))
    assert ok, why
    pl = _plans(TWO_PHASE, 8)[0]
    assert (pl.Yl, pl.Y, pl.Yg) == (8, 64, 60) and (pl.kzl, pl.KZ, pl.KZg) == (3, 24, 24)


@pytest.mark.parametrize("P", [3, 5, 6, 7])
def test_supports_takes_the_headline_shape_on_any_gpu_count(P):
    ok, why = _supports(HEADLINE, _pencil(P))
    assert ok, why
    # folded onto the pencil from an x/z split: the same engine
    ok, why = _supports(HEADLINE, _Grid([1, 1, 1, 1, P, 1]))
    assert ok, why


def test_supports_takes_folded_and_time_partitioned_ragged_grids():
    for grid in ([1, 1, 2, 3, 1, 1], [1, 1, 1, 1, 1, 6], [1, 1, 1, 7, 1, 1]):
        ok, why = _supports(TWO_PHASE, _Grid(grid))
        assert ok, (grid, why)


def test_ragged_y_off_the_round2_route_is_refused_with_its_reason():
    # 2 * 2 * modes_z = 136 > 128: round-1 route, whose head has no padded layout for the dead rows
    cfg = dict(in_shape=[2, 1, 8, 60, 128, 1], nt=8, width=12, modes=(2, 2, 34, 3))
    ok, why = _supports(cfg, _pencil(8))
    assert not ok and "round-2 route" in why and "dead rows" in why, why
    # an even y axis on the same route runs (ragged kz has no such limit: 68 modes over 8 ranks)
    cfg["in_shape"][3] = 64
    ok, why = _supports(cfg, _pencil(8))
    assert ok, why
    pl = EnginePlan(2, 1, 1, 12, 8, 8, 64, 128, (2, 2, 34, 3), world=8, rank=7)
    assert pl.KZ != pl.KZg and not pl.fused_pw


def test_padding_the_pencil_axis_stays_refused():
    cfg = dict(TWO_PHASE)
    ok, why = _supports(cfg, _pencil(8), padding=(0, 4, 0, 0))
    assert not ok and "only one GPU can pad it" in why


@pytest.mark.parametrize("P", [1, 2, 4, 8])
def test_even_plans_store_exactly_the_shares(P):
    """An axis that P divides has no dead entries: storage is the share, as before ragged pencils existed."""
    for cfg in (HEADLINE, dict(in_shape=[1, 1, 8, 8, 8, 1], nt=4, width=4, modes=(2, 2, 4, 3))):
        for pl in _plans(cfg, P):
            assert (pl.Y, pl.KZ) == (pl.Yg, pl.KZg)
            assert pl.Yl == pl.Yli == pl.Yg // P and pl.y_off == pl.rank * pl.Yl
            assert pl.kzl == pl.kzl_live == pl.KZg // P and pl.kz_off == pl.rank * pl.kzl
            assert not pl.padded
    assert pencil_storage(60, 24, 4) == (15, 6)          # 15 rows: not rounded when 4 divides 60


# ------------------------------------------------------------------ live partition and operators
@pytest.mark.parametrize("P", [3, 5, 6, 7, 8])
@pytest.mark.parametrize("cfg", [TWO_PHASE, HEADLINE], ids=["two_phase", "headline"])
def test_live_rows_and_modes_partition_the_axes(cfg, P):
    plans = _plans(cfg, P)
    pl0 = plans[0]
    assert pl0.Yl % 4 == 0 or pl0.Y == pl0.Yg
    assert pl0.KZ % 4 == 0
    ys, kzs = [], []
    for r, pl in enumerate(plans):
        assert (pl.Yl, pl.kzl, pl.Y, pl.KZ) == (pl0.Yl, pl0.kzl, pl0.Y, pl0.KZ)       # uniform storage
        assert (pl.y_off, pl.y_off + pl.Yli) == balanced_bounds(pl.Yg, P, r)          # the input shard's rows
        assert (pl.kz_off, pl.kz_off + pl.kzl_live) == balanced_bounds(pl.KZg, P, r)
        assert pl.Yli <= pl.Yl and pl.kzl_live <= pl.kzl
        assert pl.padded == (pl.Yli != pl.Yl)
        ys += range(pl.y_off, pl.y_off + pl.Yli)
        kzs += range(pl.kz_off, pl.kz_off + pl.kzl_live)
    assert sorted(ys) == list(range(pl0.Yg)) and sorted(kzs) == list(range(pl0.KZg))
    ym, km = pl0.y_map(), pl0.kz_map()
    assert sorted(v for v in ym if v >= 0) == list(range(pl0.Yg)) and len(ym) == pl0.Y
    assert sorted(v for v in km if v >= 0) == list(range(pl0.KZg)) and len(km) == pl0.KZ
    for pl in plans:             # rank r's stored entries: its live ones in order, then dead ones
        r = pl.rank
        assert ym[r * pl.Yl:(r + 1) * pl.Yl] == list(range(pl.y_off, pl.y_off + pl.Yli)) + [-1] * (pl.Yl - pl.Yli)
        assert km[r * pl.kzl:(r + 1) * pl.kzl] == (list(range(pl.kz_off, pl.kz_off + pl.kzl_live))
                                                     + [-1] * (pl.kzl - pl.kzl_live))


@pytest.mark.parametrize("P", [3, 5, 6, 7, 8])
def test_storage_operators_are_the_dft_at_live_entries_and_zero_at_dead_ones(P):
    pl = _plans(HEADLINE, P)[0]
    ops = pl.operators()
    Y, Z = pl.Yg, pl.Z
    ky = OPS.retained_frequencies(Y, pl.my, True).numpy()
    kz = OPS.retained_frequencies(Z, pl.mz, True).numpy()
    G2, iG2, G1a, iG1a = (ops[k].numpy() for k in ("G2", "iG2", "G1a", "iG1a"))
    assert G2.shape == (2 * pl.KY, 2 * pl.Y) and iG2.shape == (2 * pl.Y, 2 * pl.KY)
    assert G1a.shape == (2 * pl.KZ, Z) and iG1a.shape == (Z, 2 * pl.KZ)
    for s, y in enumerate(pl.y_map()):
        fwd = G2[0::2, 2 * s] + 1j * G2[1::2, 2 * s]            # image of a real unit sample at stored row s
        inv = iG2[2 * s, 0::2] + 1j * iG2[2 * s + 1, 0::2]        # the stored row's output from a real unit mode
        if y < 0:
            assert not G2[:, 2 * s:2 * s + 2].any() and not iG2[2 * s:2 * s + 2].any()
        else:
            np.testing.assert_allclose(fwd, np.exp(-2j * np.pi * ky * y / Y), atol=1e-12)
            np.testing.assert_allclose(inv, np.exp(2j * np.pi * ky * y / Y) / Y, atol=1e-12)
    zz = np.arange(Z)
    for s, k in enumerate(pl.kz_map()):
        if k < 0:
            assert not G1a[2 * s:2 * s + 2].any() and not iG1a[:, 2 * s:2 * s + 2].any()
        else:
            np.testing.assert_allclose(G1a[2 * s] + 1j * G1a[2 * s + 1], np.exp(-2j * np.pi * kz[k] * zz / Z),
                                       atol=1e-12)
            np.testing.assert_allclose(iG1a[:, 2 * s], np.cos(2 * np.pi * kz[k] * zz / Z) / Z, atol=1e-12)
    # the adjoint chain's operators are the mirrors' transposes: zero at the same dead entries
    assert torch.equal(ops["G2_adj"], ops["iG2"].t()) and torch.equal(ops["iG1a_adj"], ops["G1a"].t())


@pytest.mark.parametrize("P,staged,T,Y,mz", [(3, False, 4, 12, 2), (3, True, 4, 12, 2), (6, False, 4, 20, 4),
                                             (5, True, 4, 16, 2), (3, False, 1, 16, 4), (7, True, 1, 16, 4)])
def test_ragged_stage_plan_reproduces_the_spectral_convolution(P, staged, T, Y, mz):
    """Every rank's ragged chain replayed in float64 with the engine's own scatter tables (the replay of
    tests/test_engine_plan.py) against the portable block, forward and adjoint; dead rows come out exactly zero."""
    from test_engine_plan import _run_chain
    import dfno_b200 as d
    B, C, X, Z = 2, 3, 8, 16
    modes = (2, 2, mz, 1 if T == 1 else 2)
    torch.manual_seed(0)
    _, P1, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    blk = d.DistributedFNOBlock(P1, [B, C, X, Y, Z, T], modes, dtype=torch.float64)
    Wg = torch.zeros(C, C, *blk.fft_shape[2:], dtype=torch.complex128)
    for w, sl in zip(blk.weights, blk.slices):
        Wg[sl] = w.detach()
    x = torch.randn(B, C, X, Y, Z, T, dtype=torch.float64)
    want = blk.spectral_forward(x).detach()
    plans = []
    for r in range(P):
        pl = EnginePlan(B, 1, 1, C, T, X, Y, Z, modes, world=P, rank=r)
        pl.finish(1)
        plans.append(pl)
    assert plans[0].Y != plans[0].Yg or plans[0].KZ != plans[0].KZg
    ops = plans[0].operators()

    def stored(t):               # engine layout [BC, X, Yl, T, Z] of this rank's live rows, dead rows zero
        h = t.permute(0, 1, 2, 3, 5, 4).contiguous().numpy()
        out = []
        for pl in plans:
            a = np.zeros((B, C, X, pl.Yl, T, Z))
            a[:, :, :, :pl.Yli] = h[:, :, :, pl.y_off:pl.y_off + pl.Yli]
            out.append(a.reshape(pl.BC, X, pl.Yl, T, Z))
        return out

    def gathered(outs):
        return torch.from_numpy(np.concatenate(
            [o.reshape(B, C, X, pl.Yl, T, Z)[:, :, :, :pl.Yli] for o, pl in zip(outs, plans)], axis=3)
        ).permute(0, 1, 2, 3, 5, 4)

    weights = []
    for pl in plans:             # native [i, o, (kzl, mt, KY, KX)], dead kz zero
        wn = torch.zeros(C, C, pl.kzl, pl.mt, pl.KY, pl.KX, dtype=torch.complex128)
        wn[:, :, :pl.kzl_live] = Wg[:, :, :, :, pl.kz_off:pl.kz_off + pl.kzl_live, :].permute(0, 1, 4, 5, 3, 2)
        weights.append(wn.reshape(C, C, pl.Q).numpy())
    outs = _run_chain(plans, ops, stored(x), weights, staged=staged)
    for o, pl in zip(outs, plans):
        assert not o.reshape(B, C, X, pl.Yl, T, Z)[:, :, :, pl.Yli:].any()       # dead rows stay exactly zero
    got = gathered(outs)
    assert torch.allclose(got, want, atol=1e-10), float((got - want).abs().max())

    g = torch.randn(B, C, X, Y, Z, T, dtype=torch.float64)
    wadj = [np.conj(np.transpose(w, (1, 0, 2))) for w in weights]
    gouts = _run_chain(plans, ops, stored(g), wadj, adj=True, staged=staged)
    for o, pl in zip(gouts, plans):
        assert not o.reshape(B, C, X, pl.Yl, T, Z)[:, :, :, pl.Yli:].any()
    lhs = float((got * g).sum())
    rhs = float((gathered(gouts) * x).sum())
    assert abs(lhs - rhs) < 1e-9 * max(1.0, abs(lhs)), (lhs, rhs)


# ------------------------------------------------------------------ canonical state
def _flat(meta, gen):
    n = max(off + int(np.prod(s)) for off, s in meta["segments"].values())
    return torch.randn(n, generator=gen, dtype=torch.float64).float()


def _metas(P, modes=(4, 4, 6, 3)):
    """theta descriptions of the P ranks of a small model with 2 * modes_z = 12 kz modes (ragged over 5 and 8)."""
    out = []
    for r in range(P):
        pl = EnginePlan(1, 1, 1, 4, 4, 8, 40, 16, modes, world=P, rank=r)
        pl.finish(2)
        out.append(pl.theta_meta())
    return out


def _to_canonical(metas, flats):
    parts = [FusedDistributedFNO.theta_to_canonical(f, m, include_pointwise=m["rank"] == 0)
             for m, f in zip(metas, flats)]
    return FusedDistributedFNO.merge_canonical(parts, metas[0])


def _from_canonical(state, metas):
    flats = []
    for m in metas:
        n = max(off + int(np.prod(s)) for off, s in m["segments"].values())
        t = torch.full((n,), float("nan"))
        FusedDistributedFNO.canonical_to_theta(state, m, t)
        flats.append(t)
    return flats


def test_canonical_round_trip_ragged_even_ragged():
    """Weights (and FusedAdam moments, which share theta's layout) go ragged (5 ranks) -> canonical -> even (4, 2, 1
    ranks) -> canonical -> ragged (5 and 8 ranks) unchanged; dead kz modes load as zeros."""
    gen = torch.Generator().manual_seed(0)
    rag5 = _metas(5)
    assert rag5[0]["kzl"] != rag5[0]["kzl_live"] or rag5[-1]["kzl"] != rag5[-1]["kzl_live"]
    for kind in ("theta", "adam_m"):
        flats = []
        for m in rag5:
            f = _flat(m, gen)
            if kind == "adam_m":
                f = f.abs()
            flats.append(f)
        state = _to_canonical(rag5, flats)
        assert state["blocks.0.spectral"].shape[4] == 12
        for P in (4, 2, 1):
            even = _metas(P)
            assert all(m["kzl"] == m["kzl_live"] for m in even)
            back = _to_canonical(even, _from_canonical(state, even))
            assert sorted(back) == sorted(state)
            for k in state:
                assert torch.equal(back[k], state[k]), (P, k)
        for P in (5, 8):
            rag = _metas(P)
            loaded = _from_canonical(state, rag)
            for m, f in zip(rag, loaded):
                for name, (off, shape) in m["segments"].items():
                    assert not torch.isnan(f[off:off + int(np.prod(shape))]).any(), name
                    if name.endswith(".spectral"):
                        w = f[off:off + int(np.prod(shape))].view(shape[0], shape[1], m["kzl"], -1)
                        assert not w[:, :, m["kzl_live"]:].any()
            back = _to_canonical(rag, loaded)
            for k in state:
                assert torch.equal(back[k], state[k]), (P, k)
        # the ragged source itself: live entries reproduced bit for bit
        again = _from_canonical(state, rag5)
        for m, f0, f1 in zip(rag5, flats, again):
            for name, (off, shape) in m["segments"].items():
                a, b = f0[off:off + int(np.prod(shape))], f1[off:off + int(np.prod(shape))]
                if name.endswith(".spectral"):
                    a = a.view(shape[0], shape[1], m["kzl"], -1)[:, :, :m["kzl_live"]]
                    b = b.view(shape[0], shape[1], m["kzl"], -1)[:, :, :m["kzl_live"]]
                if name.endswith(".spectral") or m["rank"] == 0:
                    assert torch.equal(a, b), name


# ------------------------------------------------------------------ tools/plan.py
def test_plan_tool_reports_the_two_phase_shape_on_eight_gpus():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "plan.py"), "--shape", "60", "60", "64", "30",
                          "--width", "20", "--modes", "12", "12", "12", "8", "--gpus", "8"],
                         capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert out.returncode == 0, out.stderr
    assert "fused engine: yes" in out.stdout
    assert "64 in all for 60 live (storage / live 1.0667, dead fraction 6.25%)" in out.stdout, out.stdout
