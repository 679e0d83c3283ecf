"""The inverse y-DFT (iG2) into T1 through the box-store epilogue against the pair scatter it replaced, on one GPU.

Both run the engine's own descriptor (EnginePlan.chain(): M, K, lda, column parts, peers), with the forward and the
adjoint chain's operator, for a rank r of a P-rank run whose P destination buffers are P tensors here.  Each row's
wgmma result does not depend on which rows share its tile, so the live T1 entries must be bitwise equal; the box
also writes the kt pad words of the rank's kz slab, as zeros, and nothing else: NaN guard bands before and after
every destination buffer and the other ranks' kz slabs stay untouched."""
import pytest
import torch

from dfno_b200.models.fused import EnginePlan
from dfno_b200.ops import build
from dfno_b200.ops.gemm import pad_operator

pytestmark = pytest.mark.gpu

GUARD = 4096          # bf16 elements of NaN before and after every destination buffer (16-byte multiple)


def _plan(P, r, B=1, C=4, X=8, Y=128, Z=64, T=20, modes=(4, 12, 12, 10), pad=None):
    pl = EnginePlan(B, 1, 1, C, T, X, Y, Z, modes, world=P, rank=r, pad=pad)
    pl.finish(1)
    return pl


def _ig2(pl):
    (st,) = [s for s in pl.chain(staged=pl.staged) if s["name"] == "iG2"]
    return st


def _run(pl, st, A, op, box):
    """iG2 of rank pl.rank into P NaN-filled destination buffers with guard bands; returns the padded buffers."""
    dev = A.device
    P = pl.world
    bufs = [torch.full((pl.n_T1 + 2 * GUARD,), float("nan"), device=dev, dtype=torch.bfloat16) for _ in range(P)]
    ptrs = [b[GUARD:].data_ptr() for b in bufs]
    if not box:
        st = {k: v for k, v in st.items() if k != "box"}
    for j0, n, spec, p0, pn in pl.parts(st):
        opp = pad_operator(op[2 * j0:2 * (j0 + n)], device=dev)
        build.load().dft_gemm(A, st["M"], st["K"], st["lda"], opp, 2 * n, pl.epi(st, j0, n, spec),
                              ptrs if pn is None else ptrs[p0:p0 + pn], None, 0, 0)
    torch.cuda.synchronize()
    return bufs


def _check(pl, adj):
    st = _ig2(pl)
    assert "box" in st, "this shape should take the box store"
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(7 + pl.rank)
    A = torch.randn(st["M"] * st["lda"], device=dev, generator=g).to(torch.bfloat16)
    op = pl.operators()[st["op"] + ("_adj" if adj else "")]
    box = _run(pl, st, A, op, True)
    ref = _run(pl, st, A, op, False)
    kz0 = pl.rank * pl.kzl
    for p in range(pl.world):
        b, s = box[p].view(torch.int16), ref[p].view(torch.int16)
        for band in (slice(0, GUARD), slice(GUARD + pl.n_T1, None)):
            assert torch.isnan(box[p][band].float()).all(), f"destination {p}: guard band written"
        t1b = b[GUARD:GUARD + pl.n_T1].view(pl.BC * pl.X, pl.Yl, pl.KZ, pl.mtp, 2)
        t1s = s[GUARD:GUARD + pl.n_T1].view(pl.BC * pl.X, pl.Yl, pl.KZ, pl.mtp, 2)
        mine = slice(kz0, kz0 + pl.kzl)
        assert torch.equal(t1b[:, :, mine, :pl.mt], t1s[:, :, mine, :pl.mt]), f"destination {p}: live entries differ"
        assert (t1b[:, :, mine, pl.mt:] == 0).all(), f"destination {p}: pad words not zero"
        others = torch.ones(pl.KZ, dtype=torch.bool, device=dev)
        others[mine] = False
        tb = box[p][GUARD:GUARD + pl.n_T1].view(pl.BC * pl.X, pl.Yl, pl.KZ, pl.mtp * 2)
        assert torch.isnan(tb[:, :, others].float()).all(), f"destination {p}: another rank's kz slab written"


CASES = {
    "headline-local-x8": dict(),
    "B2": dict(B=2),
    "mt7-groups-do-not-divide-kzl": dict(modes=(4, 12, 12, 7)),
    "Y256-column-parts": dict(Y=256),
    "padded": dict(pad=(4, 0, 8, 2)),
    "2d-plus-time": dict(X=1, modes=(1, 12, 12, 10)),
    "Y64-128-row-tiles": dict(Y=64, modes=(4, 8, 12, 10)),
}


@pytest.mark.parametrize("adj", [False, True], ids=["fwd", "adj"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_box_store_matches_pair_scatter_one_gpu(case, adj):
    _check(_plan(1, 0, **CASES[case]), adj)


@pytest.mark.parametrize("adj", [False, True], ids=["fwd", "adj"])
@pytest.mark.parametrize("P", [2, 3, 5, 7])
def test_box_store_matches_pair_scatter_ranks(P, adj):
    """P destination buffers; ragged kz storage at P = 5, 7 (24 modes) and ragged y at 3, 5, 7 (120 rows)"""
    for r in sorted({0, P - 1}):
        _check(_plan(P, r, Y=120), adj)


def test_box_store_column_parts_across_ranks():
    """Y = 256 on 2 ranks: each 128-pair launch is one whole destination buffer"""
    for r in (0, 1):
        pl = _plan(2, r, Y=256, X=4)
        assert [(p0, pn) for _, _, _, p0, pn in pl.parts(_ig2(pl))] == [(0, 1), (1, 1)]
        _check(pl, False)


def test_mt1_keeps_the_pair_scatter():
    pl = _plan(1, 0, modes=(4, 12, 12, 1))
    assert "box" not in _ig2(pl)
