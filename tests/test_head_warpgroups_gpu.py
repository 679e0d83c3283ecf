"""The projection head's tile scheduling against float64 (H100 only): head_fwd at KR <= 48 deals its 128-position tiles
to 4 consumer warpgroups over an 8-stage TMA ring and runs MMA1 in two hidden halves; head_bwd2 deals them to 2.

The cases cover what that schedule makes new: tile counts that leave the warpgroups of a CTA uneven (and some with no
tile at all), rings that wrap many times, a last tile that is partial, two batches, a zero-padded layout, and the
weight-gradient sums over thousands of tiles, at the dout scale of a relative loss (3e-7) and at 1.  Tolerances and
the float64 reference are those of test_head_gpu.py."""
import pytest
import torch

from test_head_gpu import C_, DEV, H, check, failures, make_case, measure, operands, reference

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# total tiles as a function of the SM count n (the grid is min(tiles, n)): every CTA's share differs in its residue
# mod 4 (forward warpgroups) and mod 2 (backward warpgroups), and every S ends in a partial tile
TILES = {
    "5_tiles": lambda n: 5,                          # 5 CTAs of one tile: three forward warpgroups idle
    "n+1": lambda n: n + 1,                          # one CTA with two tiles
    "5n+3": lambda n: 5 * n + 3,                     # five or six tiles per CTA
    "26n+7": lambda n: 26 * n + 7,                   # 26 or 27 tiles per CTA: the 8-stage ring wraps 3 times
}


@pytest.mark.parametrize("dscale", [3e-7, 1.0])
@pytest.mark.parametrize("C", [8, 20, 40])
@pytest.mark.parametrize("tiles", list(TILES))
def test_head_tile_counts(tiles, C, dscale):
    nt = TILES[tiles](_sms())
    S = 128 * nt - 40                                # the last tile holds 88 positions
    case = make_case(1, C, 1, 1, 8, S // 8, seed=5000 + nt + C)
    m, bad = check(case, dscale)
    print(f"{tiles} ({nt} tiles) C={C} dout~{dscale:g}: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("C", [16, 20])
def test_head_two_batches_uneven(C):
    """B = 2, each batch ending in a partial tile, with 2 * 1204 tiles: the tiles of one CTA cross the batch boundary"""
    case = make_case(2, C, 7, 11, 40, 50, seed=6000 + C)
    m, bad = check(case, 3e-7)
    print(f"B=2 C={C}: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)


@pytest.mark.parametrize("dscale", [3e-7, 1.0])
@pytest.mark.parametrize("C", [8, 20])
def test_head_padded_layout(C, dscale):
    """A zero-padded activation (z 20 -> 24, t 10 -> 16, B = 2): pad rows store no output and add nothing to the
    weight gradients; their g is exactly 0"""
    B, X, Y, Z, T, Zp, Tp = 2, 9, 7, 20, 10, 24, 16
    case = make_case(B, C, X, Y, Zp, Tp, seed=7000 + C)    # h over the padded rows (pad rows hold nonzero values)
    S = case["S"]
    g_ = case["gen"]
    dy_pub = torch.randn(B, 1, X, Y, Z, T, device=DEV, generator=g_) * dscale
    dy_rows = torch.zeros(B, X, Y, Tp, Zp, device=DEV)
    dy_rows[:, :, :, :T, :Z] = dy_pub.squeeze(1).permute(0, 1, 2, 4, 3)
    ref = reference(case, dy_rows.reshape(-1))
    interior = torch.zeros(B, X, Y, Tp, Zp, dtype=torch.bool, device=DEV)
    interior[:, :, :, :T, :Z] = True
    interior = interior.reshape(-1)

    R, SR, lim = [Zp, Tp, B * X * Y], [T, 1, Z * T], [Z, T, B * X * Y]
    w3a, w3t = operands(case["W3"], case["b3"], C)
    out = torch.full((B, 1, X, Y, Z, T), float("nan"), device=DEV)
    C_().head_fwd(case["h"], w3a, case["w4b4"], out, B, C, S, R, SR, lim)
    g = torch.full((B * C, S), float("nan"), device=DEV, dtype=torch.bfloat16)
    grads = {"dW3": torch.zeros(H, C, device=DEV), "db3": torch.zeros(H, device=DEV),
             "dW4": torch.zeros(H, device=DEV), "db4": torch.zeros(1, device=DEV)}
    ws = torch.zeros(1, device=DEV, dtype=torch.int32)
    C_().head_bwd2(case["h"], w3a, w3t, case["w4b4"][:H].contiguous(), dy_pub.contiguous(), ws, g,
                   grads["dW3"], grads["db3"], grads["dW4"], grads["db4"], B, C, S, R, SR, lim)
    torch.cuda.synchronize()

    got = {"out": out.squeeze(1).permute(0, 1, 2, 4, 3).reshape(-1), "g": g, **grads}
    ref["out"] = ref["out"][interior]
    finite = {"out": bool(torch.isfinite(out).all()), "g": bool(torch.isfinite(g).all())}
    m = measure(got, ref)
    bad = failures(m, finite)
    pad_g = g.view(B, C, -1)[:, :, ~interior.view(B, -1)[0]]
    print(f"padded C={C} dout~{dscale:g}: " + " ".join(f"{k}={v:.2e}" for k, v in m.items()))
    assert not bad, (bad, m)
    assert bool((pad_g == 0).all())
