"""spectral_in at every operator width it is compiled for: one kernel instantiation per (n1_pad, MMA2 width class),
n1_pad = ceil16(2 KZ) = 16 .. 128 and N2 = ceil16(2 mt) = 16 .. 80 or 128 (n2_pad 96 / 112), each against the fp32
two-GEMM reference of test_spectral_in_gpu.py, plus the planner's corner cases: a store clipped at the row end, eight
destination buffers with 16 local y, and a TMA ring that wraps many times."""
import pytest
import torch

from test_spectral_in_gpu import _ops, _reference

pytestmark = pytest.mark.gpu

MZ_FOR_N1 = {16: 2, 32: 6, 48: 10, 64: 14, 80: 18, 96: 22, 112: 26, 128: 30}     # n1_pad = ceil16(4 mz)
MT_T_FOR_N2 = {16: (8, 16), 32: (16, 32), 48: (24, 48), 64: (32, 64), 80: (33, 64), 128: (48, 64)}


def _check(BC, X, Yl, T, Z, mz, mt, P, expect=None):
    from dfno_b200.ops import build
    C_ = build.load()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    KZ = 2 * mz
    kzl = KZ // P
    o1, o2, p1, p2 = _ops(Z, mz, T, mt, dev)
    h = torch.randn(BC, X, Yl, T, Z, device=dev).to(torch.bfloat16)
    Y = (Yl + 3) // 4 * 4
    dstr = [Y * 2, X * Y * 2, mt * X * Y * 2, kzl * mt * X * Y * 2]
    a = (p1.shape[0], p1.shape[1], p2.shape[0], p2.shape[1], P, 0, dstr, BC, X, Yl, T, Z, KZ, mt)
    why = C_.spectral_in_check(*a)
    assert why == "", why
    cfg = C_.spectral_in_config(*a)
    if expect:
        for k, v in expect.items():
            assert cfg[k] == v, (cfg, expect)
    n = BC * kzl * mt * X * Y * 2
    bufs = [torch.full((n + 64,), 7.0, device=dev, dtype=torch.bfloat16) for _ in range(P)]
    C_.spectral_in(h, p1, p2, [b.data_ptr() for b in bufs], 0, dstr, BC, X, Yl, T, Z, KZ, mt)
    torch.cuda.synchronize()
    ref = _reference(h, o1, o2, BC, X, Yl, T, Z, KZ, mt)
    scale = ref.abs().max().item()
    for j in range(P):
        got = bufs[j][:n].float().view(BC, kzl, mt, X, Y, 2)
        assert torch.all(bufs[j][n:] == 7.0) and torch.all(got[..., Yl:, :] == 7.0), "wrote past the destination"
        err = (got[..., :Yl, :] - ref[:, j * kzl:(j + 1) * kzl]).abs().max().item()
        assert err <= 6e-3 * scale, (j, err, scale, cfg)


@pytest.mark.parametrize("n1", sorted(MZ_FOR_N1))
@pytest.mark.parametrize("n2", sorted(MT_T_FOR_N2))
def test_spectral_in_every_width_class(n1, n2):
    mz = MZ_FOR_N1[n1]
    mt, T = MT_T_FOR_N2[n2]
    _check(2, 3, 8, T, 64, mz, mt, 1)


@pytest.mark.parametrize("BC,X,Yl,T,Z,mz,mt,P,expect", [
    (3, 2, 20, 20, 128, 12, 10, 1, {1: 32}),       # Yl < Yc = 32: the 128-byte swizzled box is clipped at the row end
    (2, 3, 16, 20, 128, 12, 10, 8, {0: 4, 1: 16}),  # eight destination buffers, 16 local y (64-byte swizzled rows)
    (2, 2, 8, 20, 128, 12, 10, 2, {1: 8}),          # 32-byte swizzle
    (2, 2, 4, 20, 128, 12, 10, 2, {1: 4}),          # 16-byte rows: no swizzle
    (4, 64, 128, 20, 128, 12, 10, 1, {2: 2}),       # 8192 tiles, about 62 per CTA: the ring wraps about ten times
])
def test_spectral_in_planner_corners(BC, X, Yl, T, Z, mz, mt, P, expect):
    _check(BC, X, Yl, T, Z, mz, mt, P, expect)
