"""spectral_in (csrc/spectral_in_sm90.cu): truncated z-DFT -> t-DFT chained through registers / shared memory, with the
pencil-transpose store, against an fp32 reference of the same two GEMMs (bf16 rounding of Z1 included)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops(Z, mz, T, mt, dev):
    from dfno_b200.ops import operators as OPS
    from dfno_b200.ops.gemm import pad_operator
    o1, o2 = OPS.fwd_real_to_complex(Z, mz), OPS.fwd_complex(T, mt, False)
    return o1, o2, pad_operator(o1, device=dev), pad_operator(o2, device=dev)


def _reference(h, o1, o2, BC, X, Yl, T, Z, KZ, mt):
    b = lambda v: v.to(torch.bfloat16).float()
    z1 = b(h.float().view(-1, Z) @ b(o1.to(h.device)).t())                      # [(bc,x,y,t), (kz,ri)]
    a2 = z1.view(BC * X * Yl, T, KZ, 2).permute(0, 2, 1, 3).reshape(-1, 2 * T)     # [(bc,x,y,kz), (t,ri)]
    s = a2 @ b(o2.to(h.device)).t()                                              # [(bc,x,y,kz), (kt,ri)]
    return s.view(BC, X, Yl, KZ, mt, 2).permute(0, 3, 4, 1, 2, 5).contiguous()     # [bc, kz, kt, x, y, ri]


@pytest.mark.parametrize("BC,X,Yl,T,Z,mz,mt,P", [
    (6, 5, 32, 20, 128, 12, 10, 1),       # the headline tile: Rp = 4, Yc = 32
    (8, 16, 128, 20, 128, 12, 10, 1),     # 512 chunks on 132 CTAs (H100 SXM): several chunks per CTA, both staging buffers
    (8, 64, 256, 4, 8, 2, 2, 1),          # tiny tiles (T = 4, Z = 8), 32 tiles per CTA: the issuing warps run far ahead of the epilogue
    (4, 3, 12, 30, 64, 12, 8, 1),         # T = 30 (two-phase), Yl < Yc = 16: the store is clipped at the row end
    (4, 1, 16, 32, 256, 16, 8, 1),        # 2-D + time (X = 1), Z = 256: four K blocks
    (5, 3, 16, 20, 128, 12, 10, 4),       # four destination "ranks" (buffers): one TMA store per rank and chunk
    (2, 2, 8, 64, 64, 4, 6, 2),           # T = 64: Rp = 2, two K blocks in the second GEMM
])
def test_spectral_in_matches_two_gemms(BC, X, Yl, T, Z, mz, mt, P):
    from dfno_b200.ops import build
    C_ = build.load()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    KZ = 2 * mz
    kzl = KZ // P
    o1, o2, p1, p2 = _ops(Z, mz, T, mt, dev)
    h = torch.randn(BC, X, Yl, T, Z, device=dev).to(torch.bfloat16)
    # destination: P buffers [BC, kzl, mt, X, Y >= Yl (16-byte row pitch), 2] with a guard band that must stay untouched
    Y = (Yl + 3) // 4 * 4
    dstr = [Y * 2, X * Y * 2, mt * X * Y * 2, kzl * mt * X * Y * 2]
    why = C_.spectral_in_check(p1.shape[0], p1.shape[1], p2.shape[0], p2.shape[1], P, 0, dstr, BC, X, Yl, T, Z, KZ, mt)
    assert why == "", why
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
        assert err <= 6e-3 * scale, (j, err, scale)


def test_spectral_in_strided_destination_with_offset():
    """Staged layout of an 8-rank run seen from source rank 3: [bc, kz', kt, r_src, x, y_loc, ri], written at r_src = 3."""
    from dfno_b200.ops import build
    C_ = build.load()
    dev = torch.device("cuda", 0)
    torch.manual_seed(1)
    BC, X, Yl, T, Z, mz, mt, P, r = 3, 4, 16, 20, 128, 12, 10, 8, 3
    KZ = 2 * mz
    kzl = KZ // P
    o1, o2, p1, p2 = _ops(Z, mz, T, mt, dev)
    h = torch.randn(BC, X, Yl, T, Z, device=dev).to(torch.bfloat16)
    dstr = [Yl * 2, P * X * Yl * 2, mt * P * X * Yl * 2, kzl * mt * P * X * Yl * 2]
    off = r * X * Yl * 2
    n = BC * kzl * mt * P * X * Yl * 2
    bufs = [torch.zeros(n, device=dev, dtype=torch.bfloat16) for _ in range(P)]
    C_.spectral_in(h, p1, p2, [b.data_ptr() for b in bufs], off, dstr, BC, X, Yl, T, Z, KZ, mt)
    torch.cuda.synchronize()
    ref = _reference(h, o1, o2, BC, X, Yl, T, Z, KZ, mt)
    scale = ref.abs().max().item()
    for j in range(P):
        got = bufs[j].float().view(BC, kzl, mt, P, X, Yl, 2)
        assert (got[:, :, :, r] - ref[:, j * kzl:(j + 1) * kzl]).abs().max().item() <= 6e-3 * scale
        mask = torch.ones(P, dtype=torch.bool); mask[r] = False
        assert got[:, :, :, mask].abs().max().item() == 0.0
