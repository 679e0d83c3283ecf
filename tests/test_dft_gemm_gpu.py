"""wgmma resident-operator GEMM vs a plain fp32 PyTorch reference (H100 only)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(M, K, N, lda=None, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lda = lda or K
    A = torch.randn(M, lda, device="cuda", generator=g).to(torch.bfloat16)
    B = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    return A, B, lda


@pytest.mark.parametrize("M,K,N,lda,fp32", [
    (1000, 128, 48, None, True),          # z-DFT shape, M tail
    (128 * 300 + 77, 128, 48, None, False),
    (647, 40, 20, 40, True),              # t-DFT: K tail inside one swizzle row, N tail
    (5000, 256, 48, None, False),         # y/x-DFT, 4 K blocks
    (3000, 48, 256, 48, False),           # inverse y/x-DFT, widest N
    (2048, 48, 128, 64, True),            # inverse z-DFT, padded pitch
    (129, 20, 40, 24, False),             # inverse t-DFT with padded (kt,ri) pitch
    (70000, 64, 16, None, False),         # many tiles per CTA
    (128 * 200 + 5, 512, 48, None, False),  # 256-sample complex axis: K chunks stream through the ring
    (4000, 384, 32, None, True),          # 192-sample axis, chunked (6 K blocks -> 3 per stage)
])
def test_rowmajor_matches_fp32_reference(M, K, N, lda, fp32):
    from dfno_b200.ops.gemm import gemm_rowmajor, pad_operator
    A, B, lda = _mk(M, K, N, lda)
    out = torch.full((M, N + 3), -7.0, device="cuda", dtype=torch.float32 if fp32 else torch.bfloat16)
    gemm_rowmajor(A, M, K, lda, pad_operator(B), N, out, N + 3)
    torch.cuda.synchronize()
    ref = A[:, :K].float() @ B.float().t()
    got = out[:, :N].float()
    tol = 2e-2 if not fp32 else 2e-3
    assert torch.allclose(got, ref, atol=tol, rtol=tol), float((got - ref).abs().max())
    assert (out[:, N:] == -7.0).all()     # nothing written outside the valid columns


def test_rowmajor_fused_add():
    from dfno_b200.ops.gemm import gemm_rowmajor, pad_operator
    M, K, N = 3333, 48, 128
    A, B, lda = _mk(M, K, N)
    add = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    gemm_rowmajor(A, M, K, lda, pad_operator(B), N, out, N, add=add, ld_add=N)
    ref = A.float() @ B.float().t() + add.float()
    assert torch.allclose(out.float(), ref, atol=3e-2, rtol=3e-2)


def _scatter_reference(ref, spec, npeers, size):
    M, N = ref.shape
    bufs = [torch.zeros(size, dtype=torch.float32) for _ in range(npeers)]
    refc = ref.cpu()
    for r in range(M):
        for j in range(N // 2):
            p, off = spec.address(r, j)
            bufs[p][off] = refc[r, 2 * j]
            bufs[p][off + 1] = refc[r, 2 * j + 1]
    return bufs


def test_pair_scatter_transposed_layout():
    """G1a-style: rows (line, t) x cols (kz, ri) -> out[line, kz, t, ri]."""
    from dfno_b200.ops.gemm import gemm_scatter, pad_operator, ScatterSpec
    lines, T, KZ = 37, 20, 24
    M, K, N = lines * T, 128, 2 * KZ
    A, B, lda = _mk(M, K, N)
    out = torch.zeros(lines * KZ * T * 2, device="cuda", dtype=torch.bfloat16)
    spec = ScatterSpec(rows=[(T, 2), (lines, KZ * T * 2)], cols=(KZ, T * 2, 0))
    gemm_scatter(A, M, K, lda, pad_operator(B), N, [out.data_ptr()], spec)
    ref = (A.float() @ B.float().t())
    want = ref.view(lines, T, KZ, 2).permute(0, 2, 1, 3).reshape(-1)
    assert torch.allclose(out.float(), want, atol=2e-2, rtol=2e-2)


def test_pair_scatter_peer_by_row_and_col():
    """Peer selection (all 'peers' are local buffers here): by a row digit and by the pair index."""
    from dfno_b200.ops.gemm import gemm_scatter, pad_operator, ScatterSpec
    R0, R1, R2 = 4, 6, 5           # row = (r2, r1, r0); r1 selects the peer (div 2 -> 3 peers)
    M, K, N = R0 * R1 * R2, 64, 20
    A, B, lda = _mk(M, K, N)
    size = 4096
    bufs = [torch.zeros(size, device="cuda", dtype=torch.bfloat16) for _ in range(3)]
    spec = ScatterSpec(rows=[(R0, 2), (R1, 400), (R2, 8)], cols=(10, 40, 0), peer=("row", 1, 2), base_off=16)
    gemm_scatter(A, M, K, lda, pad_operator(B), N, [b.data_ptr() for b in bufs], spec)
    ref = A.float() @ B.float().t()
    want = _scatter_reference(ref, spec, 3, size)
    for b, w in zip(bufs, want):
        assert torch.allclose(b.float().cpu(), w, atol=2e-2, rtol=2e-2)
    # by column pair: 10 pairs, div 5 -> 2 peers
    bufs = [torch.zeros(size, device="cuda", dtype=torch.bfloat16) for _ in range(2)]
    spec = ScatterSpec(rows=[(M, 12)], cols=(5, 2, 0), peer=("col", 5))
    gemm_scatter(A, M, K, lda, pad_operator(B), N, [b.data_ptr() for b in bufs], spec)
    want = _scatter_reference(ref, spec, 2, size)
    for b, w in zip(bufs, want):
        assert torch.allclose(b.float().cpu(), w, atol=2e-2, rtol=2e-2)
