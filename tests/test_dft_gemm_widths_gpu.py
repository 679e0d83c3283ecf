"""dft_gemm per operator width (csrc/dft_gemm_sm90.cu is instantiated for every n_pad from 16 to 256) against the fp32
reference, with test_dft_gemm_gpu.py's tolerances: every width, odd N, short and chunked K, M tails, and every
epilogue (staged and direct row-major bf16, fp32 out, fused add, pair scatter with row / column peers into several
buffers, column parts, projection head).  H100 only."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = list(range(16, 257, 16)) + [20, 40, 250]


def _mk(M, K, N, lda=None, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lda = lda or K
    A = torch.randn(M, lda, device="cuda", generator=g).to(torch.bfloat16)
    B = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    return A, B, lda


def _ref(A, K, B):
    return A[:, :K].float() @ B.float().t()


@pytest.mark.parametrize("N", WIDTHS)
@pytest.mark.parametrize("fp32", [False, True])
def test_rowmajor_every_width(N, fp32):
    """aligned rows (staged when N divides 256, else direct vector stores) and unaligned rows (scalar stores)"""
    from dfno_b200.ops.gemm import gemm_rowmajor, pad_operator
    M, K = 128 * 23 + 45, 64
    A, B, lda = _mk(M, K, N, seed=N)
    Bp = pad_operator(B)
    ref = _ref(A, K, B)
    tol = 2e-3 if fp32 else 2e-2
    dt = torch.float32 if fp32 else torch.bfloat16
    for ldc in ((N + 7) // 8 * 8, N + 3):
        out = torch.full((M, ldc), -7.0, device="cuda", dtype=dt)
        gemm_rowmajor(A, M, K, lda, Bp, N, out, ldc)
        got = out[:, :N].float()
        assert torch.allclose(got, ref, atol=tol, rtol=tol), (ldc, float((got - ref).abs().max()))
        assert (out[:, N:] == -7.0).all(), ldc


@pytest.mark.parametrize("K,N", [(K, N) for K in (20, 40, 48, 256, 512) for N in (48, 128, 256)
                                 if (K, N) != (512, 256)])      # a 256 x 512 operator does not fit shared memory
def test_rowmajor_k_lengths(K, N):
    """K tails inside one block, whole blocks, and K = 512 (chunked through the ring); M tail of 5 rows"""
    from dfno_b200.ops.gemm import gemm_rowmajor, pad_operator
    M = 64 * 97 + 5
    A, B, lda = _mk(M, K, N, lda=(K + 7) // 8 * 8, seed=K + N)
    out = torch.full((M, N), -7.0, device="cuda", dtype=torch.float32)
    gemm_rowmajor(A, M, K, lda, pad_operator(B), N, out, N)
    ref = _ref(A, K, B)
    assert torch.allclose(out, ref, atol=2e-3, rtol=2e-3), float((out - ref).abs().max())


@pytest.mark.parametrize("N,ldc,fp32", [(128, 128, False), (256, 256, False), (64, 64, True), (48, 48, False),
                                        (48, 56, True), (40, 40, False)])
def test_rowmajor_fused_add(N, ldc, fp32):
    """staged (N = 64, 128, 256) and direct (N = 40, 48) stores with the bf16 tensor added"""
    from dfno_b200.ops.gemm import gemm_rowmajor, pad_operator
    M, K = 3333, 48
    A, B, lda = _mk(M, K, N, seed=7)
    add = torch.randn(M, ldc, device="cuda").to(torch.bfloat16)
    out = torch.full((M, ldc), -7.0, device="cuda", dtype=torch.float32 if fp32 else torch.bfloat16)
    gemm_rowmajor(A, M, K, lda, pad_operator(B), N, out, ldc, add=add, ld_add=ldc)
    ref = _ref(A, K, B) + add[:, :N].float()
    assert torch.allclose(out[:, :N].float(), ref, atol=3e-2, rtol=3e-2)
    assert (out[:, N:] == -7.0).all()


def _addresses(spec, M, npairs):
    """vectorised ScatterSpec.address: (peer, offset) of pair j of row r as [M, npairs] arrays"""
    r = np.arange(M, dtype=np.int64)[:, None].repeat(npairs, 1)
    j = np.arange(npairs, dtype=np.int64)[None, :].repeat(M, 0)
    off, peer = np.full_like(r, spec.base_off), np.zeros_like(r)
    for l, (radix, stride) in enumerate(spec.rows):
        last = l == len(spec.rows) - 1
        d = r if last else r % radix
        r = np.zeros_like(r) if last else r // radix
        if spec.peer is not None and spec.peer[0] == "row" and spec.peer[1] == l:
            peer, d = d // spec.peer[2], d % spec.peer[2]
        off = off + d * stride
    if spec.peer is not None and spec.peer[0] == "col":
        peer, j = j // spec.peer[1], j % spec.peer[1]
    J0, SJ0, SJ1 = spec.cols
    return peer, off + (j % J0) * SJ0 + (j // J0) * SJ1


def _check_scatter(A, K, B, N, spec, npeers, size):
    from dfno_b200.ops.gemm import gemm_scatter, pad_operator
    M = A.shape[0]
    bufs = [torch.zeros(size, device="cuda", dtype=torch.bfloat16) for _ in range(npeers)]
    gemm_scatter(A, M, K, A.shape[1], pad_operator(B), N, [b.data_ptr() for b in bufs], spec)
    ref = _ref(A, K, B).cpu().numpy()
    peer, off = _addresses(spec, M, N // 2)
    want = [np.zeros(size, dtype=np.float32) for _ in range(npeers)]
    for p in range(npeers):
        m = peer == p
        want[p][off[m]] = ref[:, 0::2][m]
        want[p][off[m] + 1] = ref[:, 1::2][m]
    for b, w in zip(bufs, want):
        got = b.float().cpu()
        assert torch.allclose(got, torch.from_numpy(w), atol=2e-2, rtol=2e-2), float((got - torch.from_numpy(w)).abs().max())


@pytest.mark.parametrize("N", [n for n in WIDTHS if n % 2 == 0])
def test_pair_scatter_every_width(N):
    """transposed layout (consecutive rows are adjacent pairs, as in G2 / iG2 / iG1b), M tail"""
    from dfno_b200.ops.gemm import ScatterSpec
    R0 = 24
    M, K = R0 * 23 + 7, 48                       # the last row group is partial
    A, B, _ = _mk(M, K, N, seed=N + 1)
    npairs, groups = N // 2, (M + R0 - 1) // R0
    spec = ScatterSpec(rows=[(R0, 2), (groups, npairs * R0 * 2)], cols=(npairs, R0 * 2, 0))
    _check_scatter(A, K, B, N, spec, 1, groups * npairs * R0 * 2)


@pytest.mark.parametrize("N", [48, 128, 256])
def test_pair_scatter_row_peers(N):
    """a row digit selects one of 4 destination buffers (the t-DFT / pencil transpose layout)"""
    from dfno_b200.ops.gemm import ScatterSpec
    R0, R1, R2 = 10, 8, 29                        # row = (r2, r1, r0); r1 // 2 selects the peer
    M, K = R0 * R1 * R2, 256
    A, B, _ = _mk(M, K, N, seed=3)
    npairs = N // 2
    spec = ScatterSpec(rows=[(R0, 2), (R1, R0 * 2 * npairs), (R2, R0 * 2 * npairs * 2)], cols=(npairs, R0 * 2, 0),
                       peer=("row", 1, 2), base_off=6)
    _check_scatter(A, K, B, N, spec, 4, R2 * 2 * R0 * 2 * npairs + 64)


@pytest.mark.parametrize("N,div", [(256, 16), (48, 12), (128, 32)])
def test_pair_scatter_column_peers(N, div):
    """the pair index selects the destination buffer (iG2's pencil transpose), up to 8 buffers"""
    from dfno_b200.ops.gemm import ScatterSpec
    M, K = 64 * 41 + 9, 48
    A, B, _ = _mk(M, K, N, seed=4)
    npeers = N // 2 // div
    spec = ScatterSpec(rows=[(10, 2), (M, 20 * div)], cols=(div, 20, 0), peer=("col", div))
    _check_scatter(A, K, B, N, spec, npeers, ((M + 9) // 10) * 20 * div + 64)


def test_pair_scatter_column_parts():
    """a 512-wide stage issued as two 256-wide column parts lands where the whole stage would"""
    from dfno_b200.ops.gemm import ScatterSpec, gemm_scatter, pad_operator
    M, K, N = 64 * 30 + 3, 48, 512
    A, B, _ = _mk(M, K, N, seed=5)
    spec = ScatterSpec(rows=[(10, 2), (M, 10 * 2 * 256)], cols=(256, 20, 0))
    size = ((M + 9) // 10) * 10 * 2 * 256
    out = torch.zeros(size, device="cuda", dtype=torch.bfloat16)
    for j0 in (0, 128):
        part, p0, pn = spec.column_part(j0, 128)
        gemm_scatter(A, M, K, K, pad_operator(B[2 * j0:2 * (j0 + 128)]), 256, [out.data_ptr()], part)
    ref = _ref(A, K, B).cpu().numpy()
    peer, off = _addresses(spec, M, N // 2)
    want = np.zeros(size, dtype=np.float32)
    want[off] = ref[:, 0::2]
    want[off + 1] = ref[:, 1::2]
    assert torch.allclose(out.float().cpu(), torch.from_numpy(want), atol=2e-2, rtol=2e-2)


@pytest.mark.parametrize("N", [16, 20, 48, 128, 250])
def test_projection_head(N):
    """EPI_HEAD: out[row] = b4 + sum_j W4[j] gelu(acc[row, j] + b3[j]), fp32, against float64 erf-GELU"""
    from dfno_b200.ops import build
    from dfno_b200.ops.gemm import pad_operator
    M, K = 128 * 19 + 100, 20
    A, B, lda = _mk(M, K, N, lda=24, seed=N + 2)
    g = torch.Generator(device="cuda").manual_seed(9)
    v0 = torch.randn(N, device="cuda", generator=g)
    v1 = torch.randn(N + 1, device="cuda", generator=g) / N ** 0.5
    out = torch.full((M + 5,), -7.0, device="cuda", dtype=torch.float32)
    epi = [2, 1, 0, 1, M, 1, 1, 1, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1, 0]
    build.load().dft_gemm(A, M, K, lda, pad_operator(B), N, epi, [out.data_ptr()], None, 0, 0, v0, v1, 0.0)
    pre = _ref(A, K, B).double() + v0.double()
    ref = torch.nn.functional.gelu(pre) @ v1[:N].double() + v1[N].double()
    assert torch.allclose(out[:M].double(), ref, atol=1e-3, rtol=1e-3), float((out[:M].double() - ref).abs().max())
    assert (out[M:] == -7.0).all()
