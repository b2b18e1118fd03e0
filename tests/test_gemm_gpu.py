"""GPU: the strided fp32 GEMM of the PointWiseMLP path -- both implementations, the wgmma 3xTF32 kernel and the
fp32 FMA kernel -- against a float64 torch product (floating point: tolerance 1e-5 relative to the result's max
magnitude, written here)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

ALGOS = [0, 1, 2]  # CL3D_GEMM_AUTO, CL3D_GEMM_FFMA, CL3D_GEMM_TC3X


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("M,N,K", [(1000, 144, 75), (4096, 72, 144), (33, 5, 7), (257, 130, 40), (300, 300, 36),
                                   (32768, 144, 80)])
def test_sgemm_row_major_times_transposed_weights(cuda, M, N, K, algo):
    from closerlook3d_b200 import ops
    g = torch.Generator().manual_seed(M + N + K)
    lda = K + 5
    a = torch.randn(M, lda, generator=g).to(cuda)
    w = torch.randn(N, K, generator=g).to(cuda)
    out = ops.sgemm(a, lda, 1, w, 1, K, M, N, K, algo=algo)  # out[m][n] = sum_k a[m][k] w[n][k]
    ref = (a[:, :K].double() @ w.double().t()).float()
    assert float((out[:, :N] - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("algo", ALGOS)
def test_sgemm_plain_and_ldc(cuda, algo):
    from closerlook3d_b200 import ops
    g = torch.Generator().manual_seed(3)
    M, N, K, ldc = 777, 72, 144, 80
    a = torch.randn(M, K, generator=g).to(cuda)
    b = torch.randn(K, N + 3, generator=g).to(cuda)  # only the first N columns are used
    out = ops.sgemm(a, K, 1, b, N + 3, 1, M, N, K, ldc=ldc, algo=algo)
    ref = (a.double() @ b[:, :N].double()).float()
    assert out.shape == (M, ldc)
    assert float((out[:, :N] - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("splitk", [1, 7, 64])
def test_sgemm_transposed_a_splitk(cuda, splitk, algo):
    """splitk = 1 with the tensor-core kernel: one CTA reduces all k = 5000 (accumulator promotion keeps it exact
    to fp32 level)"""
    from closerlook3d_b200 import ops
    g = torch.Generator().manual_seed(11)
    P, M, N = 5000, 144, 75  # out (M x N) = ga^T (M x P) @ f (P x N): the weight-gradient shape
    ga = torch.randn(P, M, generator=g).to(cuda)
    f = torch.randn(P, N + 5, generator=g).to(cuda)
    out = ops.sgemm(ga, 1, M, f, N + 5, 1, M, N, P, splitk=splitk, algo=algo)
    ref = (ga.double().t() @ f[:, :N].double()).float()
    assert float((out[:, :N] - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


def test_sgemm_tc_aligned_weight_gradient(cuda):
    """the shapes of the c2 backward: d/dW (144 x 80) over 32768 points, split-K, float4 staging on both sides"""
    from closerlook3d_b200 import ops
    g = torch.Generator().manual_seed(5)
    P, M, N = 32768, 144, 80
    ga = torch.randn(P, M, generator=g).to(cuda)
    f = torch.randn(P, N, generator=g).to(cuda)
    ref = (ga.double().t() @ f.double()).float()
    for algo in (1, 2):
        out = ops.sgemm(ga, 1, M, f, N, 1, M, N, P, splitk=128, algo=algo)
        assert float((out[:, :N] - ref).abs().max()) <= 1e-5 * float(ref.abs().max()), algo


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("M,N,K", [(512, 144, 150), (132, 72, 16), (4096, 80, 37)])
def test_sgemm_row_contiguous_operands(cuda, M, N, K, algo):
    """both operands stored k-major-outer (rows are the unit stride, 16-byte aligned): the tensor-core kernel
    stages them with float4 loads along the rows and a register transpose; K = 150 / 37 exercise the k tail"""
    from closerlook3d_b200 import ops
    g = torch.Generator().manual_seed(M + K)
    at = torch.randn(K, M, generator=g).to(cuda)      # A[m][k] = at[k][m]
    b = torch.randn(K, N, generator=g).to(cuda)       # B[k][n]
    out = ops.sgemm(at, 1, M, b, N, 1, M, N, K, algo=algo)
    ref = (at.double().t() @ b.double()).float()
    assert float((out[:, :N] - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))
