"""wgmma GEMM (dense layers of MultiVAE / NeuMF) vs a bf16-rounded fp64 matmul."""
import pytest
import torch

from elliot_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("M,N,K", [(512, 600, 26744), (512, 400, 600), (26744, 600, 512), (130, 70, 200), (1, 1, 8),
                                  (257, 129, 1000), (600, 200, 512)])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_gemm_matches_bf16_matmul(M, N, K, act):
    if act and M * N * K > 3e9:
        pytest.skip("activation variants on the small shapes only")
    g = torch.Generator(device=DEV); g.manual_seed(M + N + K)
    A = torch.randn(M, K, device=DEV, generator=g) / K ** 0.5
    B = torch.randn(N, K, device=DEV, generator=g)
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    Ab, Bb = ops.to_bf16(A), ops.to_bf16(B)
    C = ops.gemm_bf16_tn(Ab, Bb, M, N, K, bias=bias, alpha=0.5, act=act)
    ref = 0.5 * (A.bfloat16().double() @ B.bfloat16().double().T) + bias.double()
    if act == 1: ref = torch.tanh(ref)
    if act == 2: ref = torch.relu(ref)
    assert (C.double() - ref).abs().max().item() < 2e-4      # fp32 accumulation of <= 26744 products


def test_convert_transpose_roundtrip():
    g = torch.Generator(device=DEV); g.manual_seed(0)
    X = torch.randn(301, 77, device=DEV, generator=g)
    a = ops.to_bf16(X); t = ops.to_bf16(X, transpose=True)
    assert a.shape == (301, 80) and t.shape == (77, 304)
    assert torch.equal(a[:, :77], X.bfloat16()) and not a[:, 77:].any()
    assert torch.equal(t[:, :301], X.bfloat16().T) and not t[:, 301:].any()
    # GEMM on transposed operands: X^T X
    C = ops.gemm_bf16_tn(t, t, 77, 77, 301)
    ref = X.bfloat16().double().T @ X.bfloat16().double()
    assert (C.double() - ref).abs().max().item() < 1e-3


@pytest.mark.parametrize("M,N,K", [(600, 200, 512), (26744, 600, 512), (512, 600, 26744), (130, 70, 200), (64, 128, 1 << 20), (8, 16, 8),
                                  (257, 129, 1000)])
@pytest.mark.parametrize("a_mn,b_mn", [(True, True), (True, False), (False, True)])
def test_gemm_with_rows_are_k_operands(M, N, K, a_mn, b_mn):
    """An operand stored [K][M] (rows are K) is read through MN-major descriptors: same result as the K-major GEMM on the
    transposed copy — which is what the backward passes used to build."""
    if M * N * K > 2e10:
        pytest.skip("too large")
    g = torch.Generator(device=DEV); g.manual_seed(M + 3 * N + K)
    A = torch.randn(M, K, device=DEV, generator=g) / K ** 0.5
    B = torch.randn(N, K, device=DEV, generator=g)
    Aop = ops.to_bf16(A.T.contiguous()) if a_mn else ops.to_bf16(A)          # [K][M(+pad)] or [M][K(+pad)]
    Bop = ops.to_bf16(B.T.contiguous()) if b_mn else ops.to_bf16(B)
    C = ops.gemm_bf16(Aop, Bop, M, N, K, a_rows_are_k=a_mn, b_rows_are_k=b_mn, alpha=0.5)
    ref = 0.5 * (A.bfloat16().double() @ B.bfloat16().double().T)
    tol = 2e-4 if K < 100000 else 2e-3                                       # split-K atomics over 1M products
    assert (C.double() - ref).abs().max().item() < tol


@pytest.mark.parametrize("M,N,K,act", [(1000, 256, 128, 2), (130, 70, 200, 0), (512, 600, 600, 1)])
def test_gemm_second_output_is_the_bf16_copy(M, N, K, act):
    g = torch.Generator(device=DEV); g.manual_seed(M + N)
    A = torch.randn(M, K, device=DEV, generator=g) / K ** 0.5; B = torch.randn(N, K, device=DEV, generator=g)
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    C, Cb = ops.gemm_bf16_tn(ops.to_bf16(A), ops.to_bf16(B), M, N, K, bias=bias, act=act, out_bf16=True)
    C2 = ops.gemm_bf16_tn(ops.to_bf16(A), ops.to_bf16(B), M, N, K, bias=bias, act=act)
    assert torch.equal(C, C2) and torch.equal(Cb[:, :N], C.bfloat16()) and not Cb[:, N:].any()
