"""Split-K path of the wgmma GEMM (no bias / activation, few output tiles, long K: partial tiles are stored in a
workspace and summed in split order) vs a bf16-rounded fp64 matmul.  The path is also exercised through the MultiVAE tests
(dh2 = dlogits . W4); this file sorts last on purpose."""
import pytest
import torch

from elliot_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("M,N,K", [(512, 600, 26744), (77, 600, 3001), (1, 1, 4096), (130, 70, 2048), (256, 128, 8192)])
def test_split_k_matches_bf16_matmul(M, N, K):
    g = torch.Generator(device=DEV); g.manual_seed(M + N + K)
    A = torch.randn(M, K, device=DEV, generator=g) / K ** 0.5
    B = torch.randn(N, K, device=DEV, generator=g)
    C = ops.gemm_bf16_tn(ops.to_bf16(A), ops.to_bf16(B), M, N, K, alpha=0.5)
    ref = 0.5 * (A.bfloat16().double() @ B.bfloat16().double().T)
    assert (C.double() - ref).abs().max().item() < 2e-4


def test_split_k_respects_row_stride_padding():
    """C with ldc > N: the split-K sums must stay inside the N columns."""
    M, N, K, pad = 100, 200, 4096, 12
    g = torch.Generator(device=DEV); g.manual_seed(3)
    A = torch.randn(M, K, device=DEV, generator=g) / K ** 0.5
    B = torch.randn(N, K, device=DEV, generator=g)
    buf = torch.full((M, N + pad), 7.0, device=DEV)
    out = buf[:, :N]
    ops.gemm_bf16_tn(ops.to_bf16(A), ops.to_bf16(B), M, N, K, out=out)
    ref = A.bfloat16().double() @ B.bfloat16().double().T
    assert (out.double() - ref).abs().max().item() < 4e-4
    assert bool((buf[:, N:] == 7.0).all())
