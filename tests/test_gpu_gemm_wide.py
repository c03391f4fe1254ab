"""GPU tests (H100) of the split-K order of the 128 x 256 GEMM tile (256 x 256 per 2-CTA cluster).

Every instantiation's per-element float64 contract, at the tile boundaries, K tails, persistent loops and the image
tower's shapes, is in tests/kernel_contract_cases.py (check_gemm); this file keeps the exact split-K property that the
contract does not restate.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(params=[0, 1], ids=["1cta", "cluster"])
def gemm_mode(request):
    """0: one CTA per 128 x 256 tile; 1: 2-CTA clusters (256 x 256 tiles, B multicast to both CTAs)."""
    from multimodal_b200 import _lib

    assert _lib.lib().mmb_gemm_set_mode(request.param, 8) == 0
    yield request.param
    assert _lib.lib().mmb_gemm_set_mode(-1, 0) == 0


def _operands(dev, M, N, K, a_mn, b_mn, seed=0):
    torch.manual_seed(seed)
    A2 = torch.randn(M, K, device=dev).bfloat16()
    B2 = torch.randn(N, K, device=dev).bfloat16()
    A = A2.t().contiguous() if a_mn else A2
    B = B2.t().contiguous() if b_mn else B2
    return A2, B2, A, B


@pytest.mark.parametrize("M,N,K,splits", [(768, 768, 8192 + 200, 5), (2304, 768, 6000, 7), (520, 1032, 3000, 3)])
def test_splitk_is_in_order_sum_of_slices(dev, gemm_mode, M, N, K, splits):
    """split-K == ((0 + P0) + P1) + ... bit for bit, P_s the splits=1 product over the s-th kb_per_split k-blocks."""
    from multimodal_b200 import ops

    _, _, A, B = _operands(dev, M, N, K, 1, 1, seed=3)   # wgrad layout: both operands [K, *]
    kb = (K + 63) // 64
    kb_per = (kb + splits - 1) // splits
    ref = torch.zeros(M, N, device=dev)
    for k0 in range(0, K, kb_per * 64):
        k1 = min(K, k0 + kb_per * 64)
        ref = ref + ops.gemm(A[k0:k1], B[k0:k1], a_mn=True, b_mn=True, epilogue=ops.EPI_F32, splits=1)
    out1 = ops.gemm(A, B, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, splits=splits)
    out2 = ops.gemm(A, B, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, splits=splits)
    torch.cuda.synchronize()
    assert torch.equal(out1, ref)
    assert torch.equal(out1, out2)
