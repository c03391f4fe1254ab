"""GPU tests (H100) of the 128 x 256 GEMM tile (256 x 256 per 2-CTA cluster) and its TMA-store epilogue.

Every kernel instantiation runs in both modes at shapes whose M and N cross the 256-row / 256-column tile boundaries
and whose K leaves a tail shorter than one 64-deep k-block, against an fp32 matmul of the same bf16 operands.
Tolerances are those of test_gpu_parity.test_gemm_tcgen05: 6e-3 of max |ref| for bf16 outputs (output rounding),
2e-5 * sqrt(K) for fp32 outputs (accumulation order only).
"""
import math

import pytest
import torch

from oracle import clip_oracle as O

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


def _rel(got, ref):
    got, ref = got.float(), ref.float()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-20)).item()


def _act(x, act):
    return O.quick_gelu(x) if act == 0 else torch.nn.functional.gelu(x)


def _act_grad(x, act):
    x = x.clone().requires_grad_(True)
    _act(x, act).sum().backward()
    return x.grad


def _operands(dev, M, N, K, a_mn, b_mn, seed=0):
    torch.manual_seed(seed)
    A2 = torch.randn(M, K, device=dev).bfloat16()
    B2 = torch.randn(N, K, device=dev).bfloat16()
    A = A2.t().contiguous() if a_mn else A2
    B = B2.t().contiguous() if b_mn else B2
    return A2, B2, A, B


def _check_kind(dev, M, N, K, a_mn, b_mn, epi, act, splits):
    from multimodal_b200 import ops

    A2, B2, A, B = _operands(dev, M, N, K, a_mn, b_mn)
    bias = torch.randn(N, device=dev)
    ref = A2.float() @ B2.float().t()
    if epi == 0:
        cs = torch.ones(N, device=dev)
        out = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=0, bias=bias, alpha=0.5, colsum=cs)
        assert _rel(out, 0.5 * ref + bias) < 6e-3
        torch.testing.assert_close(cs, 1.0 + out.float().sum(0), rtol=1e-4, atol=1e-3 * out.float().abs().sum(0).max().item())
    elif epi == 1:
        pre, actv = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=1, bias=bias, alpha=0.125, act=act)
        assert _rel(pre, 0.125 * ref + bias) < 6e-3
        assert _rel(actv, _act(pre.float(), act)) < 6e-3
    elif epi == 2:
        aux = torch.randn(M, N, device=dev).bfloat16()
        cs = torch.zeros(N, device=dev)
        out = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=2, aux=aux, alpha=0.125, colsum=cs, act=act)
        torch.testing.assert_close(cs, out.float().sum(0), rtol=1e-4, atol=1e-3 * out.float().abs().sum(0).max().item())
        assert _rel(out, 0.125 * ref * _act_grad(aux.float(), act)) < 6e-3
    else:
        out = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=3, bias=bias, splits=splits)
        assert _rel(out, ref + bias) < 2e-5 * math.sqrt(K) + 1e-5
        # accumulate: D += result (a TMA reduce-add without split-K)
        out2 = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=3, splits=splits, out=out.clone(), accumulate=True)
        assert _rel(out2, 2 * ref + bias) < 2e-5 * math.sqrt(K) + 1e-5


# every instantiation gemm_launch dispatches to: (a_mn, b_mn, epilogue, act, splits)
_KINDS = [(0, 0, 0, 0, 1), (0, 0, 1, 0, 1), (0, 0, 1, 1, 1), (0, 0, 3, 0, 1), (0, 1, 0, 0, 1), (0, 1, 2, 0, 1),
          (0, 1, 2, 1, 1), (0, 1, 3, 0, 1), (1, 1, 3, 0, 3), (1, 0, 3, 0, 2)]
# M and N on both sides of the 256 boundaries (one row / column tile more than a multiple, or one less), K tails
_SHAPES = [(255, 520, 136), (257, 264, 200), (4097, 776, 72), (1000, 1032, 584)]


@pytest.mark.parametrize("M,N,K", _SHAPES)
@pytest.mark.parametrize("a_mn,b_mn,epi,act,splits", _KINDS)
def test_gemm_wide_tile_boundaries(dev, gemm_mode, M, N, K, a_mn, b_mn, epi, act, splits):
    if a_mn:   # an MN-major A is stored [K, M]: its row pitch M must be a multiple of 8 elements
        M = {255: 248, 257: 264, 4097: 4104}.get(M, M)
    _check_kind(dev, M, N, K, a_mn, b_mn, epi, act, splits)


# the ViT-B/16 image tower's GEMMs at the benchmark's N and K (M cut from 100 864 tokens to 8 k rows)
_IMAGE_TOWER = [
    (8192, 2304, 768, 0, 0, 0, 0, 1),    # QKV projection
    (8192, 3072, 768, 0, 0, 1, 0, 1),    # FC1 + QuickGELU
    (8192, 768, 3072, 0, 0, 0, 0, 1),    # FC2
    (8192, 768, 3072, 0, 1, 0, 0, 1),    # FC1 dgrad
    (8192, 3072, 768, 0, 1, 2, 0, 1),    # FC2 dgrad x QuickGELU'
    (768, 3072, 8192, 1, 1, 3, 0, 5),    # FC1 wgrad, split-K
]


@pytest.mark.parametrize("M,N,K,a_mn,b_mn,epi,act,splits", _IMAGE_TOWER)
def test_gemm_wide_image_tower_shapes(dev, gemm_mode, M, N, K, a_mn, b_mn, epi, act, splits):
    _check_kind(dev, M, N, K, a_mn, b_mn, epi, act, splits)


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


def test_f32_output_not_16_byte_aligned(dev, gemm_mode):
    """An fp32 column slice (base 4 bytes past a 16-byte boundary) cannot take TMA stores: direct stores instead."""
    from multimodal_b200 import ops

    M, N, K = 300, 516, 200
    A2, B2, A, B = _operands(dev, M, N, K, 0, 0, seed=5)
    ref = A2.float() @ B2.float().t()
    full = torch.zeros(M, N + 4, device=dev)
    out = full[:, 1:N + 1]
    assert out.data_ptr() % 16 != 0
    ops.gemm(A, B, epilogue=ops.EPI_F32, out=out)
    assert _rel(out, ref) < 2e-5 * math.sqrt(K) + 1e-5
    ops.gemm(A, B, epilogue=ops.EPI_F32, out=out, accumulate=True)
    assert _rel(out, 2 * ref) < 2e-5 * math.sqrt(K) + 1e-5
    assert full[:, 0].abs().max().item() == 0 and full[:, N + 1:].abs().max().item() == 0

