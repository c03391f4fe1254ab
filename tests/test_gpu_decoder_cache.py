"""GPU: decoding with a key / value cache on the split-KV decode kernel (attention_decode.cu).

* The decode kernel against fp32 attention: Sq 1 / 2 / 15 / 16 over Skv 1 ... 4097 at head_dim 64 / 96 / 128, with one
  split and with many; masks ([B, Sq, Skv], key padding, one mask shared by the batch), causal, exact zeros for rows
  with no visible key; bit-exact run-to-run determinism.
* MultiHeadAttentionWithCache / TransformerDecoderLayer / TransformerDecoder reproduce the reference goldens.
* A past in the reference's contiguous layout and in ours gives the same result, for fp32 and bf16 callers.
* Incremental decoding of a CoCa-width TransformerDecoder (d 768, 12 heads, cross-attention over 256 image tokens,
  2 layers) one token at a time and in chunks of 5 and 17 equals the full-sequence forward under a causal mask, and the
  layer-0 cache equals the full-sequence keys / values bit for bit.
"""
import math
import os

import pytest
import torch

import decoder_cache_cases as DC
from multimodal_b200 import ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dev = torch.device("cuda")


def _ref_attn(q, k, v, B, Sq, Skv, H, D, mask3=None, causal=False):
    qh = q.float().view(B, Sq, H, D).transpose(1, 2)
    kh, vh = k.float().view(B, Skv, H, D).transpose(1, 2), v.float().view(B, Skv, H, D).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) / math.sqrt(D)
    if causal:
        s = s.masked_fill(~torch.ones(Sq, Skv, dtype=torch.bool, device=dev).tril(), float("-inf"))
    if mask3 is not None:
        s = s.masked_fill(~mask3.bool()[:, None], float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
    return (p @ vh).transpose(1, 2).reshape(B * Sq, H * D)


def _decode(q, k, v, B, Sq, Skv, H, D, mask=None, mask_bs=0, mask_qs=0, causal=False):
    out = torch.empty(B * Sq, H * D, device=dev, dtype=torch.bfloat16)
    ops.attention_fwd_decode(q, k, v, out, B=B, Sq=Sq, Skv=Skv, H=H, head_dim=D, bsq=Sq * H * D, bsk=Skv * k.stride(0),
                             bsv=Skv * v.stride(0), bso=Sq * H * D, scale=1 / math.sqrt(D), mask=mask, mask_bs=mask_bs,
                             mask_qs=mask_qs, causal=causal)
    return out


def _operands(B, Sq, Skv, H, D, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    q = torch.randn(B * Sq, H * D, device=dev, generator=g).bfloat16()
    kv = torch.randn(B * Skv, 2 * H * D, device=dev, generator=g).bfloat16()   # packed K|V rows, as the KV GEMM writes
    return q, kv[:, :H * D], kv[:, H * D:]


@pytest.mark.parametrize("BH", [(1, 2), (3, 88)])   # many splits (where Skv allows) / always one split
@pytest.mark.parametrize("Skv", [1, 63, 64, 65, 77, 1000, 4097])
@pytest.mark.parametrize("Sq", [1, 2, 15, 16])
@pytest.mark.parametrize("D", [64, 96, 128])
def test_decode_kernel_matches_fp32(D, Sq, Skv, BH):
    B, H = BH
    q, k, v = _operands(B, Sq, Skv, H, D)
    out = _decode(q, k, v, B, Sq, Skv, H, D)
    ref = _ref_attn(q, k, v, B, Sq, Skv, H, D)
    assert (out.float() - ref).abs().max().item() < 2e-2
    if BH == (3, 88):
        assert ops.attention_decode_splits(B, H, Skv) == 1
    elif Skv >= 1000:
        assert ops.attention_decode_splits(B, H, Skv) > 1


@pytest.mark.parametrize("kind", ["full", "key", "shared", "causal", "causal_mask"])
@pytest.mark.parametrize("Skv", [77, 1000, 4097])
@pytest.mark.parametrize("Sq", [1, 5, 16])
@pytest.mark.parametrize("D", [64, 128])
def test_decode_kernel_masks_causal_and_empty_rows(D, Sq, Skv, kind):
    B, H = 2, 3
    q, k, v = _operands(B, Sq, Skv, H, D, seed=1)
    g = torch.Generator(device=dev).manual_seed(2)
    full = torch.rand(B, Sq, Skv, device=dev, generator=g) > 0.5
    mask, bs, qs, mask3, causal = None, 0, 0, None, kind.startswith("causal")
    if kind in ("full", "causal_mask"):
        full[0, 0] = False                       # a row with no visible key
        mask, bs, qs, mask3 = full.to(torch.uint8).contiguous(), Sq * Skv, Skv, full
    elif kind == "key":
        kp = full[:, 0]
        kp[1] = False                            # a batch with no visible key at all
        mask, bs, qs, mask3 = kp.to(torch.uint8).contiguous(), Skv, 0, kp[:, None].expand(B, Sq, Skv)
    elif kind == "shared":
        sh = full[0]
        sh[-1] = False
        mask, bs, qs, mask3 = sh.to(torch.uint8).contiguous(), 0, Skv, sh[None].expand(B, Sq, Skv)
    out = _decode(q, k, v, B, Sq, Skv, H, D, mask, bs, qs, causal)
    ref = _ref_attn(q, k, v, B, Sq, Skv, H, D, mask3, causal)
    assert (out.float() - ref).abs().max().item() < 2e-2
    if mask3 is not None:
        vis = mask3.clone()
        if causal:
            vis &= torch.ones(Sq, Skv, dtype=torch.bool, device=dev).tril()
        empty = ~vis.any(-1)                     # [B, Sq]
        assert empty.any()
        assert (out.view(B, Sq, -1)[empty] == 0).all()


def test_decode_kernel_run_to_run_bit_exact():
    B, H, Sq, Skv, D = 1, 12, 4, 20000, 128
    q, k, v = _operands(B, Sq, Skv, H, D, seed=3)
    assert ops.attention_decode_splits(B, H, Skv) > 1
    a = _decode(q, k, v, B, Sq, Skv, H, D)
    for _ in range(3):
        assert torch.equal(a, _decode(q, k, v, B, Sq, Skv, H, D))


# ---- modules -------------------------------------------------------------------------------------------------------
def _ours():
    from multimodal_b200.modules.layers import multi_head_attention, transformer

    return DC.namespace(multi_head_attention, transformer)


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "decoder_cache_golden.pt"), map_location="cpu",
                      weights_only=False)


@pytest.mark.parametrize("name", list(DC.CASES))
def test_modules_reproduce_reference_goldens(gold, name):
    g = gold[name]
    m = DC.build(_ours(), name).to(dev)
    with torch.no_grad():
        res = DC.run(m, name, DC.to(g["inputs"], dev))
    assert sorted(res) == sorted(g["results"])
    for k, ref in g["results"].items():
        r = res[k]
        assert r.is_cuda and r.dtype == ref.dtype and r.shape == ref.shape, (k, r.dtype, r.shape)
        err = (r.float().cpu() - ref.float()).abs().max().item()
        assert err <= 2e-2 * ref.float().abs().max().item(), (name, k, err)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_past_layout_does_not_matter(dtype):
    """A past returned by an earlier call (transposed view of our row buffer) and the same values as a contiguous
    [B, H, S, hd] tensor (what the reference returns after torch.cat) give the same output and cache."""
    from multimodal_b200.modules.layers.multi_head_attention import MultiHeadAttentionWithCache

    torch.manual_seed(0)
    m = MultiHeadAttentionWithCache(768, 768, 12).to(dev).eval()
    x0 = torch.randn(2, 9, 768, device=dev, dtype=dtype)
    x1 = torch.randn(2, 1, 768, device=dev, dtype=dtype)
    with torch.no_grad():
        _, past = m(x0, x0, x0, use_cache=True)
        assert past[0].dtype == dtype and not past[0].is_contiguous()
        a = m(x1, x1, x1, past_key_value=past, use_cache=True)
        b = m(x1, x1, x1, past_key_value=tuple(t.contiguous() for t in past), use_cache=True)
    assert torch.equal(a.attn_output, b.attn_output)
    assert torch.equal(a.past_key_value[0], b.past_key_value[0]) and torch.equal(a.past_key_value[1], b.past_key_value[1])
    assert a.attn_output.dtype == dtype and a.past_key_value[0].dtype == dtype
    assert torch.equal(a.past_key_value[0][:, :, :9], past[0])


def _coca_decoder():
    from multimodal_b200.modules.layers.transformer import TransformerDecoder

    torch.manual_seed(0)
    dec = TransformerDecoder(2, 768, 12, 3072, activation=torch.nn.GELU, norm_first=True, use_cross_attention=True,
                             dim_kv=768, final_layer_norm_eps=1e-5)
    with torch.no_grad():   # non-trivial LayerNorm parameters
        for n, p in dec.named_parameters():
            if "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
    return dec.to(dev).eval()


def test_incremental_decoding_equals_full_forward():
    dec = _coca_decoder()
    B, T = 2, 40
    x = torch.randn(B, T, 768, device=dev)
    img = torch.randn(B, 256, 768, device=dev)
    causal = torch.ones(T, T, dtype=torch.bool, device=dev).tril()
    with torch.no_grad():
        full = dec(x, img, attention_mask=causal, use_cache=True)
        scale = full.last_hidden_state.abs().max().item()
        for chunk in (1, 5, 17):
            past, t0 = None, 0
            while t0 < T:
                t1 = min(T, t0 + chunk)
                n = t1 - t0
                mask = None if n == 1 else torch.ones(n, t1, dtype=torch.bool, device=dev).tril(t0)
                o = dec(x[:, t0:t1], img, attention_mask=mask, past_key_values=past, use_cache=True)
                err = (o.last_hidden_state - full.last_hidden_state[:, t0:t1]).abs().max().item()
                assert err <= 2e-2 * scale, (chunk, t0, err)
                past, t0 = o.current_key_values, t1
            # LayerNorm is per row and the GEMM's per-element k order does not depend on M: the layer-0 cache is exact
            assert torch.equal(past[0][0], full.current_key_values[0][0]), chunk
            assert torch.equal(past[0][1], full.current_key_values[0][1]), chunk


def test_forward_only_guard_under_grad_mode():
    from multimodal_b200._lib import MMBError

    dec = _coca_decoder()
    x = torch.randn(1, 1, 768, device=dev)
    with pytest.raises(MMBError, match="forward values only"):
        dec(x, torch.randn(1, 4, 768, device=dev))
    with pytest.raises(MMBError, match="forward values only"):
        dec.layer[0].attention(x, x, x)
