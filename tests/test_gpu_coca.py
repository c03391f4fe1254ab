"""GPU parity of the CoCa forward (BASELINE.json config 5) against the reference goldens and the oracle, plus the
kernels only this path uses (general cross-attention, CoCa text embedding, label cross-entropy).

Tolerance: bf16 GEMM operands with fp32 accumulation / statistics; unit-norm embeddings agree to 5e-3 absolute, logits
to 2e-2 of their absmax, losses to 1e-2.  Token gathers and masks are bit-exact.
"""
import math
import os

import pytest
import torch

import coca_cases as CC
from oracle import coca_oracle as CO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "coca_golden.pt")


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _inference():
    """This file pins the no_grad forwards of the CoCa runtimes (engine_coca_train.py); their training forwards and
    backwards are covered by tests/test_gpu_coca_train.py."""
    with torch.no_grad():
        yield



@pytest.mark.parametrize("B,Sq,Skv,H,D,shared_q,causal,mask_kind", [
    (3, 32, 64, 4, 96, True, False, None),      # pooler: batch-shared queries, head_dim 96
    (2, 256, 256, 8, 96, True, False, None),    # CoCa ViT-L/14 captioning pooler shape
    (4, 1, 32, 4, 96, True, False, None),       # contrastive pooler: a single query
    (3, 12, 32, 6, 64, False, False, None),     # multimodal decoder cross-attention
    (3, 13, 13, 6, 64, False, False, "full"),   # text decoder: [B, S, S] mask
    (2, 77, 77, 12, 64, False, True, "key"),    # causal + key-padding mask
    (2, 275, 275, 2, 64, False, False, None),   # long self-attention through the general kernel
    (2, 40, 100, 2, 128, False, False, None),
])
def test_attention_fwd_generic(dev, B, Sq, Skv, H, D, shared_q, causal, mask_kind):
    from multimodal_b200 import ops

    torch.manual_seed(2)
    d = H * D
    q = torch.randn((1 if shared_q else B) * Sq, d, device=dev).bfloat16()
    kv = torch.randn(B * Skv, 2 * d, device=dev).bfloat16()
    mask = mask_bs = mask_qs = None
    ref_mask = None
    if mask_kind == "full":
        mask = (torch.rand(B, Sq, Skv, device=dev) < 0.7)
        mask[:, :, 0] = True
        ref_mask = mask[:, None]
        mask_bs, mask_qs = Sq * Skv, Skv
    elif mask_kind == "key":
        mask = (torch.rand(B, Skv, device=dev) < 0.8)
        mask[:, 0] = True
        ref_mask = mask[:, None, None, :]
        mask_bs, mask_qs = Skv, 0
    out = torch.empty(B * Sq, d, device=dev, dtype=torch.bfloat16)
    ops.attention_fwd_generic(q, kv[:, :d], kv[:, d:], out, B=B, Sq=Sq, Skv=Skv, H=H, head_dim=D, bsq=0 if shared_q else Sq * d,
                              bsk=Skv * 2 * d, bsv=Skv * 2 * d, bso=Sq * d, scale=1.0 / math.sqrt(D),
                              mask=mask.to(torch.uint8).contiguous() if mask is not None else None,
                              mask_bs=mask_bs or 0, mask_qs=mask_qs or 0, causal=causal)
    qf = (q.float().view(1, Sq, H, D).expand(B, -1, -1, -1) if shared_q else q.float().view(B, Sq, H, D)).transpose(1, 2)
    kf = kv[:, :d].float().reshape(B, Skv, H, D).transpose(1, 2)
    vf = kv[:, d:].float().reshape(B, Skv, H, D).transpose(1, 2)
    s = qf @ kf.transpose(-1, -2) / math.sqrt(D)
    if ref_mask is not None:
        s = s.masked_fill(~ref_mask, float("-inf"))
    if causal:
        s = s.masked_fill(~torch.tril(torch.ones(Sq, Skv, device=dev)).bool(), float("-inf"))
    ref = (torch.softmax(s, -1) @ vf).transpose(1, 2).reshape(B * Sq, d)
    err = (out.float() - ref).abs().max().item()
    assert err < 2.5e-2, err


def test_coca_helper_kernels(dev):
    from multimodal_b200 import ops

    torch.manual_seed(0)
    B, S, d, V = 4, 9, 128, 40
    ids = torch.randint(0, V, (B, S - 1), device=dev)
    emb, cls, pos = torch.randn(V, d, device=dev), torch.randn(d, device=dev), torch.randn(S, d, device=dev)
    x = torch.empty(B * S, d, device=dev)
    ops.coca_text_embed_fwd(ids, emb, cls, pos, x, B, S, d, V)
    ref = torch.cat([emb[ids], cls.view(1, 1, d).expand(B, 1, d)], 1) + pos
    assert torch.equal(x.view(B, S, d), ref)
    # label cross-entropy with ignore_index
    M, V2 = 37, 1000
    logits = torch.randn(M, V2, device=dev) * 3
    labels = torch.randint(0, V2, (M,), device=dev)
    labels[::5] = 0
    acc = torch.zeros(2, device=dev)
    ops.ce_labels(logits, labels, 1, 0, M, V2, None, acc)
    ref = torch.nn.functional.cross_entropy(logits, labels, ignore_index=0)
    assert abs((acc[0] / acc[1]).item() - ref.item()) < 1e-4
    assert acc[1].item() == (labels != 0).sum().item()
    # no-CLS token assembly (include_cls_embed=False)
    P = 16
    po = torch.randn(B * P, d, device=dev).bfloat16()
    posi = torch.randn(1, P, d, device=dev)
    xo = torch.empty(B * P, d, device=dev)
    ops.vit_assemble_fwd(po, None, posi, None, None, xo, B, P, d)
    assert torch.equal(xo.view(B, P, d), po.float().view(B, P, d) + posi)


@pytest.mark.parametrize("name", list(CC.CASES))
def test_coca_forward_against_reference_golden(dev, name):
    from multimodal_b200.models.coca import coca_for_pretraining

    g = torch.load(GOLD)[name]
    m = CC.build(coca_for_pretraining, name)
    assert CC.param_checksum(m) == pytest.approx(g["param_checksum"], rel=1e-12)
    m = m.to(dev)
    images, texts = g["inputs"]["images"].to(dev), g["inputs"]["texts"].to(dev)
    o = m.model(images, texts)
    assert o.image_pooled_output.shape == g["image_pooled_output"].shape
    e_img = (o.image_pooled_output.cpu() - g["image_pooled_output"]).abs().max().item()
    e_txt = (o.text_pooled_output.cpu() - g["text_pooled_output"]).abs().max().item()
    mm_ref = g["multimodal_embeddings"]
    e_mm = (o.multimodal_embeddings.cpu() - mm_ref).abs().max().item() / mm_ref.abs().max().item()
    print(f"{name}: |d img| {e_img:.2e} |d txt| {e_txt:.2e} rel d logits {e_mm:.2e}")
    assert e_img < 5e-3 and e_txt < 5e-3 and e_mm < 2e-2
    with torch.no_grad():
        losses = m(images, texts)
    with torch.enable_grad():         # grad mode on + trainable parameters: the autograd path, same values
        tl = m(images, texts)
    assert tl["contrastive"].requires_grad and tl["captioning"].requires_grad
    assert abs(tl["contrastive"].item() - losses["contrastive"].item()) < 1e-2
    assert abs(tl["captioning"].item() - losses["captioning"].item()) < 1e-2
    ref = CO.coca_forward(m.state_dict(), CC.CASES[name]["kwargs"], images.cpu(), texts.cpu())
    assert abs(losses["contrastive"].item() - ref["contrastive"].item()) < 1e-2
    assert abs(losses["captioning"].item() - ref["captioning"].item()) < 1e-2
    if "contrastive" in g:   # reference CoCaForPretraining values (parallel pooler)
        assert abs(losses["contrastive"].item() - g["contrastive"].item()) < 1e-2
        assert abs(losses["captioning"].item() - g["captioning"].item()) < 1e-2
    # explicit padding mask == the pad-derived default
    o2 = m.model(images, texts, texts != 0)
    assert torch.equal(o2.text_pooled_output, o.text_pooled_output)


def test_coca_vit_l_14_shapes_against_oracle(dev):
    """The real CoCa ViT-L/14 layer shapes (d=1024/16 heads, 256 tokens, pooler head_dim 96, text 77 positions, vocab
    49408) at reduced depth (2+1+1 layers) and B=2, against the oracle."""
    from multimodal_b200.models.coca import coca_for_pretraining

    kw = dict(vision_patch_size=14, vision_n_layer=2, vision_n_head=16, vision_dim_feedforward=4096,
              vision_include_cls_embed=False, vocab_size=49408, num_text_positions=77, text_hidden_dim=768,
              text_n_layer=1, text_n_head=12, text_dim_feedforward=3072, text_output_dim=768, fusion_n_layer=1,
              fusion_n_head=12, fusion_dim_feedforward=3072, multimodal_output_projection_dim=49408,
              pooler_input_embed_dim=1024, pooler_output_embed_dim=768, pooler_n_head=8, cascaded_pooler=True)
    torch.manual_seed(0)
    m = coca_for_pretraining(**kw).eval()
    gen = torch.Generator().manual_seed(1)
    images = torch.randn(2, 3, 224, 224, generator=gen)
    texts = torch.randint(1, 49408, (2, 77), generator=gen)
    texts[1, 50:] = 0
    ref = CO.coca_forward(m.state_dict(), kw, images, texts)
    m = m.to(dev)
    o = m.model(images.to(dev), texts.to(dev))
    assert o.multimodal_embeddings.shape == (2, 76, 49408)
    assert (o.image_pooled_output.cpu() - ref["image_pooled_output"]).abs().max().item() < 5e-3
    assert (o.text_pooled_output.cpu() - ref["text_pooled_output"]).abs().max().item() < 5e-3
    mm = ref["multimodal_embeddings"]
    assert (o.multimodal_embeddings.cpu() - mm).abs().max().item() / mm.abs().max().item() < 2e-2
    with torch.no_grad():
        losses = m(images.to(dev), texts.to(dev))
    assert abs(losses["captioning"].item() - ref["captioning"].item()) < 2e-2
