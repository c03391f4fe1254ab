"""GPU tests of random patch dropping (PatchEmbeddings(patch_drop_rate=...), FLIP, arXiv 2212.00794): the gathered
patch front-end kernels against their CPU emulations and float64 sums, random-number parity with the reference's
draws on the device, gradients of CoCa and of real-width ViTs against autograd over the fp32 oracle fed the same kept
patches, grad-mode invariance, unchanged eval behaviour and a short training run."""
import math

import pytest
import torch
import torch.nn.functional as F

import coca_cases as CC
import patch_drop_cases as PD
from oracle import coca_oracle as CO

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _exact_fp32_reference():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


def _keep(B, P, L, gen, never=()):
    """int32 [B, L]: per sample L distinct patches in random order, none of `never` (so those rows are kept by no one)."""
    allowed = torch.tensor([p for p in range(P) if p not in never])
    return torch.stack([allowed[torch.randperm(len(allowed), generator=gen)[:L]] for _ in range(B)]).to(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
# kernel contracts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,ps,L", [(3, 28, 42, 14, 5), (2, 64, 48, 16, 12), (4, 224, 224, 14, 64)])
def test_im2col_gather_equals_im2col_rows(dev, B, H, W, ps, L):
    from multimodal_b200 import ops

    gen = torch.Generator().manual_seed(1)
    P, K = (H // ps) * (W // ps), 3 * ps * ps
    Kp = -(-K // 8) * 8
    img = torch.randn(B, 3, H, W, generator=gen).to(dev)
    keep = _keep(B, P, L, gen).to(dev)
    full = torch.zeros(B * P, Kp, device=dev, dtype=torch.bfloat16)
    ops.im2col(img, ps, full[:, :K])
    out = torch.full((B * L, Kp), float("nan"), device=dev, dtype=torch.bfloat16)
    ops._im2col_gather(img, keep, ps, out[:, :K])
    rows = (torch.arange(B, device=dev)[:, None] * P + keep.long()).reshape(-1)
    assert torch.equal(out[:, :K].view(torch.int16), full[rows, :K].view(torch.int16))
    assert torch.isnan(out[:, K:].float()).all()   # the pitch padding is not written


def _assembly_case(dev, B, P, L, d, cls, masked, seed):
    gen = torch.Generator().manual_seed(seed)
    off = 1 if cls else 0
    keep = _keep(B, P, L, gen, never=(0, P - 1))
    t = dict(
        keep=keep,
        po=torch.randn(B * L, d, generator=gen).to(torch.bfloat16),
        cls=torch.randn(1, 1, d, generator=gen) if cls else None,
        pos=torch.randn(1, off + P, d, generator=gen),
        mt=torch.randn(1, 1, d, generator=gen) if masked else None,
        pm=(torch.rand(B, P, generator=gen) < 0.4).to(torch.uint8) if masked else None,
        g=torch.randn(B * (off + L), d, generator=gen),
    )
    return t, {k: (v.to(dev) if v is not None else None) for k, v in t.items()}


def _emu_fwd(t, B, P, L, d):
    """CPU emulation of the gathered assembly: bf16 -> fp32, then one fp32 add."""
    keep = t["keep"].long()
    off = 1 if t["cls"] is not None else 0
    e = t["po"].float().view(B, L, d)
    if t["pm"] is not None:
        m = torch.gather(t["pm"], 1, keep).bool().unsqueeze(-1)
        e = torch.where(m, t["mt"].view(1, 1, d).expand(B, L, d), e)
    pos = t["pos"].view(off + P, d)
    x = e + pos[off + keep]
    if off:
        x = torch.cat([(t["cls"].view(d) + pos[0]).view(1, 1, d).expand(B, 1, d), x], 1)
    return x.reshape(B * (off + L), d)


@pytest.mark.parametrize("B,P,L,d,cls,masked", [
    (5, 64, 17, 96, True, True),
    (3, 196, 98, 768, True, False),      # ViT-B/16 at 0.5: 1 + 98 tokens
    (64, 256, 64, 1024, False, True),    # ViT-L/14 at 0.75, no CLS
    (2, 12, 1, 32, False, False),        # one kept token
])
def test_gathered_assembly_forward_and_backward(dev, B, P, L, d, cls, masked):
    from multimodal_b200 import ops

    t, u = _assembly_case(dev, B, P, L, d, cls, masked, seed=B * 7 + L)
    off = 1 if cls else 0
    S = off + L
    x = torch.full((B * S, d), float("nan"), device=dev)
    ops._vit_assemble_gather_fwd(u["po"], u["cls"], u["pos"], u["mt"], u["pm"], u["keep"], x, P, d)
    assert torch.equal(x.cpu(), _emu_fwd(t, B, P, L, d))

    def bwd():
        dp = torch.full((B * L, d), float("nan"), device=dev, dtype=torch.bfloat16)
        dpos = torch.zeros(off + P, d, device=dev)
        dcls = torch.zeros(d, device=dev) if cls else None
        dmt = torch.zeros(d, device=dev) if masked else None
        ops._vit_assemble_gather_bwd(u["g"], u["pm"], u["keep"], dp, dmt, dcls, dpos, P, d, cls)
        torch.cuda.synchronize()
        return dp, dpos, dcls, dmt

    dp, dpos, dcls, dmt = bwd()
    keep = t["keep"].long()
    g = t["g"].view(B, S, d).double()
    gp = g[:, off:]
    m = torch.gather(t["pm"], 1, keep).bool() if masked else torch.zeros(B, L, dtype=torch.bool)
    want_dp = torch.where(m.unsqueeze(-1), torch.zeros_like(gp), gp).float().to(torch.bfloat16).reshape(B * L, d)
    assert torch.equal(dp.cpu().view(torch.int16), want_dp.view(torch.int16))

    def check(got, want, want_abs, n_terms, what):
        # fp32 sums of n terms in any association order: |err| <= (depth) u sum|v|, depth <= n + the 8-way final sums
        bound = (n_terms + 10) * EPS32 * want_abs + 1e-30
        err = (got.cpu().double() - want).abs()
        assert (err <= bound).all(), (what, (err - bound).max().item())

    ref_pos = torch.zeros(off + P, d, dtype=torch.float64)
    abs_pos = torch.zeros(off + P, d, dtype=torch.float64)
    ref_pos[off:].index_add_(0, keep.reshape(-1), gp.reshape(B * L, d))
    abs_pos[off:].index_add_(0, keep.reshape(-1), gp.abs().reshape(B * L, d))
    if cls:
        ref_pos[0], abs_pos[0] = g[:, 0].sum(0), g[:, 0].abs().sum(0)
        check(dcls, ref_pos[0], abs_pos[0], B, "dcls")
    check(dpos, ref_pos, abs_pos, B, "dpos")
    unkept = [off + 0, off + P - 1]
    assert (dpos[unkept] == 0).all() and not torch.signbit(dpos[unkept]).any()
    if masked:
        gm = gp * m.unsqueeze(-1)
        check(dmt, gm.sum((0, 1)), gm.abs().sum((0, 1)), B * L, "dmask_token")
    again = bwd()
    for a, b in zip((dp, dpos, dcls, dmt), again):
        if a is not None:
            assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                               b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# random-number parity with the reference's draws on the device
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(PD.PATCH_EMBED))
def test_standalone_patch_embeddings_draw_like_the_reference(dev, name):
    from multimodal_b200.modules.layers.patch_embedding import PatchEmbeddings
    from multimodal_b200.modules.masking.random_masking import random_masking, random_masking_2d

    c = PD.PATCH_EMBED[name]
    pe = PD.build_patch_embed(PatchEmbeddings, name).to(dev)
    images, mask = PD.patch_embed_inputs(name)
    images = images.to(dev)
    torch.manual_seed(c["seed"])
    with torch.no_grad():
        out = pe(images, image_patches_mask=mask.to(dev) if mask is not None else None)
    state = torch.cuda.get_rng_state()
    # the reference's forward draws inside random_masking(_2d) on the embeddings' device, after the projection
    B, P, d = images.shape[0], pe.num_patches_h * pe.num_patches_w, pe.position_embeddings.shape[-1]
    x = torch.randn(B, P, d, device=dev)
    torch.manual_seed(c["seed"])
    rate = c["kw"]["patch_drop_rate"]
    if isinstance(rate, tuple):
        xm = random_masking_2d(x, rate[0], rate[1], pe.num_patches_h, pe.num_patches_w)
        assert out.random_mask is None and out.ids_restore is None
        n_tok = xm.shape[1]
    else:
        r = random_masking(x, rate)
        assert torch.equal(out.random_mask, r.mask) and torch.equal(out.ids_restore, r.ids_restore)
        n_tok = r.ids_keep.shape[1]
    assert torch.equal(torch.cuda.get_rng_state(), state)
    off = 1 if pe.include_cls_embed else 0
    assert out.embeddings.shape == (B, off + n_tok, d)
    # values: the oracle on the same kept patches (bf16 patch GEMM on the device)
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices
    torch.manual_seed(c["seed"])
    keep = patch_keep_indices(pe, B, dev)[0]
    sd = {k: v.detach().cpu() for k, v in pe.state_dict().items()}
    ref = PD.patch_embed(images.cpu(), sd, "", c["kw"]["patch_size"], keep.cpu(), mask)
    assert _rel(out.embeddings.cpu(), ref) < 1e-2


# ---------------------------------------------------------------------------------------------------------------------
# gradients against autograd over the fp32 oracle fed the same kept patches
# ---------------------------------------------------------------------------------------------------------------------
def _check_grads(m, sd, bar, tag, skip=()):
    rows = []
    for k, p in m.named_parameters():
        ref = sd[k].grad
        if ref is None or ref.norm().item() == 0.0:
            assert p.grad is None or p.grad.abs().max().item() < 1e-5, k
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        if k.endswith("k_proj.bias") or k in skip:
            continue
        rows.append((k, _rel(p.grad.cpu(), ref)))
    errs = sorted(r[1] for r in rows)
    print(f"{tag}: relative-L2 gradient error over {len(rows)} parameter tensors: median {errs[len(errs) // 2]:.3e} "
          f"max {errs[-1]:.3e}")
    for k, a in rows:
        assert a < bar, (k, a)
    return rows


@pytest.mark.parametrize("name,rate,seed", [("coca_small", 0.5, 41), ("coca_small", (0.5, 0.5), 42),
                                            ("coca_parallel", 0.5, 43), ("coca_parallel", (0.5, 0.5), 44)])
def test_coca_gradients_with_patch_drop(dev, name, rate, seed):
    from multimodal_b200.engine_coca_train import linear_cross_entropy
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    m = CC.build(lambda **kw: coca_for_pretraining(**kw, vision_patch_drop_rate=rate), name).to(dev).train()
    cfg = dict(CC.CASES[name]["kwargs"])
    cfg.setdefault("pad_idx", 0)
    cpu_inp = CC.inputs(name)
    images, texts = cpu_inp["images"], cpu_inp["texts"]
    torch.manual_seed(seed)
    keep = patch_keep_indices(m.model.vision_encoder.embeddings, images.shape[0], dev)[0].cpu()
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    x = PD.vision_encoder(images, sd, cfg, keep=keep)
    H = cfg["pooler_n_head"]
    if cfg.get("cascaded_pooler", True):
        cap = CO.attention_pooler(x, sd, "model.vision_pooler.poolers.0", H)
        con = CO.attention_pooler(cap, sd, "model.vision_pooler.poolers.1", H)
    else:
        both = CO.attention_pooler(x, sd, "model.vision_pooler", H)
        con, cap = both[:, 0], both[:, 1:]
    img = F.normalize(CO._lin(con, sd, "model.vision_proj"), dim=-1)
    pooled, tokens = CO.text_decoder(texts, sd, cfg)
    txt = F.normalize(pooled, dim=-1)
    logits = CO.multimodal_decoder(tokens, cap, sd, cfg)
    cap_ref = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), texts[:, 1:].reshape(-1), ignore_index=0)
    gen = torch.Generator().manual_seed(21)
    wi, wt = torch.randn(img.shape, generator=gen), torch.randn(txt.shape, generator=gen)
    total_ref = cap_ref + (wi * img).sum() + (wt * txt).sum()
    total_ref.backward()

    torch.manual_seed(seed)
    outs = m.model._forward_impl(images.to(dev), texts.to(dev), None, want_logits=False)
    cap_loss = linear_cross_entropy(outs.multimodal_embeddings.hidden, outs.multimodal_embeddings.projection,
                                    texts[:, 1:].contiguous().to(dev), m.caption_loss.ignore_index)
    total = cap_loss + (wi.to(dev) * outs.image_pooled_output).sum() + (wt.to(dev) * outs.text_pooled_output).sum()
    assert abs(total.item() - total_ref.item()) < 3e-2 * max(1.0, abs(total_ref.item())), (total.item(), total_ref.item())
    total.backward()
    pad = m.model.text_decoder.embeddings.token_embeddings.padding_idx
    rows = _check_grads(m, sd, 4e-2, f"{name} rate {rate}",
                        skip=("model.text_decoder.embeddings.token_embeddings.weight",) if pad is not None else ())
    assert any(k.endswith("position_embeddings") and "vision" in k for k, _ in rows)
    # position-embedding rows of patches no sample kept get exactly zero gradient
    pe_grad = m.model.vision_encoder.embeddings.position_embeddings.grad[0]
    off = 1 if m.model.vision_encoder.embeddings.include_cls_embed else 0
    P = pe_grad.shape[0] - off
    unkept = sorted(set(range(P)) - set(keep.reshape(-1).tolist()))
    if unkept:
        assert (pe_grad[[off + p for p in unkept]] == 0).all()


@pytest.mark.parametrize("tag,image,ps,d,heads,ff,cls,rate", [
    ("vit_l14_w_r75", 224, 14, 1024, 16, 4096, False, 0.75),   # 256 patches -> 64 tokens
    ("vit_b16_w_r50", 224, 16, 768, 12, 3072, True, 0.5),      # 196 patches + CLS -> 1 + 98 tokens
])
def test_vit_gradients_with_patch_drop_at_real_width(dev, tag, image, ps, d, heads, ff, cls, rate):
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    torch.manual_seed(0)
    vit = vision_transformer(patch_size=ps, hidden_dim=d, dim_feedforward=ff, n_layer=2, n_head=heads, image_size=image,
                             include_cls_embed=cls, layer_norm_eps=1e-5, final_layer_norm_eps=1e-5,
                             patch_drop_rate=rate)
    g = torch.Generator().manual_seed(13)
    with torch.no_grad():
        for p in vit.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    vit = vit.to(dev).train()
    B = 3
    images = torch.randn(B, 3, image, image, generator=g)
    cfg = dict(vision_patch_size=ps, vision_n_layer=2, vision_n_head=heads, vision_layer_norm_eps=1e-5,
               vision_final_layer_norm_eps=1e-5)
    torch.manual_seed(5)
    keep = patch_keep_indices(vit.embeddings, B, dev)[0].cpu()
    L = keep.shape[1]
    sd = {"v." + k: v.detach().cpu().clone().requires_grad_(True) for k, v in vit.state_dict().items()}
    ref = PD.vision_encoder(images, sd, cfg, p="v", keep=keep)
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    torch.manual_seed(5)
    out = vit(images.to(dev))
    assert out.last_hidden_state.shape == (B, (1 if cls else 0) + L, d)
    assert all(h.shape == out.last_hidden_state.shape for h in out.hidden_states)
    assert _rel(out.last_hidden_state.detach().cpu(), ref.detach()) < 2e-2
    (out.last_hidden_state * w.to(dev)).sum().backward()
    _check_grads(vit, {k[2:]: v for k, v in sd.items()}, 4e-2, tag)


# ---------------------------------------------------------------------------------------------------------------------
# grad-mode invariance, unchanged eval behaviour, training
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", [0.5, (0.5, 0.5)])
def test_no_grad_equals_grad_mode_forward_with_patch_drop(dev, rate):
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining

    m = CC.build(lambda **kw: coca_for_pretraining(**kw, vision_patch_drop_rate=rate), "coca_small").to(dev).train()
    inp = {k: v.to(dev) for k, v in CC.inputs("coca_small").items()}
    torch.manual_seed(3)
    with torch.no_grad():
        a = m.model(inp["images"], inp["texts"])
        va = m.model.vision_encoder(inp["images"])
    torch.manual_seed(3)
    b = m.model(inp["images"], inp["texts"])
    vb = m.model.vision_encoder(inp["images"])
    assert b.image_pooled_output.requires_grad
    for x, y in zip(a[:3], b[:3]):   # the fourth field (multimodal_pooled_embeddings) is None
        assert torch.equal(x, y.detach())
    assert torch.equal(va.last_hidden_state, vb.last_hidden_state.detach())
    for x, y in zip(va.hidden_states, vb.hidden_states):
        assert torch.equal(x, y.detach())


def test_eval_ignores_patch_drop_rate(dev):
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining

    plain = CC.build(lambda **kw: coca_for_pretraining(**kw), "coca_small").to(dev).eval()
    drop = CC.build(lambda **kw: coca_for_pretraining(**kw, vision_patch_drop_rate=0.5), "coca_small").to(dev).eval()
    assert CC.param_checksum(plain) == CC.param_checksum(drop)
    inp = {k: v.to(dev) for k, v in CC.inputs("coca_small").items()}
    with torch.no_grad():
        a = plain.model(inp["images"], inp["texts"])
        state = torch.cuda.get_rng_state()
        b = drop.model(inp["images"], inp["texts"])
        assert torch.equal(torch.cuda.get_rng_state(), state)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    c = drop.model(inp["images"], inp["texts"])       # grad mode on, eval(): no dropping either
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert torch.equal(c.image_pooled_output.detach(), a.image_pooled_output)


def test_coca_for_pretraining_trains_with_patch_drop(dev):
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining

    m = CC.build(lambda **kw: coca_for_pretraining(**kw, vision_patch_drop_rate=0.5), "coca_parallel").to(dev).train()
    inp = {k: v.to(dev) for k, v in CC.inputs("coca_parallel").items()}
    opt = torch.optim.SGD(m.parameters(), lr=0.02)
    hist = []
    for _ in range(4):
        torch.manual_seed(9)   # the same patches every step: the loss change measures the update, not the draw
        opt.zero_grad(set_to_none=True)
        out = m(inp["images"], inp["texts"])
        total = out["contrastive"] + out["captioning"]
        assert total.requires_grad and math.isfinite(total.item())
        total.backward()
        hist.append(total.item())
        opt.step()
    print("CoCaForPretraining (patch drop 0.5) total loss over SGD steps:", hist)
    assert hist[-1] < hist[0], hist
