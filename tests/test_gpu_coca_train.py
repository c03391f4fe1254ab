"""GPU parity of the CoCa backward building blocks (SURVEY.md §8 a14 / f3 as training steps) against torch autograd."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("B,Sq,Skv,H,hd,kind", [
    (3, 13, 37, 2, 64, "cross"),          # multimodal decoder cross-attention
    (2, 76, 256, 12, 64, "cross"),        # ... at CoCa's real sequence lengths
    (3, 5, 20, 2, 96, "shared_q"),        # attention pooler: learned queries shared by the batch, head_dim 96
    (2, 256, 257, 8, 96, "shared_q"),     # ... captioning pooler of ViT-L/14
    (4, 1, 40, 2, 128, "shared_q"),       # contrastive pooler (one query), head_dim 128
    (3, 21, 21, 2, 64, "mask"),           # text decoder: [B, S, S] boolean mask on a packed QKV buffer
    (2, 33, 33, 3, 64, "causal"),
    (2, 40, 600, 2, 64, "cross"),         # more than 512 keys: the three-sweep path of the query kernel
])
def test_attention_bwd_generic(dev, B, Sq, Skv, H, hd, kind):
    from multimodal_b200 import ops

    torch.manual_seed(5)
    d = H * hd
    scale = 1.0 / math.sqrt(hd)
    bf = torch.bfloat16
    mask = None
    if kind in ("mask", "causal"):   # self-attention on a packed [B*S, 3d] buffer (column slices as operands)
        qkv = (torch.randn(B * Sq, 3 * d, device=dev) * 0.7).to(bf)
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        bsq = bsk = bsv = Sq * 3 * d
        dqkv = torch.full_like(qkv, float("nan"))
        dq, dk, dv = dqkv[:, :d], dqkv[:, d:2 * d], dqkv[:, 2 * d:]
        if kind == "mask":
            mask = (torch.rand(B, Sq, Skv, device=dev) < 0.6)
            mask[:, :, 0] = True
            mask[1, 3, :] = False    # a fully masked query row: zeros, no NaN
    else:
        nq_rows = Sq if kind == "shared_q" else B * Sq
        q = (torch.randn(nq_rows, d, device=dev) * 0.7).to(bf)
        kv = (torch.randn(B * Skv, 2 * d, device=dev) * 0.7).to(bf)
        k, v = kv[:, :d], kv[:, d:]
        bsq = 0 if kind == "shared_q" else Sq * d
        bsk = bsv = Skv * 2 * d
        dkv = torch.full_like(kv, float("nan"))
        dk, dv = dkv[:, :d], dkv[:, d:]
        dq = None if kind == "shared_q" else torch.full_like(q, float("nan"))
    dout = (torch.randn(B * Sq, d, device=dev) * 0.5).to(bf)
    out = torch.empty(B * Sq, d, device=dev, dtype=bf)
    mu8 = mask.to(torch.uint8).contiguous() if mask is not None else None
    kw = dict(B=B, Sq=Sq, Skv=Skv, H=H, head_dim=hd, bsq=bsq, bsk=bsk, bsv=bsv, bso=Sq * d, scale=scale, mask=mu8,
              mask_bs=Sq * Skv if mask is not None else 0, mask_qs=Skv if mask is not None else 0, causal=kind == "causal")
    ops.attention_fwd_generic(q, k, v, out, **kw)
    dq32 = torch.zeros(Sq, d, device=dev) if kind == "shared_q" else None
    ops.attention_bwd_generic(q, k, v, dout, dk, dv, dq=dq, dq_f32=dq32, **kw)
    # reference
    qf = q.float().clone().requires_grad_(True)
    kf = k.float().clone().requires_grad_(True)
    vf = v.float().clone().requires_grad_(True)
    qh = (qf.view(1, Sq, H, hd).expand(B, Sq, H, hd) if kind == "shared_q" else qf.view(B, Sq, H, hd)).transpose(1, 2)
    kh, vh = kf.view(B, Skv, H, hd).transpose(1, 2), vf.view(B, Skv, H, hd).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) * scale
    if kind == "causal":
        s = s + torch.full((Sq, Skv), float("-inf"), device=dev).triu(1)
    if mask is not None:
        s = s.masked_fill(~mask[:, None], float("-inf"))
    p = torch.softmax(s, -1)
    p = torch.nan_to_num(p, nan=0.0)          # fully masked row -> zeros (the kernels' convention)
    ref = (p @ vh).transpose(1, 2).reshape(B * Sq, d)
    assert _rel(out, ref) < 1e-2
    ref.backward(dout.float())
    assert torch.isfinite(dk.float()).all() and torch.isfinite(dv.float()).all()
    assert _rel(dk, kf.grad) < 1e-2 and _rel(dv, vf.grad) < 1e-2
    if kind == "shared_q":
        assert _rel(dq32, qf.grad) < 1e-2
    else:
        assert torch.isfinite(dq.float()).all()
        assert _rel(dq, qf.grad) < 1e-2


# ---------------------------------------------------------------------------------------------------------------------
# whole model: every parameter gradient of CoCaModel + the captioning head against autograd over the fp32 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _cfg(kw):
    cfg = dict(kw)
    cfg.setdefault("pad_idx", 0)
    return cfg


def coca_grad_parity(dev, name, tag, with_contrastive=True, bar=5e-2):
    """loss = captioning cross-entropy + <w_i, image_pooled> + <w_t, text_pooled> (fixed random w: exercises both
    contrastive branches independently of the loss kernels) [+ the contrastive loss itself when with_contrastive]."""
    import coca_cases as CC
    from oracle import coca_oracle as CO
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining, TrainHidden
    from multimodal_b200.engine_coca_train import linear_cross_entropy

    F = torch.nn.functional
    m = CC.build(lambda **kw: coca_for_pretraining(**kw), name).to(dev).train()
    cfg = _cfg(CC.CASES[name]["kwargs"])
    cpu_inp = CC.inputs(name)
    inp = {k: v.to(dev) for k, v in cpu_inp.items()}
    # the oracle builds its masks on the CPU: it runs there (fp32), the drop-in on `dev`
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    images, texts = cpu_inp["images"], cpu_inp["texts"]

    # ---- oracle with autograd intact (CO.coca_forward detaches: same composition from its parts)
    x = CO.vision_encoder(images, sd, cfg)
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
    cap_ref = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), texts[:, 1:].reshape(-1), ignore_index=cfg["pad_idx"])
    gen = torch.Generator().manual_seed(21)
    wi, wt = torch.randn(img.shape, generator=gen), torch.randn(txt.shape, generator=gen)
    total_ref = cap_ref + (wi * img).sum() + (wt * txt).sum()
    if with_contrastive:
        a = img.squeeze(1) if img.dim() == 3 else img
        T = torch.exp(sd["contrastive_loss.logit_scale"].clamp(0.0, 4.6052))
        lab = torch.arange(a.shape[0])
        total_ref = total_ref + (F.cross_entropy(a @ txt.t() * T, lab) + F.cross_entropy(txt @ a.t() * T, lab)) / 2
    total_ref.backward()

    # ---- the drop-in under autograd
    images, texts, wi, wt = inp["images"], inp["texts"], wi.to(dev), wt.to(dev)
    outs = m.model._forward_impl(images, texts, None, want_logits=False)
    assert isinstance(outs.multimodal_embeddings, TrainHidden)
    cap_loss = linear_cross_entropy(outs.multimodal_embeddings.hidden, outs.multimodal_embeddings.projection,
                                    texts[:, 1:].contiguous(), m.caption_loss.ignore_index)
    assert abs(cap_loss.item() - cap_ref.item()) < 2e-2 * max(1.0, abs(cap_ref.item())), (cap_loss.item(), cap_ref.item())
    total = cap_loss + (wi * outs.image_pooled_output).sum() + (wt * outs.text_pooled_output).sum()
    if with_contrastive:
        io = outs.image_pooled_output
        total = total + m.contrastive_loss(io.squeeze(1) if io.dim() == 3 else io, outs.text_pooled_output)
    assert abs(total.item() - total_ref.item()) < 3e-2 * max(1.0, abs(total_ref.item())), (total.item(), total_ref.item())
    total.backward()

    rows = []
    for k, p in m.named_parameters():
        ref = sd[k].grad
        if ref is None or ref.norm().item() == 0.0:
            assert p.grad is None or p.grad.abs().max().item() < 1e-5, k
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        if k.endswith("k_proj.bias"):      # exactly zero in exact arithmetic (softmax shift invariance)
            continue
        if k == "model.text_decoder.embeddings.token_embeddings.weight" and m.model.text_decoder.embeddings.token_embeddings.padding_idx is not None:
            pad = m.model.text_decoder.embeddings.token_embeddings.padding_idx
            assert p.grad[pad].abs().max().item() == 0.0
            ref = ref.clone()
            ref[pad] = 0
        rows.append((k, _rel(p.grad.cpu(), ref)))
    report = [f"{tag}: total ours {total.item():.6f} oracle {total_ref.item():.6f}; captioning {cap_loss.item():.6f} / {cap_ref.item():.6f}"]
    errs = sorted(r[1] for r in rows)
    report.append(f"relative-L2 gradient error over {len(rows)} parameter tensors: median {errs[len(errs) // 2]:.3e} max {errs[-1]:.3e}")
    report += [f"{k:80s} rel {a:.3e}" for k, a in sorted(rows, key=lambda r: -r[1])[:20]]
    print("\n".join(report))
    assert len(rows) > 40
    for k, a in rows:
        assert a < bar, (k, a)
    return m


@pytest.mark.parametrize("name", ["coca_small", "coca_parallel"])
def test_coca_gradients_against_fp32_oracle(dev, name):
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        coca_grad_parity(dev, name, name, with_contrastive=(name == "coca_parallel"), bar=4e-2)   # measured max 1.8e-2
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_coca_for_pretraining_step_trains(dev):
    """CoCaForPretraining.forward under autograd: both losses carry a graph, three SGD steps lower their sum."""
    import coca_cases as CC
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining

    name = "coca_parallel"     # B = 8: the contrastive loss runs on its exact-fp32 SIMT path
    m = CC.build(lambda **kw: coca_for_pretraining(**kw), name).to(dev).train()
    inp = {k: v.to(dev) for k, v in CC.inputs(name).items()}
    opt = torch.optim.SGD(m.parameters(), lr=0.02)
    hist = []
    for _ in range(4):
        opt.zero_grad(set_to_none=True)
        out = m(inp["images"], inp["texts"])
        total = out["contrastive"] + out["captioning"]
        assert total.requires_grad and torch.isfinite(total)
        total.backward()
        hist.append(total.item())
        opt.step()
    print("CoCaForPretraining total loss over SGD steps:", hist)
    assert hist[-1] < hist[0], hist


# ---------------------------------------------------------------------------------------------------------------------
# standalone pre-norm TransformerEncoderLayer / TransformerEncoder under autograd
# ---------------------------------------------------------------------------------------------------------------------
def _encoder_ref(mod, x, mask):
    """fp32 torch restatement of modules/layers/transformer.py:95-111, 216-259 (pre-norm) on the module's parameters."""
    F = torch.nn.functional
    layers = list(mod.layer) if hasattr(mod, "layer") else [mod]
    for layer in layers:
        at, mlp = layer.attention, layer.feedforward.model
        B, S, d = x.shape
        H = at.num_heads
        h = F.layer_norm(x, (d,), layer.attention_layernorm.weight, layer.attention_layernorm.bias, layer.attention_layernorm.eps)
        q, k, v = (t.view(B, S, H, d // H).transpose(1, 2) for t in F.linear(h, at.input_proj.weight, at.input_proj.bias).chunk(3, -1))
        s = q @ k.transpose(-1, -2) / math.sqrt(d // H)
        if mask is not None:
            s = s.masked_fill(~mask.view(B, 1, S, S), float("-inf"))
        a = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, S, d)
        x = x + F.linear(a, at.output_proj.weight, at.output_proj.bias)
        h = F.layer_norm(x, (d,), layer.feedforward_layernorm.weight, layer.feedforward_layernorm.bias, layer.feedforward_layernorm.eps)
        x = x + F.linear(F.gelu(F.linear(h, mlp[0].weight, mlp[0].bias)), mlp[-1].weight, mlp[-1].bias)
    fln = getattr(mod, "final_layer_norm", None)
    if fln is not None:
        x = F.layer_norm(x, (x.shape[-1],), fln.weight, fln.bias, fln.eps)
    return x


def standalone_layers_grad_parity(dev, masked):
    import copy

    from multimodal_b200.modules.layers.transformer import TransformerEncoder

    torch.manual_seed(0)
    m = TransformerEncoder(n_layer=2, d_model=128, n_head=2, dim_feedforward=256, activation=torch.nn.GELU,
                           layer_norm_eps=1e-5, norm_first=True, final_layer_norm_eps=1e-5).to(dev)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.05 * torch.randn_like(p))
    ref_m = copy.deepcopy(m)
    B, S = 3, 19
    x = torch.randn(B, S, 128, device=dev)
    mask = None
    if masked:
        mask = torch.rand(B, S, S, device=dev) < 0.7
        mask[:, :, 0] = True
    w = torch.randn(B, S, 128, device=dev) / 11
    xr = x.clone().requires_grad_(True)
    (_encoder_ref(ref_m, xr, mask) * w).sum().backward()
    xo = x.clone().requires_grad_(True)
    out = m(xo, mask, return_hidden_states=True)
    assert out.last_hidden_state.requires_grad and len(out.hidden_states) == 3
    (out.last_hidden_state * w).sum().backward()
    assert _rel(xo.grad, xr.grad) < 5e-2
    for (k, p), (_, q) in zip(m.named_parameters(), ref_m.named_parameters()):
        assert p.grad is not None, k
        assert _rel(p.grad, q.grad) < 5e-2, (k, _rel(p.grad, q.grad))
    # a single layer called on its own
    layer, ref_l = m.layer[0], ref_m.layer[0]
    for p in list(layer.parameters()) + list(ref_l.parameters()):
        p.grad = None
    xr = x.clone().requires_grad_(True)
    (_encoder_ref(ref_l, xr, mask) * w).sum().backward()
    xo = x.clone().requires_grad_(True)
    (layer(xo, mask) * w).sum().backward()
    assert _rel(xo.grad, xr.grad) < 5e-2
    assert _rel(layer.feedforward.model[0].weight.grad, ref_l.feedforward.model[0].weight.grad) < 5e-2


@pytest.mark.parametrize("masked", [False, True])
def test_standalone_encoder_layers_train(dev, masked):
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        standalone_layers_grad_parity(dev, masked)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
