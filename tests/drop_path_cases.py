"""Shared definition of the stochastic-depth cases (`drop_path_rate` / `vision_drop_path_rate`), a recorder of the noise
the reference's `StochasticDepth` calls draw, and an fp32 oracle of the encoder layers that takes the per-(layer, branch)
noise as an input.  Used by tests/golden/make_drop_path_golden.py (on the unmodified reference),
tests/test_drop_path_cpu.py and tests/test_gpu_drop_path.py."""
import contextlib
import functools
from unittest import mock

import torch
import torch.nn.functional as F
from torch import nn
from torch.overrides import TorchFunctionMode

import coca_cases as CC
import patch_drop_cases as PD
from oracle import coca_oracle as CO

D, HEADS, FF, EPS = 128, 2, 256, 1e-5      # head_dim 64

# vision_transformer in training mode: builder kwargs, batch, forward seed
VIT = {
    "vit_cls": dict(kw=dict(patch_size=4, hidden_dim=D, dim_feedforward=FF, n_layer=3, n_head=HEADS, image_size=16,
                            layer_norm_eps=EPS, final_layer_norm_eps=EPS, drop_path_rate=0.5), B=8, seed=51),
    # CoCa's ViT form: no CLS token, no final LayerNorm (the last MLP branch's gradient enters through the scaled cast)
    "vit_nocls": dict(kw=dict(patch_size=4, hidden_dim=D, dim_feedforward=FF, n_layer=4, n_head=HEADS, image_size=16,
                              layer_norm_eps=EPS, final_layer_norm_eps=None, include_cls_embed=False,
                              drop_path_rate=0.5), B=10, seed=52),
    "vit_patch_drop": dict(kw=dict(patch_size=4, hidden_dim=D, dim_feedforward=FF, n_layer=3, n_head=HEADS,
                                   image_size=16, layer_norm_eps=EPS, final_layer_norm_eps=EPS, drop_path_rate=0.5,
                                   patch_drop_rate=0.5), B=8, seed=53),
}

# standalone layers: kind, norm_first, n_layer (encoder), grad mode, batch, sequence length, forward seed
LAYERS = {
    "layer": dict(kind="layer", norm_first=True, n_layer=1, grad=True, B=8, S=10, seed=61),
    "postnorm_nograd": dict(kind="encoder", norm_first=False, n_layer=3, grad=False, B=8, S=12, seed=62),
    "one_layer": dict(kind="encoder", norm_first=True, n_layer=1, grad=True, B=8, S=10, seed=63),
}
RATE = 0.5


def _perturb(m):
    g = torch.Generator().manual_seed(13)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    return m.train()


def build_vit(builder, name):
    """`builder` is the reference's or the drop-in's `vision_transformer`."""
    torch.manual_seed(0)
    return _perturb(builder(**VIT[name]["kw"]))


def vit_inputs(name):
    c = VIT[name]
    g = torch.Generator().manual_seed(5)
    images = torch.randn(c["B"], 3, 16, 16, generator=g)
    return images, None


def build_layers(layer_cls, encoder_cls, name):
    c = LAYERS[name]
    torch.manual_seed(0)
    if c["kind"] == "layer":
        m = layer_cls(D, HEADS, FF, activation=nn.GELU, layer_norm_eps=EPS, norm_first=c["norm_first"],
                      drop_path_rate=RATE)
    else:
        m = encoder_cls(c["n_layer"], D, HEADS, FF, activation=nn.GELU, layer_norm_eps=EPS, norm_first=c["norm_first"],
                        final_layer_norm_eps=EPS, drop_path_rate=RATE)
    return _perturb(m)


def layer_inputs(name):
    c = LAYERS[name]
    return torch.randn(c["B"], c["S"], D, generator=torch.Generator().manual_seed(6))


def upstream(shape, seed=7):
    """The fixed upstream gradient of the golden's backward."""
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


N_GRAD, N_OUT = 64, 256     # sampled entries per gradient / per output tensor in the golden


def _positions(numel, n):
    assert numel >= n, (numel, n)
    return torch.randperm(numel, generator=torch.Generator().manual_seed(numel))[:n]


def sample(tensors, n):
    """The golden keeps tensors small: per tensor its float64 L2 norm, its shape and n entries at positions seeded by
    its size, stacked into one [len(tensors), n] tensor."""
    return {"vals": torch.stack([t.detach().reshape(-1)[_positions(t.numel(), n)].float() for t in tensors]),
            "norms": [t.detach().double().norm().item() for t in tensors], "shapes": [tuple(t.shape) for t in tensors]}


def sample_errors(tensors, rec):
    """Per tensor (max |error| of the sampled entries, their relative L2 error, relative error of the norm) against
    a `sample` record."""
    assert [tuple(t.shape) for t in tensors] == rec["shapes"]
    out = []
    for t, want, norm in zip(tensors, rec["vals"], rec["norms"]):
        got = t.detach().reshape(-1)[_positions(t.numel(), want.numel())].float()
        out.append(((got - want).abs().max().item(), rel(got, want),
                    abs(t.detach().double().norm().item() - norm) / max(norm, 1e-30)))
    return out


def layer_rates(layers):
    """The p of each layer's StochasticDepth (None for a layer without one)."""
    return [getattr(layer.attention_dropout, "p", None) for layer in layers]


class NoiseRecorder(TorchFunctionMode):
    """Records the noise tensors of torchvision's stochastic_depth (created by `bernoulli_`, then scaled in place by
    `div_`) in call order, without touching any random draw."""

    def __init__(self):
        super().__init__()
        self.noise = []

    def __torch_function__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        if func is torch.Tensor.bernoulli_:
            self.noise.append(out)
        return out


def pair_draws(rates, training, draws):
    """Per layer (attention, feed-forward) noise [B] or None from the recorded draws in call order."""
    it = iter(draws)
    out = []
    for p in rates:
        if p is None or p == 0.0 or not training:
            out.append((None, None))
        else:
            out.append((next(it).reshape(-1), next(it).reshape(-1)))
    assert next(it, None) is None
    return out


# ---- fp32 oracle with the per-(layer, branch) noise as an input ---------------------------------------------------------
def _scaled(y, s):
    return y if s is None else y * s.view(-1, 1, 1)


def encoder_layers(x, sd, p, n_layer, n_head, eps, scales=None, norm_first=True):
    """TransformerEncoderLayer forwards (transformer.py:95-129) over sd[p + f".{i}..."], branch i of layer l multiplied
    by scales[l][i] ([B] or None) as StochasticDepth multiplies it."""
    for i in range(n_layer):
        lp = f"{p}.{i}"
        sa, sf = scales[i] if scales is not None else (None, None)

        def attn(h):
            q, k, v = CO._lin(h, sd, lp + ".attention.input_proj").chunk(3, dim=-1)
            return CO._lin(CO._sdpa(q, k, v, n_head), sd, lp + ".attention.output_proj")

        if norm_first:
            x = x + _scaled(attn(CO._ln(x, sd, lp + ".attention_layernorm", eps)), sa)
            x = x + _scaled(CO._mlp(CO._ln(x, sd, lp + ".feedforward_layernorm", eps), sd, lp + ".feedforward"), sf)
        else:
            x = CO._ln(x + _scaled(attn(x), sa), sd, lp + ".attention_layernorm", eps)
            x = CO._ln(x + _scaled(CO._mlp(x, sd, lp + ".feedforward"), sf), sd, lp + ".feedforward_layernorm", eps)
    return x


def vision_encoder(images, sd, cfg, p="model.vision_encoder", keep=None, scales=None):
    """oracle/coca_oracle.vision_encoder on the kept patches `keep` (or all) with the stochastic-depth noise `scales`."""
    x = PD.patch_embed(images, sd, p + ".embeddings.", cfg["vision_patch_size"], keep)
    x = encoder_layers(x, sd, p + ".encoder.layer", cfg["vision_n_layer"], cfg["vision_n_head"],
                       cfg.get("vision_layer_norm_eps", 1e-5), scales)
    if cfg.get("vision_final_layer_norm_eps"):
        x = CO._ln(x, sd, p + ".encoder.final_layer_norm", cfg["vision_final_layer_norm_eps"])
    return x


def vit_cfg(name):
    kw = VIT[name]["kw"]
    return dict(vision_patch_size=kw["patch_size"], vision_n_layer=kw["n_layer"], vision_n_head=kw["n_head"],
                vision_layer_norm_eps=kw["layer_norm_eps"], vision_final_layer_norm_eps=kw["final_layer_norm_eps"])


@contextlib.contextmanager
def oracle_drop_path(keep, scales):
    """Within the block, oracle/coca_oracle's vision encoder runs on the patches `keep` with the noise `scales`."""
    with mock.patch.object(CO, "vision_encoder", functools.partial(vision_encoder, keep=keep, scales=scales)):
        yield


# ---- CoCa with vision_drop_path_rate: gradients against autograd over the oracle fed the same draws ------------------
def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


def check_grads(m, sd, tag, bar=4e-2, cos_bar=0.995, skip=()):
    rows = []
    for k, p in m.named_parameters():
        ref = sd[k].grad
        if ref is None or ref.norm().item() == 0.0:
            assert p.grad is None or p.grad.abs().max().item() < 1e-5, k
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        if k.endswith("k_proj.bias") or k in skip:      # k bias: exactly zero in exact arithmetic
            continue
        g = p.grad.detach().cpu().float()
        cos = F.cosine_similarity(g.reshape(1, -1), ref.reshape(1, -1)).item()
        rows.append((k, rel(g, ref), cos))
    errs = sorted(r[1] for r in rows)
    print(f"{tag}: relative-L2 gradient error over {len(rows)} parameter tensors: median {errs[len(errs) // 2]:.3e} "
          f"max {errs[-1]:.3e}; min cosine {min(r[2] for r in rows):.6f}")
    for k, a, c in rows:
        assert a < bar and c > cos_bar, (k, a, c)
    return rows


def coca_grad_parity(dev, name, rate, patch_rate, seed, bar=4e-2):
    """CoCaForPretraining's losses (captioning + <w, pooled> terms) with vision_drop_path_rate: every parameter
    gradient against autograd over the fp32 oracle fed the kept patches and the noise the package drew."""
    from multimodal_b200.engine_coca_train import linear_cross_entropy
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining
    from multimodal_b200.modules.layers.stochastic_depth import drop_path_scales
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    m = CC.build(lambda **kw: coca_for_pretraining(**kw, vision_drop_path_rate=rate, vision_patch_drop_rate=patch_rate),
                 name).to(dev).train()
    cfg = dict(CC.CASES[name]["kwargs"])
    cfg.setdefault("pad_idx", 0)
    cpu_inp = CC.inputs(name)
    images, texts = cpu_inp["images"], cpu_inp["texts"]
    B = images.shape[0]
    vis = m.model.vision_encoder
    torch.manual_seed(seed)
    keep = patch_keep_indices(vis.embeddings, B, dev)
    keep = keep[0].cpu() if keep is not None else None
    scales = drop_path_scales(vis.encoder.layer, B, dev)
    scales = [tuple(s.cpu() if s is not None else None for s in pair) for pair in scales] if scales else None
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    x = vision_encoder(images, sd, cfg, keep=keep, scales=scales)
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
    check_grads(m, sd, f"{name} drop path {rate} patch {patch_rate}", bar=bar,
                skip=("model.text_decoder.embeddings.token_embeddings.weight",) if pad is not None else ())
    return scales
