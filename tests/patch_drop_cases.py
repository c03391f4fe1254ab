"""Shared definition of the patch-dropping cases (PatchEmbeddings(patch_drop_rate=...), FLIP) and an fp32 oracle of the
patch front end and the ViT that takes the kept patch indices as an input.  Used by tests/golden/make_patch_drop_golden.py
(on the unmodified reference), tests/test_patch_drop_cpu.py and tests/test_gpu_patch_drop.py."""
import contextlib
import functools
from unittest import mock

import torch
import torch.nn.functional as F

import coca_cases as CC
from oracle import coca_oracle as CO

# direct calls of random_masking / random_masking_2d: (kind, x shape, rate(s), seed)
MASKING = {
    "1d_r50": ("1d", (3, 10, 4), 0.5, 11),
    "1d_r75": ("1d", (2, 64, 3), 0.75, 12),
    "1d_odd": ("1d", (4, 7, 2), 0.3, 13),
    "2d": ("2d", (3, 6 * 5, 4), (0.5, 0.4), 14, 6, 5),
}

# PatchEmbeddings in training mode: constructor kwargs, batch, whether an image_patches_mask is passed, forward seed
PATCH_EMBED = {
    "cls_r50": dict(kw=dict(image_size=32, patch_size=4, hidden_size=32, patch_drop_rate=0.5), B=3, mask=False, seed=21),
    "nocls_r75": dict(kw=dict(image_size=32, patch_size=4, hidden_size=32, patch_drop_rate=0.75, include_cls_embed=False),
                      B=2, mask=False, seed=22),
    "cls_mask_r50": dict(kw=dict(image_size=32, patch_size=4, hidden_size=32, patch_drop_rate=0.5, use_image_masking=True),
                         B=3, mask=True, seed=23),
    "nocls_2d": dict(kw=dict(image_size=(32, 24), patch_size=4, hidden_size=16, patch_drop_rate=(0.5, 0.25),
                             include_cls_embed=False), B=2, mask=False, seed=24),
    # 14 x 14 patches + CLS at 0.5: 1 + 98 tokens, the ViT-B/16 shape
    "cls_196_r50": dict(kw=dict(image_size=56, patch_size=4, hidden_size=16, patch_drop_rate=0.5), B=2, mask=False,
                        seed=25),
}

# tiny CoCa (tests/coca_cases.py) in training mode with a vision_patch_drop_rate: case, rate, forward seed
COCA = {
    "coca_small_r50": ("coca_small", 0.5, 31),
    "coca_parallel_2d": ("coca_parallel", (0.5, 0.5), 32),
}


def masking_input(name):
    shape, seed = MASKING[name][1], MASKING[name][3]
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def build_patch_embed(cls, name):
    """PatchEmbeddings (reference or drop-in class `cls`) with every parameter moved off its zero / init value."""
    torch.manual_seed(0)
    pe = cls(**PATCH_EMBED[name]["kw"])
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for p in pe.parameters():
            p.add_(0.2 * torch.randn(p.shape, generator=g))
    return pe.train()


def patch_embed_inputs(name):
    c = PATCH_EMBED[name]
    kw = c["kw"]
    hw = kw["image_size"] if isinstance(kw["image_size"], tuple) else (kw["image_size"],) * 2
    g = torch.Generator().manual_seed(5)
    images = torch.randn(c["B"], 3, *hw, generator=g)
    P = (hw[0] // kw["patch_size"]) * (hw[1] // kw["patch_size"])
    mask = (torch.rand(c["B"], P, generator=g) < 0.4) if c["mask"] else None
    return images, mask


def build_coca(builder, name):
    base, rate, _ = COCA[name]
    return CC.build(functools.partial(builder, vision_patch_drop_rate=rate), base)


def param_checksum(m) -> float:
    return float(sum(p.detach().double().abs().sum() for p in m.parameters()))


# ---- fp32 oracle with the kept patch indices as an input ---------------------------------------------------------------
def patch_embed(images, sd, p, ps, keep, image_patches_mask=None):
    """PatchEmbeddings.forward (patch_embedding.py:104-154) with the tokens of the patches keep[b, :] (int [B, L]):
    conv, mask-token substitution, + pos[off:], gather, then [cls + pos[0] |]."""
    x = F.conv2d(images.float(), sd[p + "conv_projection.weight"], sd[p + "conv_projection.bias"],
                 stride=ps).flatten(2).transpose(1, 2)
    if image_patches_mask is not None and p + "mask_token" in sd:
        w = image_patches_mask.unsqueeze(-1).float()
        x = x * (1 - w) + sd[p + "mask_token"] * w
    pos = sd[p + "position_embeddings"]
    has_cls = p + "cls_token" in sd
    x = x + (pos[:, 1:] if has_cls else pos)
    if keep is not None:
        x = torch.gather(x, 1, keep.long().unsqueeze(-1).expand(-1, -1, x.shape[-1]))
    if has_cls:
        x = torch.cat([(sd[p + "cls_token"] + pos[:, :1]).expand(x.shape[0], -1, -1), x], 1)
    return x


def vision_encoder(images, sd, cfg, p="model.vision_encoder", keep=None):
    """oracle/coca_oracle.vision_encoder on the kept patches only."""
    x = patch_embed(images, sd, p + ".embeddings.", cfg["vision_patch_size"], keep)
    eps, H = cfg.get("vision_layer_norm_eps", 1e-5), cfg["vision_n_head"]
    for i in range(cfg["vision_n_layer"]):
        lp = f"{p}.encoder.layer.{i}"
        h = CO._ln(x, sd, lp + ".attention_layernorm", eps)
        q, k, v = CO._lin(h, sd, lp + ".attention.input_proj").chunk(3, dim=-1)
        x = x + CO._lin(CO._sdpa(q, k, v, H), sd, lp + ".attention.output_proj")
        x = x + CO._mlp(CO._ln(x, sd, lp + ".feedforward_layernorm", eps), sd, lp + ".feedforward")
    if cfg.get("vision_final_layer_norm_eps"):
        x = CO._ln(x, sd, p + ".encoder.final_layer_norm", cfg["vision_final_layer_norm_eps"])
    return x


@contextlib.contextmanager
def oracle_keeps(keep):
    """Within the block, oracle/coca_oracle's CoCa forward runs its vision encoder on the patches `keep`."""
    with mock.patch.object(CO, "vision_encoder", functools.partial(vision_encoder, keep=keep)):
        yield
