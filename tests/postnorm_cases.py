"""Shared definition of the post-norm cases at the reference defaults (`TransformerEncoderLayer(d, H, ff)` /
`TransformerEncoder(n, d, H, ff, ...)`: ReLU, norm_first=False, layer_norm_eps 1e-12) and an fp32 restatement of
those layers that takes the stochastic-depth noise as an input.  Used by tests/golden/make_postnorm_golden.py (on the
unmodified reference), tests/test_postnorm_train_cpu.py and tests/test_gpu_postnorm_train.py."""
import torch
import torch.nn.functional as F

import drop_path_cases as DP

D, HEADS, FF = 128, 2, 256      # head_dim 64

# kind, encoder layers, final LayerNorm eps, bool [B, 1, S, S] mask, drop_path_rate (train mode), batch, length, seed
CASES = {
    "layer": dict(kind="layer", n_layer=1, final_eps=None, masked=False, rate=None, B=4, S=24, seed=71),
    "layer_mask": dict(kind="layer", n_layer=1, final_eps=None, masked=True, rate=None, B=4, S=24, seed=72),
    "encoder": dict(kind="encoder", n_layer=3, final_eps=None, masked=False, rate=None, B=3, S=20, seed=73),
    "encoder_final_ln_mask": dict(kind="encoder", n_layer=3, final_eps=1e-12, masked=True, rate=None, B=3, S=20,
                                  seed=74),
    "encoder_drop": dict(kind="encoder", n_layer=3, final_eps=1e-12, masked=False, rate=0.5, B=8, S=12, seed=75),
}


def build(layer_cls, encoder_cls, name):
    """The reference's or the drop-in's module at its defaults, weights perturbed by a seeded draw."""
    c = CASES[name]
    torch.manual_seed(0)
    if c["kind"] == "layer":
        m = layer_cls(D, HEADS, FF, drop_path_rate=c["rate"])
    else:
        m = encoder_cls(c["n_layer"], D, HEADS, FF, final_layer_norm_eps=c["final_eps"], drop_path_rate=c["rate"])
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    return m.train() if c["rate"] is not None else m.eval()


def inputs(name):
    """(hidden_states [B, S, D], bool [B, 1, S, S] mask (True = attend; the reference broadcasts it over the heads) or
    None)."""
    c = CASES[name]
    g = torch.Generator().manual_seed(c["seed"])
    x = torch.randn(c["B"], c["S"], D, generator=g)
    mask = None
    if c["masked"]:
        mask = torch.rand(c["B"], c["S"], c["S"], generator=g) < 0.7
        mask[:, :, 0] = True
        mask = mask[:, None]
    return x, mask


def layers_of(m):
    return [m] if hasattr(m, "attention") else list(m.layer)


def ref_layer(layer, x, mask=None, s_a=None, s_f=None):
    """A post-norm TransformerEncoderLayer (reference transformer.py:113-128) in fp32 on the module's own parameters:
    out = LN2(x1 + s_f FF(x1)), x1 = LN1(x + s_a Attn(x))."""
    at, mlp = layer.attention, layer.feedforward.model
    B, S, d = x.shape
    H = at.num_heads
    q, k, v = F.linear(x, at.input_proj.weight, at.input_proj.bias).chunk(3, dim=-1)
    q, k, v = (t.reshape(B, S, H, d // H).transpose(1, 2) for t in (q, k, v))
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
    a = F.linear(o.transpose(1, 2).reshape(B, S, d), at.output_proj.weight, at.output_proj.bias)
    if s_a is not None:
        a = a * s_a.view(-1, 1, 1)
    ln1, ln2 = layer.attention_layernorm, layer.feedforward_layernorm
    x1 = F.layer_norm(x + a, (d,), ln1.weight, ln1.bias, ln1.eps)
    h = F.linear(mlp[1](F.linear(x1, mlp[0].weight, mlp[0].bias)), mlp[-1].weight, mlp[-1].bias)
    if s_f is not None:
        h = h * s_f.view(-1, 1, 1)
    return F.layer_norm(x1 + h, (d,), ln2.weight, ln2.bias, ln2.eps)


def ref_forward(m, x, mask=None, scales=None):
    """(output, hidden_states) of the module `m` (layer or encoder) in fp32: hidden_states are x and each layer's
    output, the last one before the final LayerNorm."""
    hidden = [x]
    for i, layer in enumerate(layers_of(m)):
        s_a, s_f = scales[i] if scales is not None else (None, None)
        x = ref_layer(layer, x, mask, s_a, s_f)
        hidden.append(x)
    fln = getattr(m, "final_layer_norm", None)
    if fln is not None:
        x = F.layer_norm(x, (x.shape[-1],), fln.weight, fln.bias, fln.eps)
    return x, hidden


# ReLU' is a step.  The bf16-operand FC1 pre-activation differs from the fp32 one by about 2^-9 of its scale, so about
# 1e-3 of its entries lie on the other side of 0 than in fp32, and each such entry moves its dPRE by a whole dY.W2
# value: the FC1 gradients carry a relative L2 error near sqrt(1e-3) = 3e-2 against fp32 autograd whatever the
# schedule (measured at the BERT-base shapes: 4.1e-2, cosine 0.9992).  Bars of the ReLU gradients:
SMALL_RELU_L2_BAR = 8e-2        # relative L2 at width 128 over ~100 tokens, where one straddle moves more of a row
BERT_RELU_FC1_L2_BAR = 6e-2     # relative L2 of the FC1 gradients at the BERT-base shapes (cosine >= 0.995 as well)
RELU_MAX_BAR = 1e-1             # relative max of the other gradients at width 128, which inherit the straddles above


def rel_max(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-30)).item()


def grad_errors(grads, ref, bar=5e-2, l2_bar=4e-2, cos_bar=0.995, relu=False):
    """{name: error} of the gradients outside their bar against fp32 autograd: relative max error < `bar`, except for
    the FC1 weight and bias under ReLU (and every gradient with `relu`), held to relative L2 < `l2_bar` and cosine >=
    `cos_bar`.  ReLU' is a step: where
    the bf16-operand pre-activation and the fp32 one straddle 0 (about 1 in 1000 entries), that token's whole
    contribution to its FC1 row moves, so the worst entry of those gradients is not a measure of the schedule."""
    bad = {}
    for k, g in grads.items():
        r = ref[k]
        if relu or ".feedforward.model.0." in "." + k:
            cos = torch.nn.functional.cosine_similarity(g.flatten().double(), r.flatten().double(), dim=0).item()
            l2 = ((g.double() - r.double()).norm() / r.double().norm().clamp_min(1e-30)).item()
            if l2 >= l2_bar or cos < cos_bar:
                bad[k] = (l2, cos)
        elif rel_max(g, r) >= bar:
            bad[k] = rel_max(g, r)
    return bad


upstream = DP.upstream
sample, sample_errors = DP.sample, DP.sample_errors
N_GRAD, N_OUT = DP.N_GRAD, DP.N_OUT
