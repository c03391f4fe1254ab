"""Cases of the key / value cache golden (tests/golden/decoder_cache_golden.pt): MultiHeadAttentionWithCache,
TransformerDecoderLayer and TransformerDecoder of torchmultimodal/modules/layers/{multi_head_attention,transformer}.py at
the head widths the tensor-core kernels take (head_dim 64 / 96 / 128; the reference's own tests use head_dim 2-4).

`build(ns, name)` creates the module from a namespace holding the three classes (the reference's or this package's) and
fills every parameter from a generator seeded by the case, in state-dict key order, so both sides get identical weights.
`inputs(name)` makes the case's inputs; `run(mod, name, inp)` calls the module the way the reference's tests do and
returns a flat dict of result tensors.
"""
import types

import torch
from torch import nn

# LayerNorm widths are multiples of 128 (the add + LayerNorm kernel)
D64, D96, D128 = dict(d=128, H=2), dict(d=384, H=4), dict(d=256, H=2)

CASES = {
    # MultiHeadAttentionWithCache(dim_q, dim_kv, num_heads, add_bias)
    "mha_self_past_d64": dict(kind="mha", **D64, dim_kv=128, B=2, Sq=3, Sk=3, Sp=5, same="qkv", use_cache=True),
    "mha_cross_d96": dict(kind="mha", **D96, dim_kv=80, B=2, Sq=4, Sk=7, Sp=0, same="kv", use_cache=False),
    "mha_nobias_d128": dict(kind="mha", **D128, dim_kv=256, B=2, Sq=5, Sk=6, Sp=0, same="", add_bias=False,
                            use_cache=True),
    "mha_mask2d_past_d64": dict(kind="mha", **D64, dim_kv=128, B=2, Sq=4, Sk=4, Sp=6, same="qkv", mask="2d",
                                use_cache=True, past_bf16=True),
    "mha_mask4d_cross_d96": dict(kind="mha", **D96, dim_kv=384, B=2, Sq=3, Sk=9, Sp=0, same="kv", mask="4d",
                                 use_cache=False),
    "mha_causal_d128": dict(kind="mha", **D128, dim_kv=256, B=2, Sq=3, Sk=9, Sp=0, same="kv", causal=True,
                            use_cache=False),
    # TransformerDecoderLayer(d_model, n_head, dim_feedforward, ..., norm_first, use_cross_attention, dim_kv)
    "layer_pre_cross_d64": dict(kind="layer", **D64, ff=256, norm_first=True, cross=True, dim_kv=96, B=2, S=4, Sp=3,
                                S_enc=6, mask=True),
    "layer_pre_nocross_d96": dict(kind="layer", **D96, ff=768, norm_first=True, cross=False, dim_kv=None, B=2, S=3,
                                  Sp=4, S_enc=0, mask=False),
    "layer_pre_cross_noenc_d64": dict(kind="layer", **D64, ff=256, norm_first=True, cross=True, dim_kv=None, B=2, S=3,
                                      Sp=2, S_enc=0, mask=False),
    "layer_post_cross_d128": dict(kind="layer", **D128, ff=512, norm_first=False, cross=True, dim_kv=128, B=2, S=4,
                                  Sp=3, S_enc=5, mask=True),
    "layer_post_nocross_d64": dict(kind="layer", **D64, ff=256, norm_first=False, cross=False, dim_kv=None, B=2, S=2,
                                   Sp=5, S_enc=0, mask=False),
    # TransformerDecoder: 2 layers + final LayerNorm, hidden states and caches returned, cross_attention_mask dropped
    "decoder_2l_d96": dict(kind="decoder", **D96, ff=768, norm_first=True, cross=True, dim_kv=128, B=2, S=3, Sp=4,
                           S_enc=6, n_layer=2, final_eps=1e-5),
}


def namespace(mha_mod, transformer_mod):
    return types.SimpleNamespace(MHA=mha_mod.MultiHeadAttentionWithCache, Layer=transformer_mod.TransformerDecoderLayer,
                                 Decoder=transformer_mod.TransformerDecoder)


def _fill(mod: nn.Module, seed: int) -> None:
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(mod.named_parameters()):
            r = torch.randn(p.shape, generator=g)
            if p.dim() == 2:
                p.copy_(r / p.shape[1] ** 0.5)
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1 + 0.1 * r)
            else:
                p.copy_(0.1 * r)


def build(ns, name):
    c = CASES[name]
    torch.manual_seed(0)
    if c["kind"] == "mha":
        m = ns.MHA(c["d"], c["dim_kv"], c["H"], add_bias=c.get("add_bias", True))
    elif c["kind"] == "layer":
        m = ns.Layer(c["d"], c["H"], c["ff"], activation=nn.GELU, norm_first=c["norm_first"],
                     use_cross_attention=c["cross"], dim_kv=c["dim_kv"])
    else:
        m = ns.Decoder(c["n_layer"], c["d"], c["H"], c["ff"], activation=nn.GELU, norm_first=c["norm_first"],
                       use_cross_attention=c["cross"], dim_kv=c["dim_kv"], final_layer_norm_eps=c["final_eps"])
    _fill(m, sum(map(ord, name)))
    return m.eval()


def _past(g, B, H, Sp, hd, bf16=False):
    k, v = torch.randn(B, H, Sp, hd, generator=g), torch.randn(B, H, Sp, hd, generator=g)
    return (k.bfloat16(), v.bfloat16()) if bf16 else (k, v)


def _causal_mask(S, Sp):
    """[S, Sp + S]: query row i (position Sp + i) sees keys j <= Sp + i."""
    return torch.arange(Sp + S)[None, :] <= (Sp + torch.arange(S))[:, None]


def inputs(name):
    c = CASES[name]
    g = torch.Generator().manual_seed(1000 + sum(map(ord, name)))
    B, d, H = c["B"], c["d"], c["H"]
    hd = d // H
    if c["kind"] == "mha":
        Sq, Sk, Sp = c["Sq"], c["Sk"], c["Sp"]
        q = torch.randn(B, Sq, d, generator=g)
        if c["same"] == "qkv":
            k = v = q
        elif c["same"] == "kv":
            k = v = torch.randn(B, Sk, c["dim_kv"], generator=g)
        else:
            k, v = torch.randn(B, Sk, c["dim_kv"], generator=g), torch.randn(B, Sk, c["dim_kv"], generator=g)
        inp = dict(query=q, key=k, value=v)
        if Sp:
            inp["past_key_value"] = _past(g, B, H, Sp, hd, c.get("past_bf16", False))
        mk = c.get("mask")
        if mk == "2d":   # [Sq, Skv]: causal over the cache, plus a few extra holes; every row keeps a key
            m = _causal_mask(Sq, Sp)
            m[1, 0] = m[2, 3] = False
            inp["attn_mask"] = m
        elif mk == "4d":  # [B, 1, Sq, Skv] random, key 0 always visible
            m = torch.rand(B, 1, Sq, Sk, generator=g) > 0.4
            m[..., 0] = True
            inp["attn_mask"] = m
        if c.get("causal"):
            inp["is_causal"] = True
        return inp
    S, Sp = c["S"], c["Sp"]
    inp = dict(hidden_states=torch.randn(B, S, d, generator=g))
    if c["S_enc"]:
        inp["encoder_hidden_states"] = torch.randn(B, c["S_enc"], c["dim_kv"] or d, generator=g)
    if c["kind"] == "layer":
        inp["past_key_value"] = _past(g, B, H, Sp, hd)
        if c["mask"]:
            inp["attention_mask"] = _causal_mask(S, Sp)
        inp["use_cache"] = True
        return inp
    inp["past_key_values"] = [_past(g, B, H, Sp, hd) for _ in range(c["n_layer"])]
    inp["attention_mask"] = _causal_mask(S, Sp)[None, None].expand(B, 1, S, Sp + S)
    inp["cross_attention_mask"] = torch.zeros(B, 1, S, c["S_enc"], dtype=torch.bool)   # dropped by TransformerDecoder
    inp["use_cache"] = True
    inp["return_hidden_states"] = True
    return inp


def to(inp, device):
    def mv(x):
        if torch.is_tensor(x):
            return x.to(device)
        if isinstance(x, (list, tuple)):
            return type(x)(mv(y) for y in x)
        return x
    out = {k: mv(v) for k, v in inp.items()}
    # keep the identity of shared inputs (query is key is value selects the packed projections)
    for a, b in (("key", "query"), ("value", "key")):
        if a in inp and inp[a] is inp[b]:
            out[a] = out[b]
    return out


def run(mod, name, inp):
    c = CASES[name]
    if c["kind"] == "mha":
        r = mod(inp["query"], inp["key"], inp["value"], attn_mask=inp.get("attn_mask"),
                past_key_value=inp.get("past_key_value"), is_causal=inp.get("is_causal", False),
                use_cache=c["use_cache"])
        if c["use_cache"]:
            return {"out": r.attn_output, "k": r.past_key_value[0], "v": r.past_key_value[1]}
        return {"out": r}
    if c["kind"] == "layer":
        out, kv = mod(**inp)
        return {"out": out, "k": kv[0], "v": kv[1]}
    o = mod(**inp)
    res = {"out": o.last_hidden_state}
    for i, h in enumerate(o.hidden_states):
        res[f"hidden{i}"] = h
    for i, (k, v) in enumerate(o.current_key_values):
        res[f"k{i}"], res[f"v{i}"] = k, v
    return res
