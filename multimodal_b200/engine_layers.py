"""Standalone (single-module) forward runtimes for the layer types of the hot path, so that the modules the reference
exposes — and tests — on their own are callable outside an encoder:

  modules/layers/multi_head_attention.py:19-80   MultiHeadSelfAttention
  modules/layers/transformer.py:31-154           TransformerEncoderLayer (pre- and post-norm), :157-259 TransformerEncoder
  modules/layers/patch_embedding.py:25-157       PatchEmbeddings
  modules/layers/mlp.py:13-66                    MLP ([Linear, activation, Linear] form)

They launch exactly the kernels the fused encoder schedules launch (wgmma GEMMs with bias / activation epilogues,
tensor-core attention, the add+LayerNorm kernel); nothing is computed by PyTorch.  `TransformerEncoderLayer` /
`TransformerEncoder` run on one runtime per module in both grad modes, `infer` under torch.no_grad(): pre-norm layers on
`EncoderLayersRuntime` (`engine.ModuleStack`: the CLIP towers' fused forward / backward schedule), post-norm layers (the
reference default) on `PostNormLayersRuntime`, a schedule of their own.  The other standalone modules compute forward
values only, and asking them for an autograd graph raises instead of returning detached tensors.
  modules/layers/multi_head_attention.py:83-180  MultiHeadAttentionWithCache (key / value cache, cross-attention)
  modules/layers/transformer.py:262-657          TransformerDecoderLayer (pre- and post-norm), TransformerDecoder

Shape limits are those of the kernels: head_dim 64 (fused attention; 96 / 128 and arbitrary boolean masks go through
the general kernels), feature sizes multiples of 8, 3-channel images.  Any sequence length: the general kernels keep a
head resident in shared memory while it fits and stream K / V through it beyond (attention_generic_stream.cu).
Autoregressive decoding (queries of at most 16 rows over a key / value cache) runs the split-KV decode kernel
(attention_decode.cu); the decoders compute forward values only (their training runs inside the CoCa runtimes).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
from torch import nn

from . import ops
from ._lib import MMBError
from .engine import ModuleStack, ParamStore, Workspace, _Shadows, act_code, as_f32, patch_embed_fwd, run, scaled
from .modules.layers.stochastic_depth import drop_path_scales


def forward_only_guard(mod: nn.Module, what: str) -> None:
    if torch.is_grad_enabled() and any(p.requires_grad for p in mod.parameters()):
        raise MMBError(f"{what} (multimodal_b200) computes forward values only when called on its own — its backward "
                       "exists inside the CLIP towers' fused schedule.  Call it under torch.no_grad().")


def _wants_graph(mod: nn.Module, x: torch.Tensor) -> bool:
    return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in mod.parameters()))


def _cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise MMBError(f"{what}: expected a CUDA tensor (multimodal_b200 has no CPU path), got device {t.device}")


class _Rt:
    """Per-module scratch: reused workspace + bf16 weight shadows (re-cast when a parameter changes)."""

    def __init__(self, device):
        self.ws, self.sh, self.device = Workspace(device), _Shadows(device), device


def _rt(mod: nn.Module, device) -> _Rt:
    rt = getattr(mod, "_mmb_rt", None)
    if rt is None or rt.device != device:
        rt = _Rt(device)
        object.__setattr__(mod, "_mmb_rt", rt)   # not a submodule / buffer: keeps the state dict untouched
    return rt


def _bool_mask_u8(mask: Optional[torch.Tensor], B: int, S: int, what: str) -> Optional[torch.Tensor]:
    """bool [B, S, S] or [B, 1, S, S] (True = attend) -> uint8 [B, S, S]; float (additive) masks are not supported."""
    if mask is None:
        return None
    if mask.dtype != torch.bool:
        raise NotImplementedError(f"{what}: only boolean attention masks (True = attend) are on the accelerated path")
    if mask.dim() == 4:
        if mask.shape[1] != 1:
            raise NotImplementedError(f"{what}: per-head masks are not on the accelerated path (the head dim must be 1)")
        mask = mask[:, 0]
    if mask.dim() == 2:
        mask = mask[None].expand(B, S, S)
    if tuple(mask.shape) != (B, S, S):
        raise ValueError(f"{what}: attention mask shape {tuple(mask.shape)} does not match [{B}, {S}, {S}]")
    return mask.to(torch.uint8).contiguous()


def _to_bf16_rows(rt: _Rt, x: torch.Tensor, name: str) -> torch.Tensor:
    xf = x.contiguous().float()
    out = rt.ws.get(name, (xf.numel() // xf.shape[-1], xf.shape[-1]), torch.bfloat16)
    ops.cast_bf16(xf.view(-1), out.view(-1))
    return out


# ---------------------------------------------------------------------------------------------------------------------
def mhsa_forward(mod: nn.Module, query: torch.Tensor, attn_mask: Optional[torch.Tensor] = None,
                 is_causal: bool = False) -> torch.Tensor:
    """MultiHeadSelfAttention.forward (multi_head_attention.py:39-80): input_proj -> SDPA -> output_proj."""
    forward_only_guard(mod, "MultiHeadSelfAttention")
    _cuda(query, "MultiHeadSelfAttention")
    B, S, d = query.shape
    H = mod.num_heads
    if d % H or (d // H) not in (64, 96, 128) or d % 8:
        raise MMBError(f"MultiHeadSelfAttention: head_dim {d / H:g} is not supported by the attention kernels (64 / 96 / 128)")
    rt = _rt(mod, query.device)
    bf = torch.bfloat16
    Xb = _to_bf16_rows(rt, query, "mhsa.X")
    QKV = rt.ws.get("mhsa.QKV", (B * S, 3 * d), bf)
    O = rt.ws.get("mhsa.O", (B * S, d), bf)
    ops.gemm(Xb, rt.sh.get("wqkv", [mod.input_proj.weight]), bias=mod.input_proj.bias, out=QKV)
    ops.self_attention(QKV, O, None, B, S, H, d // H, bool(is_causal), 1.0 / math.sqrt(d // H),
                       mask=_bool_mask_u8(attn_mask, B, S, "MultiHeadSelfAttention"))
    out = torch.empty((B * S, d), device=query.device, dtype=torch.float32)
    ops.gemm(O, rt.sh.get("wo", [mod.output_proj.weight]), bias=mod.output_proj.bias, epilogue=ops.EPI_F32, out=out)
    return out.view(B, S, d).to(query.dtype)


def mlp_forward(mod: nn.Module, x: torch.Tensor) -> torch.Tensor:
    """MLP.forward (mlp.py:62-66) for the transformer form [Linear, activation, (Dropout 0), Linear]."""
    forward_only_guard(mod, "MLP")
    _cuda(x, "MLP")
    seq = [m for m in mod.model if not isinstance(m, nn.Dropout)]
    if len(seq) != 3 or not isinstance(seq[0], nn.Linear) or not isinstance(seq[2], nn.Linear):
        raise MMBError("standalone MLP supports the [Linear, activation, Linear] form (one hidden layer, no normalisation)")
    rt = _rt(mod, x.device)
    act = act_code(seq[1])
    Xb = _to_bf16_rows(rt, x, "mlp.X")
    M = Xb.shape[0]
    ff, dout = seq[0].weight.shape[0], seq[2].weight.shape[0]
    PRE = rt.ws.get("mlp.PRE", (M, ff), torch.bfloat16)
    HACT = rt.ws.get("mlp.HACT", (M, ff), torch.bfloat16)
    ops.gemm(Xb, rt.sh.get("w1", [seq[0].weight]), bias=seq[0].bias, epilogue=ops.EPI_BF16_ACT, out=PRE, out2=HACT, act=act)
    out = torch.empty((M, dout), device=x.device, dtype=torch.float32)
    ops.gemm(HACT, rt.sh.get("w2", [seq[2].weight]), bias=seq[2].bias, epilogue=ops.EPI_F32, out=out)
    return out.view(*x.shape[:-1], dout).to(x.dtype)


class EncoderLayersRuntime:
    """A standalone pre-norm `TransformerEncoderLayer` or `TransformerEncoder` (modules/layers/transformer.py:31-259) in
    both grad modes: hidden_states [B, S, d] in, the residual stream after the last layer (and the final LayerNorm, if
    any) out.  `forward(data, diff)` / `backward` run under autograd (engine.run), `infer` under torch.no_grad()."""

    def __init__(self, owner: nn.Module, layers, final_ln: Optional[nn.Module]):
        self.s = ModuleStack(owner, layers, "lyr")
        self.store = self.s.store
        self.final_ln = final_ln

    def _forward(self, x: torch.Tensor, mask_u8, save: Optional[Workspace], hidden: Optional[List[torch.Tensor]]):
        s = self.s
        B, S, d = x.shape
        self.store.refresh()
        if save is None:
            X0 = x.contiguous().float().view(B * S, d)      # only read
        else:
            X0 = torch.empty((B * S, d), device=s.device, dtype=torch.float32)
            X0.view(B, S, d).copy_(x)    # the backward reads it: a copy the caller cannot change
        scales = drop_path_scales(s.layers, B, s.device)   # training with drop_path_rate: once, for all layers
        XM, Y = s.stack.forward(X0, B, S, save, mask3=mask_u8, scales=scales, hidden=hidden)
        XF, LAST = s.finish(XM, Y, B, S, self.final_ln, save, scales)
        if hidden is not None:
            hidden.append(XF.view(B, S, d))
        return LAST if LAST is not None else XF

    def forward(self, data, diff):
        """data: (uint8 [B, S, S] mask or None, the caller's list that receives hidden_states or None)."""
        mask_u8, hidden = data
        (x,) = diff
        save = Workspace(self.s.device)
        out = self._forward(x, mask_u8, save, hidden)
        save.B, save.S = x.shape[:2]
        return (out,), save

    def infer(self, x: torch.Tensor, mask_u8: Optional[torch.Tensor], return_hidden_states: bool = False):
        """-> (output [B, S, d], hidden_states or None), in x's dtype.  hidden_states[0] is x itself; the others are
        fresh tensors, the last one before the final LayerNorm."""
        hidden: Optional[List[torch.Tensor]] = [] if return_hidden_states else None
        out = self._forward(x, mask_u8, None, hidden)
        if hidden is not None:
            hidden = [x] + [h.to(x.dtype) for h in hidden[1:]]
        return out.view(x.shape).to(x.dtype), hidden

    def backward(self, save, dOUT):
        s = self.s
        d, B, S = s.d, save.B, save.S
        M = B * S
        fln = self.final_ln
        dOUT = as_f32(dOUT, (M, d))
        G, Gb, done = s.start_backward(save, M, fln, dOUT if fln is not None else None, None if fln is not None else dOUT)
        G = s.stack.backward(G, Gb, B, S, top_bias_done=done, save=save)
        return (G.view(B, S, d).clone(),)


class PostNormLayersRuntime:
    """A standalone post-norm `TransformerEncoderLayer` or `TransformerEncoder` (modules/layers/transformer.py:113-128,
    216-259) in both grad modes, with the same interface as EncoderLayersRuntime.  Per layer, x1 = LN1(x + s_a Attn(x))
    and out = LN2(x1 + s_f FF(x1)) (s_a / s_f: stochastic-depth factors, 1 without drop path), then the optional final
    LayerNorm.  Its own schedule, not TransformerStack's: there each LayerNorm feeds a branch, here it closes one.

    The backward runs the LayerNorm backward on the fp32 gradient of its output (no residual gradient comes in: the
    residual stream is the normalised one), and the FC1 / QKV input gradients are fp32 GEMMs that accumulate into the
    gradient that left that LayerNorm, which forms dx1 = dS2 + W1^T dPRE and dx = dS1 + Wqkv^T dQKV in place."""

    def __init__(self, owner: nn.Module, layers, final_ln: Optional[nn.Module]):
        self.layers = list(layers)
        self.final_ln = final_ln
        self.store = ParamStore(list(owner.parameters()))
        self.device = self.store.device
        self.ws = Workspace(self.device)
        l0 = self.layers[0]
        self.d = l0.attention_layernorm.normalized_shape[0]
        self.H = l0.attention.num_heads
        self.hd = self.d // self.H
        if self.d % self.H or self.hd not in (64, 96, 128):
            raise MMBError(f"TransformerEncoderLayer: head_dim {self.d / self.H:g} is not supported by the attention "
                           "kernels")
        mlp = l0.feedforward.model
        self.ff = mlp[0].weight.shape[0]
        self.act = act_code(mlp[1])

    def _forward(self, x: torch.Tensor, mask_u8, save: Optional[Workspace], hidden: Optional[List[torch.Tensor]]):
        """-> the output fp32 [B*S, d].  hidden: receives each layer's output fp32 [B, S, d] (fresh tensors).  A bf16 x
        without `save` rounds each layer's output to bf16 before the next layer reads it, as the layer-at-a-time call
        does when each layer returns in its input's dtype."""
        st, d, H, hd, ff = self.store, self.d, self.H, self.hd, self.ff
        B, S, _ = x.shape
        M = B * S
        bf, f32 = torch.bfloat16, torch.float32
        if save is not None and hd != 64:
            raise MMBError(f"training needs head_dim 64 in the layer stacks (got {hd}); call it under torch.no_grad()")
        st.refresh()
        if save is None:
            buf = lambda name, l, shape, dt: self.ws.get(f"pn.{name}", shape, dt)  # noqa: E731
        else:
            buf = lambda name, l, shape, dt: save.get(f"pn.{name}.{l}", shape, dt)  # noqa: E731
        round_bf16 = save is None and x.dtype == bf
        scales = drop_path_scales(self.layers, B, self.device)   # training with drop_path_rate: once, for all layers
        if save is not None:
            save.mask, save.B, save.S, save.scales = mask_u8, B, S, scales
        X = x.contiguous().float().view(M, d)      # only read: the residual add of the first layer
        Xb = buf("Xb", 0, (M, d), bf)
        ops.cast_bf16(X.view(-1), Xb.view(-1))
        QKV0, O0 = self.ws.get("pn.QKV", (M, 3 * d), bf), self.ws.get("pn.O", (M, d), bf)
        Y = self.ws.get("pn.Y", (M, d), bf)
        for l, layer in enumerate(self.layers):
            at, mlp = layer.attention, layer.feedforward.model
            ln1, ln2 = layer.attention_layernorm, layer.feedforward_layernorm
            s_a, s_f = scales[l] if scales is not None else (None, None)
            keep = save is not None
            QKV = buf("QKV", l, (M, 3 * d), bf) if keep else QKV0
            O = buf("O", l, (M, d), bf) if keep else O0
            LSE = buf("LSE", l, (B * H * S,), f32)
            S1 = buf("S1", l, (M, d), f32) if keep else None          # x + s_a Attn(x): LN1's input
            X1 = buf("X1", l, (M, d), f32)                             # LN1's output, fp32 + its bf16 operand copy
            X1b = buf("X1b", l, (M, d), bf)
            PRE, HACT = buf("PRE", l, (M, ff), bf), buf("HACT", l, (M, ff), bf)
            S2 = buf("S2", l, (M, d), f32) if keep else None          # x1 + s_f FF(x1): LN2's input
            m1, r1, m2, r2 = ((buf(n, l, (M,), f32) for n in ("m1", "r1", "m2", "r2")) if keep else (None,) * 4)
            last = l == len(self.layers) - 1
            OUT = (torch.empty((M, d), device=self.device, dtype=f32) if hidden is not None or last
                   else self.ws.get(f"pn.X{l % 2}", (M, d), f32))
            OUTb = buf("Xb", l + 1, (M, d), bf) if not last or round_bf16 else None   # the next QKV GEMM's operand
            ops.gemm(Xb, st.shadow(at.input_proj.weight), bias=at.input_proj.bias, out=QKV)
            ops.self_attention(QKV, O, LSE, B, S, H, hd, False, 1.0 / math.sqrt(hd), mask=mask_u8)
            ops.gemm(O, st.shadow(at.output_proj.weight), bias=at.output_proj.bias, out=Y)
            ops.add_layernorm_fwd(X, Y, S1, X1b, X1, ln1.weight, ln1.bias, m1, r1, M, d, ln1.eps, **scaled(s_a, S))
            ops.gemm(X1b, st.shadow(mlp[0].weight), bias=mlp[0].bias, epilogue=ops.EPI_BF16_ACT, out=PRE, out2=HACT,
                     act=self.act)
            ops.gemm(HACT, st.shadow(mlp[-1].weight), bias=mlp[-1].bias, out=Y)
            ops.add_layernorm_fwd(X1, Y, S2, OUTb, OUT, ln2.weight, ln2.bias, m2, r2, M, d, ln2.eps, **scaled(s_f, S))
            if round_bf16:
                ops.cast_f32(OUTb, OUT)
            if hidden is not None:
                hidden.append(OUT.view(B, S, d))
            X, Xb = OUT, OUTb
        fln = self.final_ln
        if save is not None:
            save.XF = X
        if fln is None:
            return X
        LAST = torch.empty((M, d), device=self.device, dtype=f32)
        stats = save if save is not None else self.ws
        ops.add_layernorm_fwd(X, None, None, None, LAST, fln.weight, fln.bias, stats.get("pn.mF", (M,), f32),
                              stats.get("pn.rF", (M,), f32), M, d, fln.eps)
        return LAST

    def forward(self, data, diff):
        """data: (uint8 [B, S, S] mask or None, the caller's list that receives hidden_states or None)."""
        mask_u8, hidden = data
        (x,) = diff
        save = Workspace(self.device)
        if hidden is not None:
            hidden.append(x)
        out = self._forward(x, mask_u8, save, hidden)
        return (out.view(x.shape),), save

    def infer(self, x: torch.Tensor, mask_u8: Optional[torch.Tensor], return_hidden_states: bool = False):
        """-> (output [B, S, d], hidden_states or None), in x's dtype.  hidden_states: x itself, then each layer's
        output (the last one before the final LayerNorm)."""
        hidden: Optional[List[torch.Tensor]] = [] if return_hidden_states else None
        out = self._forward(x, mask_u8, None, hidden)
        if hidden is not None:
            hidden = [x] + [h.to(x.dtype) for h in hidden]
        return out.view(x.shape).to(x.dtype), hidden

    def backward(self, save, dOUT):
        st, d, H, hd, ff = self.store, self.d, self.H, self.hd, self.ff
        B, S, mask_u8 = save.B, save.S, save.mask
        M = B * S
        bf, f32 = torch.bfloat16, torch.float32
        sp = ops.wgrad_splits
        scales = save.scales
        G = as_f32(dOUT, (M, d))                 # the gradient of the current layer's output, read only
        GA, GB = self.ws.get("pn.GA", (M, d), f32), self.ws.get("pn.GB", (M, d), f32)   # dS1 / dx, dS2 / dx1
        Gb = self.ws.get("pn.Gb", (M, d), bf)
        T1, T3 = self.ws.get("pn.T1", (M, d), bf), self.ws.get("pn.T3", (M, 3 * d), bf)
        fln = self.final_ln
        if fln is not None:
            ops.layernorm_bwd(save.XF, None, G, save.get("pn.mF", (M,), f32), save.get("pn.rF", (M,), f32), fln.weight,
                              None, GA, None, st.grad(fln.weight), st.grad(fln.bias), M, d)
            G = GA
        for l in range(len(self.layers) - 1, -1, -1):
            layer = self.layers[l]
            at, mlp = layer.attention, layer.feedforward.model
            ln1, ln2 = layer.attention_layernorm, layer.feedforward_layernorm
            s_a, s_f = scales[l] if scales is not None else (None, None)
            g = lambda n, shape, dt: save.get(f"pn.{n}.{l}", shape, dt)  # noqa: E731
            Xb, QKV, O = g("Xb", (M, d), bf), g("QKV", (M, 3 * d), bf), g("O", (M, d), bf)
            LSE = g("LSE", (B * H * S,), f32)
            S1, X1b, S2 = g("S1", (M, d), f32), g("X1b", (M, d), bf), g("S2", (M, d), f32)
            PRE, HACT = g("PRE", (M, ff), bf), g("HACT", (M, ff), bf)
            m1, r1, m2, r2 = (g(n, (M,), f32) for n in ("m1", "r1", "m2", "r2"))
            w1, w2 = mlp[0].weight, mlp[-1].weight
            dS2, dS1 = GB, GA   # G (GA below the top layer) is dead once LN2's backward has read it
            # ---- LN2:  dS2 = dLN2/dS2 (fp32), Gb = bf16(s_f dS2) enters the feed-forward branch ----
            ops.layernorm_bwd(S2, None, G, m2, r2, ln2.weight, None, dS2, Gb, st.grad(ln2.weight), st.grad(ln2.bias),
                              M, d, gsum=st.grad(mlp[-1].bias), **scaled(s_f, S))
            ops.gemm(Gb, HACT, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(w2), splits=sp(d, ff, M),
                     accumulate=True)
            dPRE = HACT   # the activation output is dead once its wgrad has been issued (same stream)
            ops.gemm(Gb, st.shadow(w2), b_mn=True, epilogue=ops.EPI_BF16_DACT, aux=PRE, out=dPRE, act=self.act,
                     colsum=st.grad(mlp[0].bias))
            ops.gemm(dPRE, X1b, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(w1), splits=sp(ff, d, M),
                     accumulate=True)
            ops.gemm(dPRE, st.shadow(w1), b_mn=True, epilogue=ops.EPI_F32, out=dS2, accumulate=True)   # dx1
            # ---- LN1:  dS1 = dLN1/dS1, Gb = bf16(s_a dS1) enters the attention branch ----
            ops.layernorm_bwd(S1, None, dS2, m1, r1, ln1.weight, None, dS1, Gb, st.grad(ln1.weight), st.grad(ln1.bias),
                              M, d, gsum=st.grad(at.output_proj.bias), **scaled(s_a, S))
            ops.gemm(Gb, O, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(at.output_proj.weight),
                     splits=sp(d, d, M), accumulate=True)
            ops.gemm(Gb, st.shadow(at.output_proj.weight), b_mn=True, out=T1)   # dO
            ops.self_attention(QKV, O, LSE, B, S, H, hd, False, 1.0 / math.sqrt(hd), mask=mask_u8, dout=T1, dqkv=T3)
            ops.gemm(T3, Xb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(at.input_proj.weight),
                     splits=sp(3 * d, d, M), accumulate=True)
            ops.colsum_bf16(T3, st.grad(at.input_proj.bias), M, 3 * d, 3 * d)
            ops.gemm(T3, st.shadow(at.input_proj.weight), b_mn=True, epilogue=ops.EPI_F32, out=dS1, accumulate=True)
            G = dS1   # dx: the gradient of the layer below's output
        return (G.view(B, S, d).clone(),)


def _runtime_forward(mod: nn.Module, hidden_states: torch.Tensor, attention_mask: Optional[torch.Tensor], what: str,
                     return_hidden_states: bool = False):
    """A TransformerEncoderLayer / TransformerEncoder on its runtime (EncoderLayersRuntime for pre-norm layers,
    PostNormLayersRuntime for post-norm ones) -> (output, hidden_states or None).  With an autograd graph the output
    is fp32."""
    B, S, _ = hidden_states.shape
    if _wants_graph(mod, hidden_states):
        hidden = [] if return_hidden_states else None
        (out,) = run(mod._runtime(), (_bool_mask_u8(attention_mask, B, S, what), hidden), (hidden_states.float(),))
        return out.view(hidden_states.shape), hidden
    _cuda(hidden_states, what)
    with torch.no_grad():
        return mod._runtime().infer(hidden_states, _bool_mask_u8(attention_mask, B, S, what), return_hidden_states)


def encoder_layer_forward(mod: nn.Module, hidden_states: torch.Tensor,
                          attention_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """TransformerEncoderLayer.forward (transformer.py:95-154), pre-norm (:95-111) or post-norm (:113-128), on the
    layer's runtime.  With a drop_path_rate in training, each branch is scaled per sample inside the residual add that
    follows it."""
    return _runtime_forward(mod, hidden_states, attention_mask, "TransformerEncoderLayer")[0]


def encoder_forward(mod: nn.Module, hidden_states: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                    return_hidden_states: bool = False):
    """TransformerEncoder.forward (transformer.py:216-259): the layers (+ optional final LayerNorm) on the encoder's
    runtime."""
    from .modules.layers.transformer import TransformerOutput

    out, hidden = _runtime_forward(mod, hidden_states, attention_mask, "TransformerEncoder", return_hidden_states)
    return TransformerOutput(last_hidden_state=out, hidden_states=hidden)


def patch_embeddings_forward(mod: nn.Module, image: torch.Tensor, image_patches_mask: Optional[torch.Tensor] = None):
    """PatchEmbeddings.forward (patch_embedding.py:104-154): conv projection as im2col + wgmma GEMM, [cls |] patches
    (mask-token substitution) + position embeddings in one assembly kernel.  In training with a patch_drop_rate, only
    the kept patches are embedded (gathered im2col and assembly) and random_mask / ids_restore are returned as the
    reference returns them (float rate; None for a (rate_h, rate_w) tuple)."""
    from .modules.layers.patch_embedding import PatchEmbeddingsOutput
    from .modules.masking.random_masking import patch_keep_indices

    forward_only_guard(mod, "PatchEmbeddings")
    _cuda(image, "PatchEmbeddings")
    conv = mod.conv_projection
    C, Hh, Ww = image.shape[1:]
    if C != 3 or (Hh, Ww) != tuple(mod.image_size):
        raise ValueError(f"Input image shape {tuple(image.shape)} doesn't match the model's 3 x {mod.image_size}")
    rt = _rt(mod, image.device)
    d = conv.weight.shape[0]
    drop = patch_keep_indices(mod, image.shape[0], image.device)
    keep, random_mask, ids_restore = drop if drop is not None else (None, None, None)
    X, B, S, _, _ = patch_embed_fwd(image, conv, rt.sh.get("conv.w", [conv.weight.view(d, -1)]),
                                    mod.cls_token if mod.include_cls_embed else None, mod.position_embeddings,
                                    mod.mask_token, image_patches_mask, rt.ws, rt.ws, "pe", keep=keep)
    return PatchEmbeddingsOutput(embeddings=X.view(B, S, d).to(image.dtype), random_mask=random_mask,
                                 ids_restore=ids_restore)


# ---------------------------------------------------------------------------------------------------------------------
# Decoding with a key / value cache: MultiHeadAttentionWithCache, TransformerDecoderLayer, TransformerDecoder
# (modules/layers/multi_head_attention.py:83-180, transformer.py:262-657)
#
# A returned cache tensor has the reference's shape [B, H, S, hd]; it is the transposed view of a fresh row-major
# [B, S, H*hd] buffer (the view the reference itself returns on a call without a past), so the attention kernels read it
# with row stride H*hd.  A past in any layout is concatenated with the new projection rows by the append kernel, which
# also writes the bf16 operand copy when the cache is fp32.  Queries of at most ops.DECODE_MAX_SQ rows run the split-KV
# decode kernel where it is the faster one (ops.decode_attention_wins), the others the general attention kernels.
# ---------------------------------------------------------------------------------------------------------------------
def _rect_mask_u8(mask: Optional[torch.Tensor], B: int, Sq: int, Skv: int, what: str):
    """bool [Sq, Skv], [B|1, Sq|1, Skv] or [B|1, 1, Sq|1, Skv] (True = attend) -> (uint8 mask, mask_bs, mask_qs): the
    broadcast dimensions get stride 0.  Float (additive) and per-head masks are not supported."""
    if mask is None:
        return None, 0, 0
    if mask.dtype != torch.bool:
        raise NotImplementedError(f"{what}: only boolean attention masks (True = attend) are on the accelerated path")
    if mask.dim() == 4:
        if mask.shape[1] != 1:
            raise NotImplementedError(f"{what}: per-head masks are not on the accelerated path (the head dim must be 1)")
        mask = mask[:, 0]
    if mask.dim() == 2:
        mask = mask[None]
    if mask.dim() != 3 or mask.shape[0] not in (1, B) or mask.shape[1] not in (1, Sq) or mask.shape[2] != Skv:
        raise ValueError(f"{what}: attention mask shape {tuple(mask.shape)} does not broadcast to [{B}, {Sq}, {Skv}]")
    Bm, Qm = mask.shape[0], mask.shape[1]
    u8 = mask.to(torch.uint8).contiguous()
    return u8, (0 if Bm == 1 else Qm * Skv), (0 if Qm == 1 else Skv)


def _attend(q, k, v, O, B, Sq, Skv, H, hd, bsq, bsk, bsv, mask, causal):
    """O [B*Sq, H*hd] = attention of 2-D bf16 views (row-major, batch strides bs*); mask = (u8, mask_bs, mask_qs)."""
    fn = ops.attention_fwd_decode if ops.decode_attention_wins(B, H, Sq, Skv) else ops.attention_fwd_generic
    fn(q, k, v, O, B=B, Sq=Sq, Skv=Skv, H=H, head_dim=hd, bsq=bsq, bsk=bsk, bsv=bsv, bso=Sq * H * hd,
       scale=1.0 / math.sqrt(hd), mask=mask[0], mask_bs=mask[1], mask_qs=mask[2], causal=causal)


def _cache_dtype(past: Optional[torch.Tensor], new_dtype: torch.dtype) -> torch.dtype:
    dt = new_dtype if past is None else torch.promote_types(past.dtype, new_dtype)   # torch.cat's promotion
    if dt not in (torch.float32, torch.bfloat16):
        raise MMBError(f"MultiHeadAttentionWithCache: key / value cache dtype {dt} is not supported (fp32 / bf16)")
    return dt


def _mha_cache(mod: nn.Module, rt: _Rt, tag: str, Xq, Xk, Xv, B: int, Sq: int, Sk: int, mask, causal: bool,
               past, use_cache: bool, kv_dtypes, out_epi: int):
    """MultiHeadAttentionWithCache on bf16 input rows Xq [B*Sq, dim_q] and Xk / Xv [B*Sk, dim_kv] (`Xk is Xv`: one
    packed K|V GEMM; `Xq is Xk is Xv`: one packed Q|K|V GEMM).  Returns (output-projection rows [B*Sq, d] in fp32
    (out_epi = EPI_F32) or bf16, (K, V) caches [B, H, S, hd] or None)."""
    ws, sh = rt.ws, rt.sh
    d = mod.q_proj.weight.shape[0]
    H = mod.num_heads
    hd = d // H
    if d % H or hd not in (64, 96, 128):
        raise MMBError(f"MultiHeadAttentionWithCache: head_dim {d / H:g} is not supported by the attention kernels "
                       "(64 / 96 / 128)")
    bf = torch.bfloat16
    qp, kp, vp = mod.q_proj, mod.k_proj, mod.v_proj
    has_bias = qp.bias is not None

    def bias(key, parts):
        return sh.cat_f32(key, [p.bias for p in parts]) if has_bias else None

    if Xq is Xk and Xk is Xv:
        QKV = ws.get(tag + ".QKV", (B * Sq, 3 * d), bf)
        ops.gemm(Xq, sh.get("wqkv", [qp.weight, kp.weight, vp.weight]), bias=bias("bqkv", (qp, kp, vp)), out=QKV)
        Q, K, V, ldkv = QKV[:, :d], QKV[:, d:2 * d], QKV[:, 2 * d:], 3 * d
    else:
        Q = ws.get(tag + ".Q", (B * Sq, d), bf)
        ops.gemm(Xq, sh.get("wq", [qp.weight]), bias=qp.bias, out=Q)
        if Xk is Xv:
            KV = ws.get(tag + ".KV", (B * Sk, 2 * d), bf)
            ops.gemm(Xk, sh.get("wkv", [kp.weight, vp.weight]), bias=bias("bkv", (kp, vp)), out=KV)
            K, V, ldkv = KV[:, :d], KV[:, d:], 2 * d
        else:
            K, V = ws.get(tag + ".K", (B * Sk, d), bf), ws.get(tag + ".V", (B * Sk, d), bf)
            ops.gemm(Xk, sh.get("wk", [kp.weight]), bias=kp.bias, out=K)
            ops.gemm(Xv, sh.get("wv", [vp.weight]), bias=vp.bias, out=V)
            ldkv = d
    Sp = 0 if past is None else past[0].shape[2]
    St = Sp + Sk
    caches = None
    bsk = bsv = Sk * ldkv
    if past is not None or use_cache:
        caches = []
        ops_kv = []
        for i, (new, p) in enumerate(((K, None if past is None else past[0]), (V, None if past is None else past[1]))):
            if p is not None and (p.dim() != 4 or tuple(p.shape[:2]) != (B, H) or p.shape[3] != hd or p.shape[2] != Sp):
                raise ValueError(f"MultiHeadAttentionWithCache: past key / value of shape {tuple(p.shape)}, expected "
                                 f"[{B}, {H}, S, {hd}] with the same S for both")
            dt = _cache_dtype(p, kv_dtypes[i])
            buf = torch.empty((B, St, d), device=Xq.device, dtype=dt) if use_cache else None
            opnd = buf if dt == bf and buf is not None else ws.get(f"{tag}.C{i}", (B, St, d), bf)
            ops.kv_cache_append(p, new, buf, None if opnd is buf else opnd, B=B, H=H, Sp=Sp, Sn=Sk, head_dim=hd)
            ops_kv.append(opnd.view(B * St, d))
            if use_cache:
                caches.append(buf.view(B, St, H, hd).transpose(1, 2))
        K, V = ops_kv
        bsk = bsv = St * d
    O = ws.get(tag + ".O", (B * Sq, d), bf)
    _attend(Q, K, V, O, B, Sq, St, H, hd, Sq * Q.stride(0), bsk, bsv, mask, causal)
    odt = torch.float32 if out_epi == ops.EPI_F32 else bf
    Y = torch.empty((B * Sq, d), device=Xq.device, dtype=odt) if odt == torch.float32 else ws.get(tag + ".Y", (B * Sq, d), bf)
    ops.gemm(O, sh.get("wo", [mod.output_proj.weight]), bias=mod.output_proj.bias, epilogue=out_epi, out=Y)
    return Y, (tuple(caches) if use_cache else None)


def _check_training_dropout(mod: nn.Module, what: str) -> None:
    if mod.training and mod.dropout > 0:
        raise NotImplementedError(f"{what}: dropout > 0 in training mode is not on the accelerated path")


def mha_cache_forward(mod: nn.Module, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                      attn_mask: Optional[torch.Tensor] = None, past_key_value=None, is_causal: bool = False,
                      use_cache: bool = False):
    """MultiHeadAttentionWithCache.forward (multi_head_attention.py:116-180): projections (packed when the inputs are
    the same tensor) -> cache append -> decode / general attention -> output projection."""
    from .modules.layers.multi_head_attention import MHAWithCacheOutput

    forward_only_guard(mod, "MultiHeadAttentionWithCache")
    _check_training_dropout(mod, "MultiHeadAttentionWithCache")
    for t, n in ((query, "query"), (key, "key"), (value, "value")):
        _cuda(t, f"MultiHeadAttentionWithCache {n}")
    B, Sq, _ = query.shape
    if key.size(0) != B or value.size(0) != B:
        raise ValueError("key and value should have the same bsz as query.")
    Sk = key.shape[1]
    if value.shape[1] != Sk:
        raise ValueError(f"MultiHeadAttentionWithCache: key and value lengths differ ({Sk} vs {value.shape[1]})")
    rt = _rt(mod, query.device)
    Xq = _to_bf16_rows(rt, query, "mhc.Xq")
    Xk = Xq if key is query else _to_bf16_rows(rt, key, "mhc.Xk")
    Xv = Xk if value is key else _to_bf16_rows(rt, value, "mhc.Xv")
    Sp = 0 if past_key_value is None else past_key_value[0].shape[2]
    mask = _rect_mask_u8(attn_mask, B, Sq, Sp + Sk, "MultiHeadAttentionWithCache")
    Y, cache = _mha_cache(mod, rt, "mhc", Xq, Xk, Xv, B, Sq, Sk, mask, bool(is_causal), past_key_value, use_cache,
                          (key.dtype, value.dtype), ops.EPI_F32)
    out = Y.view(B, Sq, -1).to(query.dtype)
    return MHAWithCacheOutput(out, cache) if use_cache else out


def _decoder_layer(mod: nn.Module, X: torch.Tensor, B: int, S: int, ENC: Optional[torch.Tensor], S_enc: int,
                   mask, cross_mask, past, use_cache: bool, kv_dtype: torch.dtype):
    """One TransformerDecoderLayer on fp32 rows X [B*S, d] (ENC: bf16 rows [B*S_enc, dim_kv] or None).  Returns fresh
    fp32 output rows and the self-attention cache."""
    rt = _rt(mod, X.device)
    ws, sh = rt.ws, rt.sh
    M, d = X.shape
    bf, f32 = torch.bfloat16, torch.float32
    mlp = mod.feedforward.model
    act = act_code(mlp[1])
    ff = mlp[0].weight.shape[0]
    LN, PRE, HACT = ws.get("d.LN", (M, d), bf), ws.get("d.PRE", (M, ff), bf), ws.get("d.HACT", (M, ff), bf)
    w1, w2 = sh.get("w1", [mlp[0].weight]), sh.get("w2", [mlp[-1].weight])
    ln1, ln2 = mod.attention_layernorm, mod.feedforward_layernorm
    cross = mod.use_cross_attention and (ENC is not None or not mod.norm_first)
    if cross and ENC is None:
        raise ValueError("encoder_hidden_states must be provided for cross attention")
    lnc = mod.cross_attention_layernorm if cross else None
    out = torch.empty((M, d), device=X.device, dtype=f32)
    kvd = (kv_dtype, kv_dtype)

    def self_attn(inp):
        return _mha_cache(mod.attention, _rt(mod.attention, X.device), "sa", inp, inp, inp, B, S, S, mask, False, past,
                          use_cache, kvd, ops.EPI_BF16)

    def cross_attn(inp):
        return _mha_cache(mod.cross_attention, _rt(mod.cross_attention, X.device), "ca", inp, ENC, ENC, B, S, S_enc,
                          cross_mask, False, None, False, kvd, ops.EPI_BF16)[0]

    if mod.norm_first:   # transformer.py:390-428
        ops.add_layernorm_fwd(X, None, None, LN, None, ln1.weight, ln1.bias, None, None, M, d, ln1.eps)
        Y, cache = self_attn(LN)
        XA = ws.get("d.XA", (M, d), f32)                        # x + self-attention
        if cross:
            ops.add_layernorm_fwd(X, Y, XA, LN, None, lnc.weight, lnc.bias, None, None, M, d, lnc.eps)
            Y = cross_attn(LN)
            XC = ws.get("d.XC", (M, d), f32)                    # ... + cross-attention
            ops.add_layernorm_fwd(XA, Y, XC, LN, None, ln2.weight, ln2.bias, None, None, M, d, ln2.eps)
        else:
            ops.add_layernorm_fwd(X, Y, XA, LN, None, ln2.weight, ln2.bias, None, None, M, d, ln2.eps)
            XC = XA
        ops.gemm(LN, w1, bias=mlp[0].bias, epilogue=ops.EPI_BF16_ACT, out=PRE, out2=HACT, act=act)
        Y = ws.get("d.Y", (M, d), bf)
        ops.gemm(HACT, w2, bias=mlp[-1].bias, out=Y)
        ops.add_layernorm_fwd(XC, Y, out, None, None, ln2.weight, ln2.bias, None, None, M, d, ln2.eps)
    else:                # transformer.py:430-470
        ops.cast_bf16(X.view(-1), LN.view(-1))
        Y, cache = self_attn(LN)
        H1 = ws.get("d.H1", (M, d), f32)                        # LN1(x + self-attention), fp32 + its bf16 copy
        ops.add_layernorm_fwd(X, Y, None, LN, H1, ln1.weight, ln1.bias, None, None, M, d, ln1.eps)
        if cross:
            Y = cross_attn(LN)
            H2 = ws.get("d.H2", (M, d), f32)
            ops.add_layernorm_fwd(H1, Y, None, LN, H2, lnc.weight, lnc.bias, None, None, M, d, lnc.eps)
            H1 = H2
        ops.gemm(LN, w1, bias=mlp[0].bias, epilogue=ops.EPI_BF16_ACT, out=PRE, out2=HACT, act=act)
        Y = ws.get("d.Y", (M, d), bf)
        ops.gemm(HACT, w2, bias=mlp[-1].bias, out=Y)
        ops.add_layernorm_fwd(H1, Y, None, None, out, ln2.weight, ln2.bias, None, None, M, d, ln2.eps)
    return out, cache


def _decoder_inputs(mod: nn.Module, hidden_states, encoder_hidden_states, what: str):
    forward_only_guard(mod, what)   # the layers' constructors already refuse dropout > 0
    _cuda(hidden_states, what)
    B, S, d = hidden_states.shape
    X = hidden_states.contiguous().float().view(B * S, d)
    ENC, S_enc = None, 0
    if encoder_hidden_states is not None:
        _cuda(encoder_hidden_states, what)
        if encoder_hidden_states.size(0) != B:
            raise ValueError("key and value should have the same bsz as query.")
        S_enc = encoder_hidden_states.shape[1]
        ENC = _to_bf16_rows(_rt(mod, hidden_states.device), encoder_hidden_states, "dec.ENC")
    return B, S, d, X, ENC, S_enc


def decoder_layer_forward(mod: nn.Module, hidden_states: torch.Tensor,
                          encoder_hidden_states: Optional[torch.Tensor] = None,
                          attention_mask: Optional[torch.Tensor] = None,
                          cross_attention_mask: Optional[torch.Tensor] = None, past_key_value=None,
                          use_cache: bool = False):
    """TransformerDecoderLayer.forward (transformer.py:472-519): (output, present_key_value or None)."""
    B, S, d, X, ENC, S_enc = _decoder_inputs(mod, hidden_states, encoder_hidden_states, "TransformerDecoderLayer")
    Sp = 0 if past_key_value is None else past_key_value[0].shape[2]
    mask = _rect_mask_u8(attention_mask, B, S, Sp + S, "TransformerDecoderLayer")
    cmask = _rect_mask_u8(cross_attention_mask, B, S, S_enc, "TransformerDecoderLayer") if ENC is not None else (None, 0, 0)
    out, cache = _decoder_layer(mod, X, B, S, ENC, S_enc, mask, cmask, past_key_value, use_cache, hidden_states.dtype)
    return out.view(B, S, d).to(hidden_states.dtype), cache


def decoder_forward(mod: nn.Module, hidden_states: torch.Tensor, encoder_hidden_states: Optional[torch.Tensor] = None,
                    attention_mask: Optional[torch.Tensor] = None, cross_attention_mask: Optional[torch.Tensor] = None,
                    past_key_values=None, use_cache: bool = False, return_hidden_states: bool = False):
    """TransformerDecoder.forward (transformer.py:588-657).  As in the reference, cross_attention_mask is accepted and
    not passed to the layers, and hidden_states / current_key_values are empty lists when not requested."""
    from .modules.layers.transformer import TransformerOutput

    B, S, d, X, ENC, S_enc = _decoder_inputs(mod, hidden_states, encoder_hidden_states, "TransformerDecoder")
    dt = hidden_states.dtype
    Sp = 0 if past_key_values is None else past_key_values[0][0].shape[2]
    mask = _rect_mask_u8(attention_mask, B, S, Sp + S, "TransformerDecoder")
    all_hidden, current = [], []
    x = X
    for i, layer in enumerate(mod.layer):
        if return_hidden_states:
            all_hidden.append(hidden_states if i == 0 else x.view(B, S, d).to(dt))
        past = past_key_values[i] if past_key_values is not None else None
        x, cache = _decoder_layer(layer, x, B, S, ENC, S_enc, mask, (None, 0, 0), past, use_cache, dt)
        if use_cache:
            current.append(cache)
    if return_hidden_states:
        all_hidden.append(x.view(B, S, d).to(dt))
    if mod.final_layer_norm is not None:
        ln = mod.final_layer_norm
        y = torch.empty_like(x)
        ops.add_layernorm_fwd(x, None, None, None, y, ln.weight, ln.bias, None, None, B * S, d, ln.eps)
        x = y
    return TransformerOutput(last_hidden_state=x.view(B, S, d).to(dt), hidden_states=all_hidden,
                             current_key_values=current)
