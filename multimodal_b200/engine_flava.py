"""Forward runtime of the FLAVA encoders (BASELINE.json config 3: image + text + multimodal towers): the inference path
(torch.no_grad); the training path with backward schedules is engine_flava_train.py.

Same kernels as the CLIP path; what differs is the parameter layout (separate query/key/value Linears, packed here
into one [3d, d] operand), the exact-erf GELU epilogue, eps = 1e-12 LayerNorms, BERT embeddings + key-padding mask,
the pooler, and the returned ``TransformerOutput`` (every layer's residual stream is kept as ``hidden_states``).

Reference call stack: models/flava/model.py:127-298, models/flava/image_encoder.py:139-234,
modules/encoders/bert_text_encoder.py:67-120, models/flava/transformer.py:47-77,155-176,255-293,
modules/layers/attention.py:120-241, modules/losses/flava.py:84-97.

``TransformerOutput.attentions``: the flash-style kernel never materialises the [B, H, S, S] probabilities (477 MB
fp32 per layer at B=256) and nothing in the library consumes them, so they are produced ON REQUEST only
(`module.output_attentions = True`, or `return_attn_weights=True` on the text encoder): one extra kernel per layer
recomputes them from the packed QKV and the row LSE.  Default: ``None`` (documented deviation, DESIGN.md §10).
Every tensor of the returned ``TransformerOutput`` is allocated per call (as the reference's are); only internal
scratch is reused between forwards.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import nn

from . import engine as _engine
from . import ops
from ._lib import MMBError
from .engine import Workspace, _Shadows, act_code, patch_embed_fwd
from .modules.layers.transformer import TransformerOutput


class FlavaStack:
    """Forward of L pre-norm FLAVA `TransformerEncoderLayer`s (models/flava/transformer.py:155-176) + final LayerNorm
    + Pooler."""

    def __init__(self, encoder: nn.Module, layernorm: nn.Module, pooler: Optional[nn.Module], prefix: str):
        self.layers = list(encoder.layer)
        l0 = self.layers[0]
        if not l0.norm_first:
            raise MMBError("only pre-norm (norm_first=True) FLAVA layers are on the accelerated path")
        self.d = l0.attention.dim_q
        self.H = l0.attention.n_head
        if self.d // self.H != 64:
            raise MMBError("attention kernels support head_dim 64 only")
        self.ff = l0.feedforward.model[0].weight.shape[0]
        self.act = act_code(l0.feedforward.model[1])
        self.layernorm, self.pooler, self.prefix = layernorm, pooler, prefix
        dev = l0.attention.query.weight.device
        _engine._require_cuda(dev)
        self.device = dev
        self.ws = Workspace(dev)
        self.sh = _Shadows(dev)

    def forward(self, X0: torch.Tensor, B: int, S: int, kmask: Optional[torch.Tensor] = None,
                want_attn: bool = False) -> TransformerOutput:
        """want_attn: also return every layer's attention probabilities fp32 [B, H, S, S] (`attentions`), recomputed
        from the packed QKV and the row LSE of the fused attention kernel (mmb_attention_probs)."""
        d, ff, H, ws, sh = self.d, self.ff, self.H, self.ws, self.sh
        M = B * S
        bf, f32 = torch.bfloat16, torch.float32
        pfx = self.prefix
        Y = ws.get(f"{pfx}.Y", (M, d), bf)
        LN = ws.get(f"{pfx}.LN", (M, d), bf)
        QKV = ws.get(f"{pfx}.QKV", (M, 3 * d), bf)
        O = ws.get(f"{pfx}.O", (M, d), bf)
        XM = ws.get(f"{pfx}.XM", (M, d), f32)
        PRE = ws.get(f"{pfx}.PRE", (M, ff), bf)
        HACT = ws.get(f"{pfx}.HACT", (M, ff), bf)
        hidden: List[torch.Tensor] = [X0.view(B, S, d)]
        attns: Optional[List[torch.Tensor]] = [] if want_attn else None
        LSE = ws.get(f"{pfx}.LSE", (B * H * S,), f32) if want_attn else None
        XA = X0
        for l, layer in enumerate(self.layers):
            at, mlp = layer.attention, layer.feedforward.model
            wqkv = sh.get(f"{l}.wqkv", [at.query.weight, at.key.weight, at.value.weight])
            bqkv = sh.cat_f32(f"{l}.bqkv", [at.query.bias, at.key.bias, at.value.bias])
            wo = sh.get(f"{l}.wo", [at.output.weight])
            w1 = sh.get(f"{l}.w1", [mlp[0].weight])
            w2 = sh.get(f"{l}.w2", [mlp[-1].weight])
            ln1, ln2 = layer.attention_layernorm, layer.feedforward_layernorm
            if l > 0:  # x_l = x_{l-1,mid} + mlp_out (fused into this LayerNorm kernel); kept as hidden_states[l]
                XA = torch.empty((M, d), device=self.device, dtype=f32)   # returned (hidden_states[l]): fresh per call
                ops.add_layernorm_fwd(XM, Y, XA, LN, None, ln1.weight, ln1.bias, None, None, M, d, ln1.eps)
                hidden.append(XA.view(B, S, d))
            else:
                ops.add_layernorm_fwd(XA, None, None, LN, None, ln1.weight, ln1.bias, None, None, M, d, ln1.eps)
            ops.gemm(LN, wqkv, bias=bqkv, out=QKV)
            ops.self_attention(QKV, O, LSE, B, S, H, 64, False, 0.125, kmask=kmask)
            if want_attn:
                P = torch.empty((B, H, S, S), device=self.device, dtype=f32)
                ops.attention_probs(QKV, LSE, kmask, P, B, S, H, False, 0.125)
                attns.append(P)
            ops.gemm(O, wo, bias=at.output.bias, out=Y)
            ops.add_layernorm_fwd(XA, Y, XM, LN, None, ln2.weight, ln2.bias, None, None, M, d, ln2.eps)
            ops.gemm(LN, w1, bias=mlp[0].bias, epilogue=ops.EPI_BF16_ACT, out=PRE, out2=HACT, act=self.act)
            ops.gemm(HACT, w2, bias=mlp[-1].bias, out=Y)
        # returned tensors are allocated per call (the reference returns fresh tensors: a caller may keep the outputs
        # of several forwards alive); only internal scratch lives in the reused workspace
        XF = torch.empty((M, d), device=self.device, dtype=f32)      # final residual stream == hidden_states[-1] (pre-LayerNorm)
        LAST = torch.empty((M, d), device=self.device, dtype=f32)    # layernorm(XF) == last_hidden_state
        ops.add_layernorm_fwd(XM, Y, XF, None, LAST, self.layernorm.weight, self.layernorm.bias, None, None, M, d,
                              self.layernorm.eps)
        hidden.append(XF.view(B, S, d))
        pooled = None
        if self.pooler is not None:
            CLSb = ws.get(f"{pfx}.CLSb", (B, d), bf)
            ops.gather_rows_cast(LAST, CLSb, B, S, 0, d)
            pooled = torch.empty((B, d), device=self.device, dtype=f32)
            ops.gemm(CLSb, sh.get("pool.w", [self.pooler.dense.weight]), bias=self.pooler.dense.bias, epilogue=ops.EPI_F32,
                     out=pooled)
            ops.tanh_(pooled)
        return TransformerOutput(last_hidden_state=LAST.view(B, S, d), pooler_output=pooled, hidden_states=hidden,
                                 attentions=attns)

    def project_first_token(self, last_hidden_state: torch.Tensor, linear: nn.Linear, key: str) -> torch.Tensor:
        """linear(last_hidden_state[:, 0, :]) (models/flava/model.py:244-246, 261-263)."""
        B, S, d = last_hidden_state.shape
        CLSb = self.ws.get(f"{self.prefix}.CLSb2", (B, d), torch.bfloat16)
        ops.gather_rows_cast(last_hidden_state.reshape(B * S, d), CLSb, B, S, 0, d)
        out = torch.empty((B, linear.weight.shape[0]), device=self.device, dtype=torch.float32)
        ops.gemm(CLSb, self.sh.get(key, [linear.weight]), bias=linear.bias, epilogue=ops.EPI_F32, out=out)
        return out


class FlavaImageRuntime:
    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.stack = FlavaStack(mod.encoder, mod.layernorm, mod.pooler, "fimg")

    def forward(self, pixel_values: torch.Tensor, image_patches_mask: Optional[torch.Tensor] = None,
                want_attn: bool = False) -> TransformerOutput:
        emb, st = self.mod.embeddings, self.stack
        conv = emb.patch_embeddings.projection
        X0, B, S, _, _ = patch_embed_fwd(pixel_values, conv, st.sh.get("conv.w", [conv.weight.view(st.d, -1)]),
                                         emb.cls_token, emb.position_embeddings, emb.mask_token, image_patches_mask,
                                         st.ws, st.ws, "fimg")   # X0 is returned as hidden_states[0]
        return st.forward(X0, B, S, want_attn=want_attn)


class FlavaTextRuntime:
    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.stack = FlavaStack(mod.encoder, mod.layernorm, mod.pooler, "ftxt")

    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                token_type_ids: Optional[torch.Tensor] = None, want_attn: bool = False) -> TransformerOutput:
        emb, st = self.mod.embeddings, self.stack
        ws, d = st.ws, st.d
        ids = input_ids.long().contiguous()
        B, S = ids.shape
        if S > emb.position_embeddings.weight.shape[0]:
            raise ValueError(f"sequence length {S} exceeds max_position_embeddings")
        X0 = torch.empty((B * S, d), device=input_ids.device, dtype=torch.float32)   # returned as hidden_states[0]
        KM = ws.get("ftxt.KM", (B * S,), torch.uint8)
        tt = token_type_ids.long().contiguous() if token_type_ids is not None else None
        ops.bert_embed_ln_fwd(ids, tt, emb.word_embeddings.weight, emb.position_embeddings.weight,
                              emb.token_type_embeddings.weight, emb.layer_norm.weight, emb.layer_norm.bias, X0, KM,
                              emb.pad_token_id, B, S, d, emb.word_embeddings.weight.shape[0], emb.layer_norm.eps)
        if attention_mask is not None:  # user-supplied [B,S] mask (1 = attend) overrides the pad-derived one
            if attention_mask.dim() != 2:
                raise NotImplementedError("only [batch, seq_len] padding masks are supported on the accelerated path")
            KM = (attention_mask != 0).to(torch.uint8).contiguous().view(-1)
        return st.forward(X0, B, S, kmask=KM, want_attn=want_attn)


class FlavaMMRuntime:
    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.stack = FlavaStack(mod.encoder, mod.layernorm, mod.pooler, "fmm")

    def forward(self, hidden_states: torch.Tensor, want_attn: bool = False) -> TransformerOutput:
        """hidden_states: fp32 [B, S, d] (already projected and concatenated image|text tokens)."""
        st = self.stack
        B, S, d = hidden_states.shape
        hs = hidden_states.contiguous().float()
        if self.mod.cls_token is not None:
            X0 = torch.empty((B * (S + 1), d), device=hs.device, dtype=torch.float32)   # returned as hidden_states[0]
            # cat(cls, hidden) == concat_tokens(cls, hidden, <empty>)
            ops.concat_tokens(self.mod.cls_token, hs, hs, X0, B, S, 0, d)
            S += 1
        else:
            X0 = hs.view(B * S, d)
        return st.forward(X0, B, S, want_attn=want_attn)

    def forward_projected(self, image_hidden: torch.Tensor, text_hidden: torch.Tensor, image_proj: nn.Linear,
                          text_proj: nn.Linear, want_attn: bool = False) -> TransformerOutput:
        """FLAVAModel.encode_mm (models/flava/model.py:283-298): project both token streams to the multimodal width
        (two wgmma GEMMs, fp32 out + bias), then [cls | image | text] assembled by one kernel straight into X0."""
        st = self.stack
        ws, sh, d = st.ws, st.sh, st.d
        B, Si, di = image_hidden.shape
        Bt, St, dt = text_hidden.shape
        if B != Bt:
            raise ValueError(f"batch mismatch between image ({B}) and text ({Bt}) hidden states")
        bf, f32 = torch.bfloat16, torch.float32
        Ib = ws.get("fmm.Ib", (B * Si, di), bf)
        Tb = ws.get("fmm.Tb", (B * St, dt), bf)
        ops.cast_bf16(image_hidden.contiguous().float().view(-1), Ib.view(-1))
        ops.cast_bf16(text_hidden.contiguous().float().view(-1), Tb.view(-1))
        Pi = ws.get("fmm.Pi", (B * Si, d), f32)
        Pt = ws.get("fmm.Pt", (B * St, d), f32)
        ops.gemm(Ib, sh.get("proj.i", [image_proj.weight]), bias=image_proj.bias, epilogue=ops.EPI_F32, out=Pi)
        ops.gemm(Tb, sh.get("proj.t", [text_proj.weight]), bias=text_proj.bias, epilogue=ops.EPI_F32, out=Pt)
        cls = self.mod.cls_token
        S = Si + St + (1 if cls is not None else 0)
        X0 = torch.empty((B * S, d), device=image_hidden.device, dtype=f32)   # returned as hidden_states[0]
        ops.concat_tokens(cls, Pi, Pt, X0, B, Si, St, d)
        return st.forward(X0, B, S, want_attn=want_attn)
