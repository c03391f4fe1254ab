"""Forward runtime of the CoCa model family (BASELINE.json config 5 / SURVEY.md §8 a14): the inference path
(torch.no_grad); the training path with backward schedules is engine_coca_train.py.

One generic pre-norm layer runner serves the TorchMultimodal `TransformerEncoder` (fused `input_proj`) and
`TransformerDecoder` (separate q/k/v projections, optional cross-attention) of modules/layers/transformer.py:31-657:

    LN -> packed QKV GEMM -> attention -> out-proj GEMM -> (+residual, LN fused) -> [cross-attention] -> MLP (GELU fused
    into the first GEMM's epilogue) -> (+residual fused into the next LayerNorm kernel)

Attention routing: unmasked / causal self-attention with head_dim 64 runs on the tensor-core attention kernel (attention.cu);
anything else — cross-attention, the pooler's head_dim 96, the text decoder's [causal x padding] mask — on the general
kernels (attention_generic.cu while a head fits in shared memory, attention_generic_stream.cu at any longer length, e.g.
the pooler over the 576 image tokens of a 336-px ViT-L/14).  Reference call stacks: models/coca/coca_model.py:69-130, models/coca/text_decoder.py
:141-203, models/coca/multimodal_decoder.py:86-108, modules/layers/attention_pooler.py:48-101,
modules/encoders/vision_transformer.py:56-89, modules/layers/patch_embedding.py:104-154.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
from torch import nn

from . import ops
from ._lib import MMBError
from .engine import Workspace, _Shadows, act_code, patch_embed_fwd, scaled


class LayerStack:
    """Runs a list of pre-norm TransformerEncoderLayer / TransformerDecoderLayer parameter containers."""

    def __init__(self, layers, prefix: str, device):
        self.layers = list(layers)
        l0 = self.layers[0]
        if not l0.norm_first:
            raise MMBError("only pre-norm (norm_first=True) layers are on the accelerated path")
        if device.type != "cuda":
            raise MMBError("multimodal_b200 modules must live on a CUDA device (no CPU path); call .cuda() first")
        self.prefix, self.device = prefix, device
        self.d = l0.attention_layernorm.normalized_shape[0]
        self.H = l0.attention.num_heads
        self.hd = self.d // self.H
        if self.hd not in (64, 96, 128):
            raise MMBError(f"unsupported head_dim {self.hd}")
        self.ff = l0.feedforward.model[0].weight.shape[0]
        self.act = act_code(l0.feedforward.model[1])
        self.ws = Workspace(device)
        self.sh = _Shadows(device)

    # -- parameter views -------------------------------------------------------------------------------------------
    def _qkv(self, l: int, at):
        if hasattr(at, "input_proj"):   # MultiHeadSelfAttention: already packed [3d, d]
            return self.sh.get(f"{l}.wqkv", [at.input_proj.weight]), at.input_proj.bias
        return (self.sh.get(f"{l}.wqkv", [at.q_proj.weight, at.k_proj.weight, at.v_proj.weight]),
                self.sh.cat_f32(f"{l}.bqkv", [at.q_proj.bias, at.k_proj.bias, at.v_proj.bias]))

    def run(self, X0: torch.Tensor, B: int, S: int, *, causal: bool = False, mask: Optional[torch.Tensor] = None,
            enc: Optional[torch.Tensor] = None, S_enc: int = 0, keep_hidden: bool = False, scales=None):
        """X0 fp32 [B*S, d].  mask: uint8 [B, S, S] (1 = attend).  enc: bf16 [B*S_enc, d_kv] cross-attention source.
        scales: stochastic depth, per layer the (attention, feed-forward) factors fp32 [B] or None
        (stochastic_depth.drop_path_scales); each scales its branch in the residual add that follows it.
        Returns the hidden_states list or None; `finish` adds the last MLP branch."""
        d, ff, H, hd, ws, sh, pfx = self.d, self.ff, self.H, self.hd, self.ws, self.sh, self.prefix
        M = B * S
        bf, f32 = torch.bfloat16, torch.float32
        scale = 1.0 / math.sqrt(hd)
        Y = ws.get(f"{pfx}.Y", (M, d), bf)
        LN = ws.get(f"{pfx}.LN", (M, d), bf)
        QKV = ws.get(f"{pfx}.QKV", (M, 3 * d), bf)
        O = ws.get(f"{pfx}.O", (M, d), bf)
        PRE = ws.get(f"{pfx}.PRE", (M, ff), bf)
        HACT = ws.get(f"{pfx}.HACT", (M, ff), bf)
        XM = ws.get(f"{pfx}.XM", (M, d), f32)
        XC = ws.get(f"{pfx}.XC", (M, d), f32)
        hidden: Optional[List[torch.Tensor]] = [X0.view(B, S, d)] if keep_hidden else None
        XA = X0
        for l, layer in enumerate(self.layers):
            at, mlp = layer.attention, layer.feedforward.model
            wqkv, bqkv = self._qkv(l, at)
            ln1, ln2 = layer.attention_layernorm, layer.feedforward_layernorm
            if l > 0:   # x_l = previous mid-stream + previous MLP output, fused into this LayerNorm
                # returned as hidden_states[l] when requested: allocated per call (never aliases a later forward)
                XA = (torch.empty((M, d), device=X0.device, dtype=f32) if keep_hidden
                      else ws.get(f"{pfx}.XA.{l % 2}", (M, d), f32))
                ops.add_layernorm_fwd(XR, Y, XA, LN, None, ln1.weight, ln1.bias, None, None, M, d, ln1.eps,
                                      **scaled(scales[l - 1][1] if scales is not None else None, S))
                if keep_hidden:
                    hidden.append(XA.view(B, S, d))
            else:
                ops.add_layernorm_fwd(XA, None, None, LN, None, ln1.weight, ln1.bias, None, None, M, d, ln1.eps)
            ops.gemm(LN, wqkv, bias=bqkv, out=QKV)
            ops.self_attention(QKV, O, None, B, S, H, hd, causal, scale, mask=mask)
            ops.gemm(O, sh.get(f"{l}.wo", [at.output_proj.weight]), bias=at.output_proj.bias, out=Y)
            XR = XM
            if getattr(layer, "use_cross_attention", False) and enc is not None:
                if scales is not None:
                    raise MMBError("stochastic depth is applied to encoder layers only (no cross-attention)")
                ca, lnc = layer.cross_attention, layer.cross_attention_layernorm
                ops.add_layernorm_fwd(XA, Y, XM, LN, None, lnc.weight, lnc.bias, None, None, M, d, lnc.eps)
                Qc = ws.get(f"{pfx}.Qc", (M, d), bf)
                KV = ws.get(f"{pfx}.KVc", (B * S_enc, 2 * d), bf)
                ops.gemm(LN, sh.get(f"{l}.cq", [ca.q_proj.weight]), bias=ca.q_proj.bias, out=Qc)
                ops.gemm(enc, sh.get(f"{l}.ckv", [ca.k_proj.weight, ca.v_proj.weight]),
                         bias=sh.cat_f32(f"{l}.cbkv", [ca.k_proj.bias, ca.v_proj.bias]), out=KV)
                ops.attention_fwd_generic(Qc, KV[:, :d], KV[:, d:], O, B=B, Sq=S, Skv=S_enc, H=H, head_dim=hd, bsq=S * d,
                                          bsk=S_enc * 2 * d, bsv=S_enc * 2 * d, bso=S * d, scale=scale)
                ops.gemm(O, sh.get(f"{l}.co", [ca.output_proj.weight]), bias=ca.output_proj.bias, out=Y)
                ops.add_layernorm_fwd(XM, Y, XC, LN, None, ln2.weight, ln2.bias, None, None, M, d, ln2.eps)
                XR = XC
            else:
                ops.add_layernorm_fwd(XA, Y, XM, LN, None, ln2.weight, ln2.bias, None, None, M, d, ln2.eps,
                                      **scaled(scales[l][0] if scales is not None else None, S))
            ops.gemm(LN, sh.get(f"{l}.w1", [mlp[0].weight]), bias=mlp[0].bias, epilogue=ops.EPI_BF16_ACT, out=PRE,
                     out2=HACT, act=self.act)
            ops.gemm(HACT, sh.get(f"{l}.w2", [mlp[-1].weight]), bias=mlp[-1].bias, out=Y)
        self._last = (XR, Y, scales[-1][1] if scales is not None else None)
        return hidden

    def finish(self, B: int, S: int, final_ln: Optional[nn.Module], want_bf16: bool = False):
        """Adds the last MLP output to the stream (XF) and applies the optional final LayerNorm.
        Returns (XF fp32 [M,d], LAST fp32 or None, LAST bf16 or None)."""
        XR, Y, scale = self._last
        M, d, ws, pfx = B * S, self.d, self.ws, self.prefix
        # XF / LAST are handed to the caller (last_hidden_state / hidden_states[-1] / tokens): fresh per call, as the
        # reference's outputs are; bf16 copies consumed inside the same forward stay in the workspace
        XF = torch.empty((M, d), device=XR.device, dtype=torch.float32)
        ln = final_ln if final_ln is not None else self.layers[0].attention_layernorm  # affine unused when no output
        LAST = torch.empty((M, d), device=XR.device, dtype=torch.float32) if final_ln is not None else None
        LASTb = ws.get(f"{pfx}.LASTb", (M, d), torch.bfloat16) if (final_ln is not None and want_bf16) else None
        ops.add_layernorm_fwd(XR, Y, XF, LASTb, LAST, ln.weight, ln.bias, None, None, M, d, ln.eps,
                              **scaled(scale, S))
        return XF, LAST, LASTb


# ---------------------------------------------------------------------------------------------------------------------
class VisionRuntime:
    """modules/encoders/vision_transformer.py:56-89 — PatchEmbeddings + TransformerEncoder (+ optional final LN)."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        dev = mod.embeddings.conv_projection.weight.device
        self.stack = LayerStack(mod.encoder.layer, "vit", dev)

    def forward(self, images: torch.Tensor, image_patches_mask: Optional[torch.Tensor] = None):
        from .modules.layers.transformer import TransformerOutput
        from .modules.layers.stochastic_depth import drop_path_scales
        from .modules.masking.random_masking import patch_keep_indices

        emb, st = self.mod.embeddings, self.stack
        d, conv = st.d, emb.conv_projection
        drop = patch_keep_indices(emb, images.shape[0], images.device)   # training with patch_drop_rate
        scales = drop_path_scales(st.layers, images.shape[0], images.device)   # training with drop_path_rate
        X0, B, S, _, _ = patch_embed_fwd(images, conv, st.sh.get("conv.w", [conv.weight.view(d, -1)]),
                                         emb.cls_token if emb.include_cls_embed else None, emb.position_embeddings,
                                         emb.mask_token, image_patches_mask, st.ws, st.ws, "vit",
                                         keep=drop[0] if drop is not None else None)   # hidden_states[0]
        hidden = st.run(X0, B, S, keep_hidden=True, scales=scales)
        fln = self.mod.encoder.final_layer_norm
        XF, LAST, _ = st.finish(B, S, fln)
        hidden.append(XF.view(B, S, d))
        last = (LAST if fln is not None else XF).view(B, S, d)
        return TransformerOutput(last_hidden_state=last, pooler_output=None, hidden_states=hidden, attentions=None)


class PoolerRuntime:
    """AttentionPooler (modules/layers/attention_pooler.py:16-72): learned queries cross-attend to the LayerNorm-ed
    input; the query projection is batch independent and computed once per call for [n_queries, d]."""

    def __init__(self, mod: nn.Module, prefix: str):
        self.mod, self.prefix = mod, prefix
        dev = mod.query.device
        if dev.type != "cuda":
            raise MMBError("multimodal_b200 modules must live on a CUDA device (no CPU path); call .cuda() first")
        self.ws, self.sh, self.device = Workspace(dev), _Shadows(dev), dev

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x fp32 [B, S, d_in] -> fp32 [B, n_queries, d_out]."""
        m, ws, sh, pfx = self.mod, self.ws, self.sh, self.prefix
        B, S, din = x.shape
        nq, dout = m.query.shape
        H = m.attn.num_heads
        hd = dout // H
        bf, f32 = torch.bfloat16, torch.float32
        xk = ws.get(f"{pfx}.xk", (B * S, din), bf)
        ops.add_layernorm_fwd(x.contiguous().float().view(B * S, din), None, None, xk, None, m.ln_k.weight, m.ln_k.bias,
                              None, None, B * S, din, m.ln_k.eps)
        qn = ws.get(f"{pfx}.qn", (nq, dout), bf)
        ops.add_layernorm_fwd(m.query.data, None, None, qn, None, m.ln_q.weight, m.ln_q.bias, None, None, nq, dout,
                              m.ln_q.eps)
        Qp = ws.get(f"{pfx}.Qp", (nq, dout), bf)
        at = m.attn
        ops.gemm(qn, sh.get("wq", [at.q_proj.weight]), bias=at.q_proj.bias, out=Qp)
        KV = ws.get(f"{pfx}.KV", (B * S, 2 * dout), bf)
        ops.gemm(xk, sh.get("wkv", [at.k_proj.weight, at.v_proj.weight]),
                 bias=sh.cat_f32("bkv", [at.k_proj.bias, at.v_proj.bias]), out=KV)
        O = ws.get(f"{pfx}.O", (B * nq, dout), bf)
        ops.attention_fwd_generic(Qp, KV[:, :dout], KV[:, dout:], O, B=B, Sq=nq, Skv=S, H=H, head_dim=hd, bsq=0,
                                  bsk=S * 2 * dout, bsv=S * 2 * dout, bso=nq * dout, scale=1.0 / math.sqrt(hd))
        Y = ws.get(f"{pfx}.Y", (B * nq, dout), bf)
        ops.gemm(O, sh.get("wo", [at.output_proj.weight]), bias=at.output_proj.bias, out=Y)
        out = torch.empty((B * nq, dout), device=self.device, dtype=f32)
        ops.add_layernorm_fwd(None, Y, None, None, out, m.ln_post.weight, m.ln_post.bias, None, None, B * nq, dout,
                              m.ln_post.eps)
        return out.view(B, nq, dout)


class TextDecoderRuntime:
    """CoCaTextDecoder (models/coca/text_decoder.py:66-203)."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        dev = mod.embeddings.token_embeddings.weight.device
        self.stack = LayerStack(mod.transformer_decoder.layer, "ctxt", dev)
        self._idx = None

    def forward(self, input_ids: torch.Tensor, mask_u8: Optional[torch.Tensor], S: int):
        """input_ids int64 [B, S-1 (embed_cls) | S]; mask_u8 [B, S, S] or None (plain causal).
        Returns (pooled fp32 [B, out_dim], tokens fp32 [B, S-1 | S, d])."""
        m, st = self.mod, self.stack
        ws, sh, d = st.ws, st.sh, st.d
        emb = m.embeddings
        ids = input_ids.long().contiguous()
        B = ids.shape[0]
        X0 = ws.get("ctxt.X0", (B * S, d), torch.float32)
        ops.coca_text_embed_fwd(ids, emb.token_embeddings.weight, emb.cls_embedding, emb.position_embeddings, X0, B, S, d,
                                emb.token_embeddings.weight.shape[0])
        st.run(X0, B, S, causal=mask_u8 is None, mask=mask_u8)
        f32, bf = torch.float32, torch.bfloat16
        ln_final = getattr(m, "ln_final", None)
        pooled_b = ws.get("ctxt.POOLb", (B, d), bf)
        if m.embed_cls:
            XF, _, _ = st.finish(B, S, None)
            if self._idx is None or self._idx.numel() != B:
                self._idx = torch.full((B,), S - 1, dtype=torch.int32, device=st.device)
            if ln_final is not None:   # LayerNorm of the CLS row only (:186-189): gathered rows
                ops.add_layernorm_fwd(XF, None, None, pooled_b, None, ln_final.weight, ln_final.bias, None, None, B, d,
                                      ln_final.eps, row_idx=self._idx, rows_per_group=S)
            else:
                ops.gather_rows_cast(XF, pooled_b, B, S, S - 1, d)
            tokens = XF.view(B, S, d)[:, :-1]
        else:
            if ln_final is None:
                raise MMBError("CoCaTextDecoder(embed_cls=False) requires final_layer_norm_eps (reference asserts too)")
            XF, LAST, _ = st.finish(B, S, ln_final)
            idx = torch.empty(B, dtype=torch.int32, device=st.device)
            ops.argmax_tokens(ids, idx, B, S)
            rows = LAST.view(B, S, d)[torch.arange(B, device=st.device), idx.long()]   # [B, d] gather: plumbing
            ops.cast_bf16(rows.contiguous().view(-1), pooled_b.view(-1))
            tokens = LAST.view(B, S, d)
        if m.text_projection is not None:
            pooled = torch.empty((B, m.text_projection.weight.shape[0]), device=st.device, dtype=f32)
            ops.gemm(pooled_b, sh.get("tproj", [m.text_projection.weight]), bias=m.text_projection.bias,
                     epilogue=ops.EPI_F32, out=pooled)
        else:
            pooled = pooled_b.float()
        return pooled, tokens


class MultimodalDecoderRuntime:
    """CoCaMultimodalDecoder (models/coca/multimodal_decoder.py:15-108)."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        dev = mod.transformer_decoder.layer[0].attention.q_proj.weight.device
        self.stack = LayerStack(mod.transformer_decoder.layer, "cmm", dev)

    def forward(self, texts: torch.Tensor, images: torch.Tensor, return_hidden: bool = False):
        """return_hidden: skip the vocabulary projection and return (hidden bf16 [B*S, d], bf16 weight [V, d]) — the
        operands of the fused Linear -> CrossEntropy kernel (CoCaForPretraining never needs the [B, S, V] logits)."""
        m, st = self.mod, self.stack
        ws, sh, d = st.ws, st.sh, st.d
        B, S, _ = texts.shape
        _, Si, dv = images.shape
        X0 = ws.get("cmm.X0", (B * S, d), torch.float32)
        X0.view(B, S, d).copy_(texts)                 # [B, S, d] slice of the text decoder's stream -> contiguous rows
        enc = ws.get("cmm.ENC", (B * Si, dv), torch.bfloat16)
        ops.cast_bf16(images.contiguous().float().view(-1), enc.view(-1))
        st.run(X0, B, S, causal=True, enc=enc, S_enc=Si)
        fln = m.transformer_decoder.final_layer_norm
        XF, LAST, LASTb = st.finish(B, S, fln, want_bf16=m.output_projection is not None)
        if m.output_projection is None:
            if return_hidden:
                raise MMBError("return_hidden needs an output projection (the vocabulary head)")
            return (LAST if fln is not None else XF).view(B, S, d)
        if LASTb is None:
            LASTb = ws.get("cmm.LASTb", (B * S, d), torch.bfloat16)
            ops.cast_bf16(XF.view(-1), LASTb.view(-1))
        if return_hidden:
            return LASTb, sh.get("oproj", [m.output_projection.weight])
        V = m.output_projection.weight.shape[0]
        out = torch.empty((B * S, V), device=st.device, dtype=torch.float32)
        ops.gemm(LASTb, sh.get("oproj", [m.output_projection.weight]), bias=m.output_projection.bias,
                 epilogue=ops.EPI_F32, out=out)
        return out.view(B, S, V)
