"""Runtime of the CoCa model family (BASELINE.json config 5 / SURVEY.md §8 a14 + f3 as a training step), one per module
for both grad modes: forwards that keep what the backward needs + explicit backward schedules, behind torch.autograd
Functions, so that `CoCaModel` / `CoCaForPretraining` train with ``loss.backward()`` like the reference
(models/coca/coca_model.py:69-130, 398-454 under autograd); under torch.no_grad() the same forwards keep nothing.

All layer stacks run on ``engine.TransformerStack`` (the CLIP towers' fused schedule and kernels) through
``engine.ModuleStack``, which also owns the parameter store, the final residual add and the backward's entry:
  vision encoder      : packed `input_proj` self-attention (tensor-core fwd / bwd), erf-GELU MLP, optional final LayerNorm
                        (modules/encoders/vision_transformer.py:56-89, patch_embedding.py:104-154)
  text decoder        : separate q / k / v projections presented as one packed operand, the [B, S, S] causal x padding
                        mask on the general attention kernels (fwd: mma.sync; bwd: SIMT while a head fits in shared
                        memory, K / V-streamed tensor cores at longer lengths), CLS row -> ln_final -> projection
                        (models/coca/text_decoder.py:141-203)
  multimodal decoder  : causal self-attention (tensor cores) + cross-attention to the pooled image tokens (general kernels) +
                        MLP per layer, final LayerNorm (models/coca/multimodal_decoder.py:86-108)
  attention pooler    : LayerNorm-ed keys / values, batch-shared learned queries (their gradient is summed over the batch:
                        fp32 atomics on the resident path, fixed-order per-chunk sums on the streamed one, e.g. 576 image
                        tokens at 336 px), ln_post (modules/layers/attention_pooler.py:48-72)
  vocabulary head     : Linear -> CrossEntropy(ignore_index) with materialised fp32 logits in training (the forward-only
                        path keeps the fused statistics GEMM), backward = d logits kernel + two GEMMs
Every training forward keeps its activations in its own Workspace (held by the autograd node).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
from torch import nn

from . import ops
from ._lib import MMBError
from .engine import ModuleStack, ParamStore, Workspace, as_f32, patch_embed_bwd, patch_embed_fwd
from .modules.layers.stochastic_depth import drop_path_scales
from .modules.masking.random_masking import patch_keep_indices


# ---------------------------------------------------------------------------------------------------------------------
# One runtime per module.  `forward(data, diff) -> (outputs, save)` / `backward(save, *d outputs)` are driven by
# engine.run under autograd; `infer(...)` is the torch.no_grad() call: the same front end, stack and finish without a
# save Workspace (scratch in the runtime's workspace, returned tensors allocated per call), then the tails only
# inference has.  A backward reads only its own save, so no_grad calls may run between a forward and its backward.
class VisionTrainRuntime:
    """VisionTransformer (modules/encoders/vision_transformer.py:56-89).  Output: last_hidden_state [B*S, d]."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.s = ModuleStack(mod, mod.encoder.layer, "cvit")
        self.store = self.s.store

    def _forward(self, images, image_patches_mask, save: Optional[Workspace], hidden: List[torch.Tensor]):
        """hidden: receives hidden_states (X0, each layer's output, XF)."""
        emb, s, st = self.mod.embeddings, self.s, self.store
        d, conv = s.d, emb.conv_projection
        st.refresh()
        drop = patch_keep_indices(emb, images.shape[0], images.device)   # training with patch_drop_rate
        keep = drop[0] if drop is not None else None
        scales = drop_path_scales(s.layers, images.shape[0], images.device)   # training with drop_path_rate
        X0, B, S, P, pm = patch_embed_fwd(images, conv, st.shadow2d(conv.weight),
                                          emb.cls_token if emb.include_cls_embed else None, emb.position_embeddings,
                                          emb.mask_token, image_patches_mask, s.ws, save if save is not None else s.ws,
                                          "cvit", keep=keep)
        XM, Y = s.stack.forward(X0, B, S, save, scales=scales, hidden=hidden)
        XF, LAST = s.finish(XM, Y, B, S, self.mod.encoder.final_layer_norm, save, scales)
        hidden.append(XF.view(B, S, d))
        return (LAST if LAST is not None else XF), (B, S, P, pm, keep)

    def forward(self, data, diff):
        """data: (images, image_patches_mask, the caller's list that receives hidden_states)."""
        images, image_patches_mask, hidden = data
        save = Workspace(self.s.device)
        last, (save.B, save.S, save.P, save.pm, save.keep) = self._forward(images, image_patches_mask, save, hidden)
        return (last,), save

    def infer(self, images, image_patches_mask=None):
        from .modules.layers.transformer import TransformerOutput

        hidden: List[torch.Tensor] = []
        last, _ = self._forward(images, image_patches_mask, None, hidden)
        return TransformerOutput(last_hidden_state=last.view(hidden[-1].shape), pooler_output=None, hidden_states=hidden,
                                 attentions=None)

    def backward(self, save, dOUT):
        emb, s = self.mod.embeddings, self.s
        d, B, S = s.d, save.B, save.S
        M = B * S
        fln = self.mod.encoder.final_layer_norm
        dOUT = as_f32(dOUT, (M, d))
        G, Gb, done = s.start_backward(save, M, fln, dOUT if fln is not None else None, None if fln is not None else dOUT)
        G = s.stack.backward(G, Gb, B, S, top_bias_done=done, save=save)
        patch_embed_bwd(G, emb.conv_projection, emb.cls_token if emb.include_cls_embed else None,
                        emb.position_embeddings, emb.mask_token, save.pm, B, S, save.P, self.store, s.ws, save, "cvit",
                        keep=save.keep)
        return ()


class PoolerTrainRuntime:
    """AttentionPooler (modules/layers/attention_pooler.py:16-72): learned queries cross-attend to the LayerNorm-ed
    input; the query projection is batch independent and computed once per call for [n_queries, d].
    Input x [B, S, d_in] (differentiable)."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        at = mod.attn
        kv = [at.k_proj.weight, at.v_proj.weight, at.k_proj.bias, at.v_proj.bias]   # first: packable
        self.store = st = ParamStore(kv + [p for p in mod.parameters() if all(p is not q for q in kv)])
        self.kv_w = st.pack([at.k_proj.weight, at.v_proj.weight])
        self.kv_b = st.pack([at.k_proj.bias, at.v_proj.bias], fp32=True)
        self.ws = Workspace(st.device)
        self.device = st.device

    def _dims(self):
        m = self.mod
        nq, dout = m.query.shape
        H = m.attn.num_heads
        return nq, dout, H, dout // H

    def _forward(self, x, save: Optional[Workspace]):
        m, st = self.mod, self.store
        at = m.attn
        B, S, din = x.shape
        nq, dout, H, hd = self._dims()
        bf, f32 = torch.bfloat16, torch.float32
        st.refresh()
        keep = save if save is not None else self.ws
        x32 = x.contiguous().float().view(B * S, din)
        xk = keep.get("xk", (B * S, din), bf)
        ops.add_layernorm_fwd(x32, None, None, xk, None, m.ln_k.weight, m.ln_k.bias, keep.get("mk", (B * S,), f32),
                              keep.get("rk", (B * S,), f32), B * S, din, m.ln_k.eps)
        qn = keep.get("qn", (nq, dout), bf)
        ops.add_layernorm_fwd(m.query.data, None, None, qn, None, m.ln_q.weight, m.ln_q.bias, keep.get("mq", (nq,), f32),
                              keep.get("rq", (nq,), f32), nq, dout, m.ln_q.eps)
        Qp = keep.get("Qp", (nq, dout), bf)
        ops.gemm(qn, st.shadow(at.q_proj.weight), bias=at.q_proj.bias, out=Qp)
        KV = keep.get("KV", (B * S, 2 * dout), bf)
        ops.gemm(xk, st.shadow(self.kv_w), bias=self.kv_b, out=KV)
        O = keep.get("O", (B * nq, dout), bf)
        ops.attention_fwd_generic(Qp, KV[:, :dout], KV[:, dout:], O, B=B, Sq=nq, Skv=S, H=H, head_dim=hd, bsq=0,
                                  bsk=S * 2 * dout, bsv=S * 2 * dout, bso=nq * dout, scale=1.0 / math.sqrt(hd))
        Y = self.ws.get("Y", (B * nq, dout), bf)
        ops.gemm(O, st.shadow(at.output_proj.weight), bias=at.output_proj.bias, out=Y)
        Y32 = save.get("Y32", (B * nq, dout), f32) if save is not None else None
        out = torch.empty((B * nq, dout), device=self.device, dtype=f32)
        ops.add_layernorm_fwd(None, Y, Y32, None, out, m.ln_post.weight, m.ln_post.bias, keep.get("mp", (B * nq,), f32),
                              keep.get("rp", (B * nq,), f32), B * nq, dout, m.ln_post.eps)
        return out, x32

    def forward(self, data, diff):
        (x,) = diff
        hd = self._dims()[3]
        if hd not in (64, 96, 128):
            raise MMBError(f"unsupported pooler head_dim {hd}")
        save = Workspace(self.device)
        out, save.x32 = self._forward(x, save)
        save.B, save.S, save.din = x.shape
        return (out,), save

    def infer(self, x: torch.Tensor) -> torch.Tensor:
        """x fp32 [B, S, d_in] -> fp32 [B, n_queries, d_out]."""
        nq, dout = self.mod.query.shape
        return self._forward(x, None)[0].view(x.shape[0], nq, dout)

    def backward(self, save, dOUT):
        m, st = self.mod, self.store
        at = m.attn
        B, S, din = save.B, save.S, save.din
        nq, dout, H, hd = self._dims()
        bf, f32 = torch.bfloat16, torch.float32
        n = B * nq
        g = lambda name, shape, dt: save.get(name, shape, dt)  # noqa: E731
        dYb = self.ws.get("dYb", (n, dout), bf)
        ops.layernorm_bwd(g("Y32", (n, dout), f32), None, as_f32(dOUT, (n, dout)), g("mp", (n,), f32), g("rp", (n,), f32),
                          m.ln_post.weight, None, None, dYb, st.grad(m.ln_post.weight), st.grad(m.ln_post.bias), n, dout,
                          gsum=st.grad(at.output_proj.bias))
        O, KV = g("O", (n, dout), bf), g("KV", (B * S, 2 * dout), bf)
        Qp, qn, xk = g("Qp", (nq, dout), bf), g("qn", (nq, dout), bf), g("xk", (B * S, din), bf)
        ops.gemm(dYb, O, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(at.output_proj.weight),
                 splits=ops.wgrad_splits(dout, dout, n), accumulate=True)
        dO = self.ws.get("dO", (n, dout), bf)
        ops.gemm(dYb, st.shadow(at.output_proj.weight), b_mn=True, out=dO)
        dQ32 = torch.zeros((nq, dout), device=self.device, dtype=f32)   # summed over the batch by the kernel
        dKV = self.ws.get("dKV", (B * S, 2 * dout), bf)
        ops.attention_bwd_generic(Qp, KV[:, :dout], KV[:, dout:], dO, dKV[:, :dout], dKV[:, dout:], dq=None, dq_f32=dQ32,
                                  B=B, Sq=nq, Skv=S, H=H, head_dim=hd, bsq=0, bsk=S * 2 * dout, bsv=S * 2 * dout,
                                  bso=nq * dout, scale=1.0 / math.sqrt(hd))
        dQb = ops.cast_bf16(dQ32)
        ops.gemm(dQb, qn, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(at.q_proj.weight), accumulate=True)
        ops.colsum_bf16(dQb, st.grad(at.q_proj.bias), nq, dout, dout)
        dqn = self.ws.get("dqn", (nq, dout), bf)
        ops.gemm(dQb, st.shadow(at.q_proj.weight), b_mn=True, out=dqn)
        gq = st.grad(m.query)
        ops.layernorm_bwd(m.query.data, dqn, None, g("mq", (nq,), f32), g("rq", (nq,), f32), m.ln_q.weight, gq, gq, None,
                          st.grad(m.ln_q.weight), st.grad(m.ln_q.bias), nq, dout)
        ops.gemm(dKV, xk, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(self.kv_w),
                 splits=ops.wgrad_splits(2 * dout, din, B * S), accumulate=True)
        ops.colsum_bf16(dKV, st.grad(self.kv_b), B * S, 2 * dout, 2 * dout)
        dxk = self.ws.get("dxk", (B * S, din), bf)
        ops.gemm(dKV, st.shadow(self.kv_w), b_mn=True, out=dxk)
        dx = torch.empty((B * S, din), device=self.device, dtype=f32)
        ops.layernorm_bwd(save.x32, dxk, None, g("mk", (B * S,), f32), g("rk", (B * S,), f32), m.ln_k.weight, None, dx,
                          None, st.grad(m.ln_k.weight), st.grad(m.ln_k.bias), B * S, din)
        return (dx.view(B, S, din),)


class TextDecoderTrainRuntime:
    """CoCaTextDecoder (models/coca/text_decoder.py:66-203).  Training (embed_cls=True, bias-free text_projection)
    outputs: pooled [B, out_dim] (projected ln_final(CLS row)) and XF [B*S, d] (tokens = XF[:, :-1])."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.s = ModuleStack(mod, mod.transformer_decoder.layer, "ctxt", fp32_only=list(mod.embeddings.parameters()))
        self.store = self.s.store
        self._idx = None

    def _forward(self, input_ids, mask_u8, S: int, save: Optional[Workspace]):
        """-> (pooled fp32 [B, out_dim], tokens fp32 [B, S-1 | S, d], XF fp32 [B*S, d], ids, CLS row index)."""
        m, s, st = self.mod, self.s, self.store
        d = s.d
        emb = m.embeddings
        ids = input_ids.long().contiguous()
        B = ids.shape[0]
        bf, f32 = torch.bfloat16, torch.float32
        st.refresh()
        keep = save if save is not None else s.ws
        X0 = torch.empty((B * S, d), device=s.device, dtype=f32) if save is not None else s.ws.get("ctxt.X0", (B * S, d), f32)
        ops.coca_text_embed_fwd(ids, emb.token_embeddings.weight, emb.cls_embedding, emb.position_embeddings, X0, B, S, d,
                                emb.token_embeddings.weight.shape[0])
        # a [B, S, S] mask already contains the causal structure
        XM, Y = s.stack.forward(X0, B, S, save, causal=mask_u8 is None, mask3=mask_u8)
        ln = getattr(m, "ln_final", None)
        POOLb = keep.get("ctxt.POOLb", (B, d), bf)
        idx = None
        if m.embed_cls:
            XF, _ = s.finish(XM, Y, B, S, None, save, None)
            if self._idx is None or self._idx.numel() != B:
                self._idx = torch.full((B,), S - 1, dtype=torch.int32, device=s.device)
            idx = self._idx
            if ln is not None:    # LayerNorm of the CLS row only (:186-189): gathered rows
                ops.add_layernorm_fwd(XF, None, save.get("ctxt.XSEL", (B, d), f32) if save is not None else None, POOLb,
                                      None, ln.weight, ln.bias, keep.get("ctxt.mL", (B,), f32),
                                      keep.get("ctxt.rL", (B,), f32), B, d, ln.eps, row_idx=idx, rows_per_group=S)
            else:
                ops.gather_rows_cast(XF, POOLb, B, S, S - 1, d)
            tokens = XF.view(B, S, d)[:, :-1]
        else:   # inference only
            if ln is None:
                raise MMBError("CoCaTextDecoder(embed_cls=False) requires final_layer_norm_eps (reference asserts too)")
            XF, LAST = s.finish(XM, Y, B, S, ln, save, None)
            am = torch.empty(B, dtype=torch.int32, device=s.device)
            ops.argmax_tokens(ids, am, B, S)
            rows = LAST.view(B, S, d)[torch.arange(B, device=s.device), am.long()]   # [B, d] gather: plumbing
            ops.cast_bf16(rows.contiguous().view(-1), POOLb.view(-1))
            tokens = LAST.view(B, S, d)
        if m.text_projection is not None:
            pooled = torch.empty((B, m.text_projection.weight.shape[0]), device=s.device, dtype=f32)
            ops.gemm(POOLb, st.shadow(m.text_projection.weight), bias=m.text_projection.bias, epilogue=ops.EPI_F32,
                     out=pooled)
        else:
            pooled = POOLb.float()
        return pooled, tokens, XF, ids, idx

    def forward(self, data, diff):
        m = self.mod
        if not m.embed_cls:
            raise NotImplementedError("training CoCaTextDecoder(embed_cls=False) is not on the accelerated path")
        if m.text_projection is None or m.text_projection.bias is not None:
            raise NotImplementedError("training expects the bias-free text_projection of the reference builder")
        input_ids, mask_u8, S = data
        save = Workspace(self.s.device)
        pooled, _, XF, save.ids, save.idx = self._forward(input_ids, mask_u8, S, save)
        save.B, save.S = input_ids.shape[0], S
        return (pooled, XF), save

    def infer(self, input_ids: torch.Tensor, mask_u8: Optional[torch.Tensor], S: int):
        """input_ids int64 [B, S-1 (embed_cls) | S]; mask_u8 [B, S, S] or None (plain causal).
        Returns (pooled fp32 [B, out_dim], tokens fp32 [B, S-1 | S, d])."""
        return self._forward(input_ids, mask_u8, S, None)[:2]

    def backward(self, save, dpooled, dXF):
        m, s, st = self.mod, self.s, self.store
        d, B, S = s.d, save.B, save.S
        M = B * S
        bf, f32 = torch.bfloat16, torch.float32
        emb = m.embeddings
        G, Gb, _ = s.start_backward(save, M, None, None, as_f32(dXF, (M, d)))
        if dpooled is not None:
            ln = getattr(m, "ln_final", None)
            W = m.text_projection.weight
            dPb = ops.cast_bf16(as_f32(dpooled, (B, W.shape[0])))
            POOLb = save.get("ctxt.POOLb", (B, d), bf)
            ops.gemm(dPb, POOLb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(W), accumulate=True)
            dL = torch.empty((B, d), device=s.device, dtype=f32)
            ops.gemm(dPb, st.shadow(W), b_mn=True, epilogue=ops.EPI_F32, out=dL)
            if ln is not None:
                ops.layernorm_bwd(save.get("ctxt.XSEL", (B, d), f32), None, dL, save.get("ctxt.mL", (B,), f32),
                                  save.get("ctxt.rL", (B,), f32), ln.weight, G, G, None, st.grad(ln.weight),
                                  st.grad(ln.bias), B, d, row_idx=save.idx, rows_per_group=S)
            else:
                ops.scatter_rows_add(dL, G, B, S, S - 1, d)
            ops.cast_bf16(G, Gb)
        G = s.stack.backward(G, Gb, B, S, top_bias_done=False, save=save)
        ops.batch_sum(G, st.grad(emb.position_embeddings), B, S * d, S * d)
        ops.batch_sum(G.view(-1)[(S - 1) * d:], st.grad(emb.cls_embedding), B, S * d, d)
        tok = emb.token_embeddings
        Gtok = G.view(B, S, d)[:, :S - 1].contiguous().view(-1, d)       # rows of the real tokens (slice copy: plumbing)
        ops.scatter_rows_idx_add(Gtok, save.ids.reshape(-1).contiguous(), st.grad(tok.weight), d)
        if tok.padding_idx is not None:
            ops.zero_(st.grad(tok.weight)[tok.padding_idx])
        return ()


class MultimodalDecoderTrainRuntime:
    """CoCaMultimodalDecoder (models/coca/multimodal_decoder.py:15-108).  Training runs up to the final LayerNorm (the
    vocabulary projection + cross-entropy is ``LinearCrossEntropyFunction``).  Inputs: texts [B, S, d], images
    [B, Si, d_kv]."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.s = ModuleStack(mod, mod.transformer_decoder.layer, "cmm")
        self.store = self.s.store

    def _forward(self, texts, images, save: Optional[Workspace], want_bf16: bool = False):
        """-> (XF, LAST or None, LASTb: bf16 copy of LAST when want_bf16 and a final LayerNorm exists, else None)."""
        s = self.s
        d = s.d
        B, S, _ = texts.shape
        _, Si, dv = images.shape
        self.store.refresh()
        X0 = torch.empty((B * S, d), device=s.device, dtype=torch.float32) if save is not None else s.ws.get(
            "cmm.X0", (B * S, d), torch.float32)
        X0.view(B, S, d).copy_(texts)                 # [B, S, d] slice of the text decoder's stream -> contiguous rows
        enc = (save if save is not None else s.ws).get("cmm.ENC", (B * Si, dv), torch.bfloat16)
        ops.cast_bf16(images.contiguous().float().view(-1), enc.view(-1))
        XM, Y = s.stack.forward(X0, B, S, save, causal=True, enc=enc, S_enc=Si)
        fln = self.mod.transformer_decoder.final_layer_norm
        LASTb = s.ws.get("cmm.LASTb", (B * S, d), torch.bfloat16) if (fln is not None and want_bf16) else None
        XF, LAST = s.finish(XM, Y, B, S, fln, save, None, LASTb=LASTb)
        return XF, LAST, LASTb

    def forward(self, data, diff):
        texts, images = diff
        save = Workspace(self.s.device)
        XF, LAST, _ = self._forward(texts, images, save)
        save.B, save.S, _ = texts.shape
        _, save.Si, save.dv = images.shape
        return ((LAST if LAST is not None else XF),), save

    def infer(self, texts: torch.Tensor, images: torch.Tensor, return_hidden: bool = False):
        """return_hidden: skip the vocabulary projection and return (hidden bf16 [B*S, d], bf16 weight [V, d]) — the
        operands of the fused Linear -> CrossEntropy kernel (CoCaForPretraining never needs the [B, S, V] logits)."""
        m, s = self.mod, self.s
        B, S, _ = texts.shape
        d = s.d
        XF, LAST, LASTb = self._forward(texts, images, None, want_bf16=m.output_projection is not None)
        if m.output_projection is None:
            if return_hidden:
                raise MMBError("return_hidden needs an output projection (the vocabulary head)")
            return (LAST if LAST is not None else XF).view(B, S, d)
        if LASTb is None:
            LASTb = s.ws.get("cmm.LASTb", (B * S, d), torch.bfloat16)
            ops.cast_bf16(XF.view(-1), LASTb.view(-1))
        W = self.store.shadow(m.output_projection.weight)
        if return_hidden:
            return LASTb, W
        V = m.output_projection.weight.shape[0]
        out = torch.empty((B * S, V), device=s.device, dtype=torch.float32)
        ops.gemm(LASTb, W, bias=m.output_projection.bias, epilogue=ops.EPI_F32, out=out)
        return out.view(B, S, V)

    def backward(self, save, dOUT):
        s = self.s
        d, B, S = s.d, save.B, save.S
        M = B * S
        fln = self.mod.transformer_decoder.final_layer_norm
        dOUT = as_f32(dOUT, (M, d))
        G, Gb, done = s.start_backward(save, M, fln, dOUT if fln is not None else None, None if fln is not None else dOUT)
        G = s.stack.backward(G, Gb, B, S, top_bias_done=done, save=save)
        return (G.view(B, S, d).clone(), save.dENC.view(B, save.Si, save.dv))


class LinearF32Function(torch.autograd.Function):
    """y = x @ W^T (+ b) for a 2-D fp32 x, tensor-core GEMMs both ways.  The output width is padded to a multiple of 8
    internally (bf16 rows of d y must be 16-byte multiples for the TMA operands of the backward GEMMs)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        N, K = weight.shape
        Np = (N + 7) // 8 * 8
        dev = x.device
        xb = ops.cast_bf16(x.detach().contiguous().float())
        wb = ops.cast_bf16(weight.detach().contiguous())
        bp = bias.detach().float().contiguous() if bias is not None else None
        if Np != N:
            wp = torch.zeros((Np, K), device=dev, dtype=torch.bfloat16)
            wp[:N].copy_(wb)
            wb = wp
            if bp is not None:
                b2 = torch.zeros(Np, device=dev, dtype=torch.float32)
                b2[:N].copy_(bp)
                bp = b2
        out = torch.empty((xb.shape[0], Np), device=dev, dtype=torch.float32)
        ops.gemm(xb, wb, bias=bp, epilogue=ops.EPI_F32, out=out)
        ctx.save_for_backward(xb, wb)
        ctx.has_bias, ctx.N = bias is not None, N
        return out[:, :N]

    @staticmethod
    def backward(ctx, dy):
        xb, wb = ctx.saved_tensors
        N, Np = ctx.N, wb.shape[0]
        dyf = dy.contiguous().float()
        if Np != N:
            pad = torch.zeros((dyf.shape[0], Np), device=dy.device, dtype=torch.float32)
            pad[:, :N].copy_(dyf)
            dyf = pad
        dyb = ops.cast_bf16(dyf)
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(xb.shape, device=dy.device, dtype=torch.float32)
            ops.gemm(dyb, wb, b_mn=True, epilogue=ops.EPI_F32, out=dx)
        if ctx.needs_input_grad[1]:
            gw = torch.empty(wb.shape, device=dy.device, dtype=torch.float32)
            ops.gemm(dyb, xb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=gw)
            dW = gw[:N]
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = torch.zeros(Np, device=dy.device, dtype=torch.float32)
            ops.colsum_bf16(dyb, gb, dyb.shape[0], Np, Np)
            db = gb[:N]
        return dx, dW, db


class LinearCrossEntropyFunction(torch.autograd.Function):
    """mean CrossEntropy(ignore_index)(hidden @ W^T (+ b), labels) — the captioning head (coca_model.py:443-454).
    Training materialises the fp32 logits [M, V] once (saved for the backward); the label-free forward path of
    CoCaForPretraining keeps the fused statistics GEMM."""

    @staticmethod
    def forward(ctx, hidden, weight, bias, labels, ignore_index):
        dev = hidden.device
        hb = ops.cast_bf16(hidden.detach().contiguous().float())
        M, d = hb.shape
        V = weight.shape[0]
        Vp = (V + 7) // 8 * 8
        wb = ops.cast_bf16(weight.detach().contiguous())
        if Vp != V:
            wp = torch.zeros((Vp, d), device=dev, dtype=torch.bfloat16)
            wp[:V].copy_(wb)
            wb = wp
        bp = None
        if bias is not None:
            bp = torch.zeros(Vp, device=dev, dtype=torch.float32)
            bp[:V].copy_(bias.detach().float())
        logits = torch.empty((M, Vp), device=dev, dtype=torch.float32)
        ops.gemm(hb, wb, bias=bp, epilogue=ops.EPI_F32, out=logits)
        lab = labels.reshape(-1).contiguous().long()
        accum = torch.zeros(2, device=dev, dtype=torch.float32)
        ops.ce_labels(logits[:, :V], lab, 1, ignore_index, M, V, None, accum)
        ctx.save_for_backward(hb, wb, logits, lab, accum)
        ctx.meta = (V, Vp, int(ignore_index), bias is not None)
        return accum[0] / accum[1]

    @staticmethod
    def backward(ctx, dloss):
        hb, wb, logits, lab, accum = ctx.saved_tensors
        V, Vp, ignore_index, has_bias = ctx.meta
        M, d = hb.shape
        dev = hb.device
        dlog = torch.zeros((M, Vp), device=dev, dtype=torch.bfloat16)
        ops.ce_labels_bwd(logits[:, :V], lab, 1, ignore_index, M, V, accum, 1.0, dlog[:, :V],
                          gscale=dloss.detach().float().reshape(1).contiguous())
        dh = dW = db = None
        if ctx.needs_input_grad[0]:
            dh = torch.empty((M, d), device=dev, dtype=torch.float32)
            ops.gemm(dlog, wb, b_mn=True, epilogue=ops.EPI_F32, out=dh)
        if ctx.needs_input_grad[1]:
            gw = torch.empty((Vp, d), device=dev, dtype=torch.float32)
            ops.gemm(dlog, hb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=gw, splits=ops.wgrad_splits(Vp, d, M))
            dW = gw[:V]
        if has_bias and ctx.needs_input_grad[2]:
            gb = torch.zeros(Vp, device=dev, dtype=torch.float32)
            ops.colsum_bf16(dlog, gb, M, Vp, Vp)
            db = gb[:V]
        return dh, dW, db, None, None


def linear_f32(x: torch.Tensor, linear: nn.Linear) -> torch.Tensor:
    """linear(x) over the last dim of x (any leading shape)."""
    lead = x.shape[:-1]
    y = LinearF32Function.apply(x.reshape(-1, x.shape[-1]), linear.weight, linear.bias)
    return y.view(*lead, -1)


def linear_cross_entropy(hidden: torch.Tensor, linear: nn.Linear, labels: torch.Tensor, ignore_index: int) -> torch.Tensor:
    return LinearCrossEntropyFunction.apply(hidden.reshape(-1, hidden.shape[-1]), linear.weight, linear.bias, labels,
                                            ignore_index)
