"""Runtime of the FLAVA encoders (BASELINE.json config 3, forward and training step), one per encoder for both grad
modes: forward that keeps what the backward needs + the explicit backward schedule, behind torch.autograd Functions so
that the drop-in modules train with ``loss.backward()`` exactly like the reference's (models/flava/model.py:127-298
under autograd); under torch.no_grad() the same forward keeps nothing and returns the reference's ``TransformerOutput``
(every tensor allocated per call; ``attentions`` on request, recomputed from the packed QKV and the row LSE by one
extra kernel per layer: DESIGN.md §10).

The layer stack is the CLIP towers' ``engine.TransformerStack`` (same kernels, same fused schedule), reached through
``engine.ModuleStack`` as CoCa's stacks are: the separate query / key / value Linears are presented to it as one packed
in-projection (``ParamStore.pack``), the MLP activation is the exact-erf GELU epilogue pair, and the text tower's
key-padding mask goes to the masked attention kernels (forward and fused single-pass backward).  What is specific to FLAVA is on either side of the stack:

  image  : im2col + patch GEMM (+bias) -> [cls | mask_token or patch] + pos      bwd: mmb_vit_assemble_bwd, batch sums,
           patch-projection weight / bias gradients                                   (image_encoder.py:139-175)
  text   : LayerNorm(word + pos + type) with pad-derived key mask                 bwd: mmb_bert_embed_ln_bwd (recomputes
           the pre-norm sum, scatter-adds into the three tables)                      (text_embedding.py:70-104)
  mm     : two projections -> [cls | image | text]                              bwd: mmb_split_tokens_cast, projection
           gradients, gradients w.r.t. both incoming hidden states                    (model.py:283-298)
  all    : final LayerNorm -> last_hidden_state; its input is hidden_states[-1], which the multimodal encoder consumes,
           so BOTH are differentiable outputs.  Pooler / `linear(last_hidden_state[:, 0])` projections are
           ``FirstTokenLinearFunction`` (gather, GEMM, tanh; backward scatters into the dense gradient).

One encoder instance runs twice per pre-training step (unmasked + masked inputs): every training forward keeps its
activations in its OWN Workspace (held by the autograd node, freed after its backward), so any number of forwards may
be in flight.  ``hidden_states[1:-1]`` of a training forward are views of those saved buffers: values are the
reference's, but they carry no autograd history (nothing in the library differentiates through them).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
from torch import nn

from . import ops
from .engine import (ModuleStack, Workspace, _Shadows, as_f32, patch_embed_bwd, patch_embed_fwd, require_head_dim_64,
                     run)
from .modules.layers.transformer import TransformerOutput


class _FlavaRuntime:
    """What the three FLAVA encoder runtimes share around their ModuleStack: the encoder's final LayerNorm and
    pooler, and FLAVAModel's projections of the first token.  One runtime per encoder: `forward(data, diff)` /
    `backward` under autograd (engine.run), `infer(...)` under torch.no_grad(): the same front end and stack without a
    save Workspace, then the pooler.  `data` ends with the caller's list that receives hidden_states."""

    def __init__(self, mod: nn.Module, prefix: str, extra: Sequence[nn.Module] = (),
                 fp32_only: Sequence[nn.Parameter] = ()):
        at = mod.encoder.layer[0].attention
        require_head_dim_64(at.dim_q, at.n_head)
        self.mod = mod
        self.s = ModuleStack(mod, mod.encoder.layer, prefix, extra=extra, fp32_only=fp32_only)
        self.store, self.device = self.s.store, self.s.device
        self.sh = _Shadows(self.device)    # FLAVAModel's projections of the first token (project_first_token)

    def _stack(self, X0, B: int, S: int, kmask, save: Optional[Workspace], hidden: List[torch.Tensor], attns=None):
        """-> (LAST, XF) fp32 [B*S, d]: XF = hidden_states[-1], LAST = layernorm(XF)."""
        s = self.s
        XM, Y = s.stack.forward(X0, B, S, save, kmask=kmask, hidden=hidden, attns=attns)
        XF, LAST = s.finish(XM, Y, B, S, self.mod.layernorm, save, None)
        hidden.append(XF.view(B, S, s.d))
        if save is not None:
            save.B, save.S = B, S
        return LAST, XF

    def _infer(self, X0: torch.Tensor, B: int, S: int, kmask: Optional[torch.Tensor] = None,
               want_attn: bool = False) -> TransformerOutput:
        """want_attn: also return every layer's attention probabilities fp32 [B, H, S, S] (`attentions`), recomputed
        from the packed QKV and the row LSE of the fused attention kernel (mmb_attention_probs)."""
        s, pooler = self.s, self.mod.pooler
        d = s.d
        hidden: List[torch.Tensor] = []
        attns: Optional[List[torch.Tensor]] = [] if want_attn else None
        LAST, _ = self._stack(X0, B, S, kmask, None, hidden, attns)
        pooled = None
        if pooler is not None:
            CLSb = s.ws.get(f"{s.prefix}.CLSb", (B, d), torch.bfloat16)
            ops.gather_rows_cast(LAST, CLSb, B, S, 0, d)
            pooled = torch.empty((B, d), device=self.device, dtype=torch.float32)
            ops.gemm(CLSb, self.store.shadow(pooler.dense.weight), bias=pooler.dense.bias, epilogue=ops.EPI_F32,
                     out=pooled)
            ops.tanh_(pooled)
        return TransformerOutput(last_hidden_state=LAST.view(B, S, d), pooler_output=pooled, hidden_states=hidden,
                                 attentions=attns)

    def project_first_token(self, last_hidden_state: torch.Tensor, linear: nn.Linear, key: str) -> torch.Tensor:
        """linear(last_hidden_state[:, 0, :]) (models/flava/model.py:244-246, 261-263)."""
        B, S, d = last_hidden_state.shape
        CLSb = self.s.ws.get(f"{self.s.prefix}.CLSb2", (B, d), torch.bfloat16)
        ops.gather_rows_cast(last_hidden_state.reshape(B * S, d), CLSb, B, S, 0, d)
        out = torch.empty((B, linear.weight.shape[0]), device=self.device, dtype=torch.float32)
        ops.gemm(CLSb, self.sh.get(key, [linear.weight]), bias=linear.bias, epilogue=ops.EPI_F32, out=out)
        return out

    def _backward(self, save: Workspace, dLAST: Optional[torch.Tensor], dXF: Optional[torch.Tensor]) -> torch.Tensor:
        """Gradient w.r.t. X0 (fp32 [B*S, d], scratch: consume before the next backward of this encoder); parameter
        gradients are accumulated into the store's flat buffer."""
        s = self.s
        M = save.B * save.S
        G, Gb, done = s.start_backward(save, M, self.mod.layernorm, as_f32(dLAST, (M, s.d)), as_f32(dXF, (M, s.d)))
        return s.stack.backward(G, Gb, save.B, save.S, top_bias_done=done, save=save)


class FlavaImageTrainRuntime(_FlavaRuntime):
    def __init__(self, mod: nn.Module):
        super().__init__(mod, "fimg")

    def _embed(self, pixel_values, image_patches_mask, save: Optional[Workspace]):
        emb, ws, st = self.mod.embeddings, self.s.ws, self.store
        conv = emb.patch_embeddings.projection
        st.refresh()
        return patch_embed_fwd(pixel_values, conv, st.shadow2d(conv.weight), emb.cls_token, emb.position_embeddings,
                               emb.mask_token, image_patches_mask, ws, save if save is not None else ws, "fimg")

    def forward(self, data, diff):
        pixel_values, image_patches_mask, hidden = data
        save = Workspace(self.device)
        X0, B, S, save.P, save.pm = self._embed(pixel_values, image_patches_mask, save)
        return self._stack(X0, B, S, None, save, hidden), save

    def infer(self, pixel_values: torch.Tensor, image_patches_mask: Optional[torch.Tensor] = None,
              want_attn: bool = False) -> TransformerOutput:
        X0, B, S, _, _ = self._embed(pixel_values, image_patches_mask, None)   # X0 is returned as hidden_states[0]
        return self._infer(X0, B, S, want_attn=want_attn)

    def backward(self, save, dLAST, dXF):
        emb = self.mod.embeddings
        G = self._backward(save, dLAST, dXF)
        patch_embed_bwd(G, emb.patch_embeddings.projection, emb.cls_token, emb.position_embeddings, emb.mask_token,
                        save.pm, save.B, save.S, save.P, self.store, self.s.ws, save, "fimg")
        return ()


class FlavaTextTrainRuntime(_FlavaRuntime):
    def __init__(self, mod: nn.Module):
        super().__init__(mod, "ftxt", fp32_only=list(mod.embeddings.parameters()))

    def _embed(self, input_ids, attention_mask, token_type_ids, save: Optional[Workspace]):
        emb, st = self.mod.embeddings, self.store
        d = self.s.d
        ids = input_ids.long().contiguous()
        B, S = ids.shape
        if S > emb.position_embeddings.weight.shape[0]:
            raise ValueError(f"sequence length {S} exceeds max_position_embeddings")
        st.refresh()
        X0 = torch.empty((B * S, d), device=ids.device, dtype=torch.float32)   # hidden_states[0]
        KM = (save if save is not None else self.s.ws).get("ftxt.KM", (B * S,), torch.uint8)
        tt = token_type_ids.long().contiguous() if token_type_ids is not None else None
        V = emb.word_embeddings.weight.shape[0]
        ops.bert_embed_ln_fwd(ids, tt, emb.word_embeddings.weight, emb.position_embeddings.weight,
                              emb.token_type_embeddings.weight, emb.layer_norm.weight, emb.layer_norm.bias, X0, KM,
                              emb.pad_token_id, B, S, d, V, emb.layer_norm.eps)
        if attention_mask is not None:  # user-supplied [B,S] mask (1 = attend) overrides the pad-derived one
            if attention_mask.dim() != 2:
                raise NotImplementedError("only [batch, seq_len] padding masks are supported on the accelerated path")
            KM = (attention_mask != 0).to(torch.uint8).contiguous().view(-1)
        return X0, B, S, KM, ids, tt, V

    def forward(self, data, diff):
        *inputs, hidden = data
        save = Workspace(self.device)
        X0, B, S, KM, save.ids, save.tt, save.V = self._embed(*inputs, save)
        return self._stack(X0, B, S, KM, save, hidden), save

    def infer(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
              token_type_ids: Optional[torch.Tensor] = None, want_attn: bool = False) -> TransformerOutput:
        X0, B, S, KM, _, _, _ = self._embed(input_ids, attention_mask, token_type_ids, None)
        return self._infer(X0, B, S, kmask=KM, want_attn=want_attn)

    def backward(self, save, dLAST, dXF):
        emb, st = self.mod.embeddings, self.store
        d, B, S = self.s.d, save.B, save.S
        G = self._backward(save, dLAST, dXF)
        word = emb.word_embeddings
        ops.bert_embed_ln_bwd(save.ids, save.tt, word.weight, emb.position_embeddings.weight,
                              emb.token_type_embeddings.weight, emb.layer_norm.weight, G, st.grad(word.weight),
                              st.grad(emb.position_embeddings.weight), st.grad(emb.token_type_embeddings.weight),
                              st.grad(emb.layer_norm.weight), st.grad(emb.layer_norm.bias), B, S, d, save.V,
                              emb.layer_norm.eps)
        if word.padding_idx is not None:   # nn.Embedding(padding_idx): that row receives no gradient
            ops.zero_(st.grad(word.weight)[word.padding_idx])
        return ()


class FlavaMMTrainRuntime(_FlavaRuntime):
    """[cls | image_to_mm(image_hidden) | text_to_mm(text_hidden)] -> stack.  The two projection Linears belong to
    FLAVAModel, not to the multimodal encoder; they live in this runtime's ParamStore (image_proj / text_proj None:
    the module was called directly with an already fused token sequence)."""

    def __init__(self, mod: nn.Module, image_proj: Optional[nn.Linear] = None, text_proj: Optional[nn.Linear] = None):
        super().__init__(mod, "fmm", extra=[m for m in (image_proj, text_proj) if m is not None])
        self.image_proj, self.text_proj = image_proj, text_proj

    def _embed(self, diff, save: Optional[Workspace]):
        """-> (X0, B, S, Si, St, di, dt): Si = the fused sequence length and St = 0 for a direct call."""
        ws, st = self.s.ws, self.store
        d = self.s.d
        bf, f32 = torch.bfloat16, torch.float32
        cls = self.mod.cls_token
        off = 1 if cls is not None else 0
        st.refresh()
        if self.image_proj is None:   # direct call: hidden_states [B, S, d] already fused
            (hs,) = diff
            B, Sa, _ = hs.shape
            hs = hs.contiguous().float()
            if cls is None and save is None:
                return hs.view(B * Sa, d), B, Sa, Sa, 0, None, None   # hidden_states[0] is the input itself
            X0 = torch.empty((B * (Sa + off), d), device=hs.device, dtype=f32)
            ops.concat_tokens(cls, hs, hs, X0, B, Sa, 0, d)   # cat(cls, hidden) == concat_tokens(cls, hidden, <empty>)
            return X0, B, Sa + off, Sa, 0, None, None
        image_hidden, text_hidden = diff
        B, Si, di = image_hidden.shape
        Bt, St, dt = text_hidden.shape
        if B != Bt:
            raise ValueError(f"batch mismatch between image ({B}) and text ({Bt}) hidden states")
        keep = save if save is not None else ws
        Ib = keep.get("fmm.Ib", (B * Si, di), bf)
        Tb = keep.get("fmm.Tb", (B * St, dt), bf)
        ops.cast_bf16(image_hidden.contiguous().float().view(-1), Ib.view(-1))
        ops.cast_bf16(text_hidden.contiguous().float().view(-1), Tb.view(-1))
        Pi = ws.get("fmm.Pi", (B * Si, d), f32)
        Pt = ws.get("fmm.Pt", (B * St, d), f32)
        ops.gemm(Ib, st.shadow(self.image_proj.weight), bias=self.image_proj.bias, epilogue=ops.EPI_F32, out=Pi)
        ops.gemm(Tb, st.shadow(self.text_proj.weight), bias=self.text_proj.bias, epilogue=ops.EPI_F32, out=Pt)
        S = Si + St + off
        X0 = torch.empty((B * S, d), device=image_hidden.device, dtype=f32)   # hidden_states[0]
        ops.concat_tokens(cls, Pi, Pt, X0, B, Si, St, d)
        return X0, B, S, Si, St, di, dt

    def forward(self, data, diff):
        (hidden,) = data
        save = Workspace(self.device)
        X0, B, S, save.Si, save.St, save.di, save.dt = self._embed(diff, save)
        return self._stack(X0, B, S, None, save, hidden), save

    def infer(self, *hidden: torch.Tensor, want_attn: bool = False) -> TransformerOutput:
        """hidden: the fused token sequence fp32 [B, S, d] (direct call), or the image and text encoders' hidden
        states (FLAVAModel.encode_mm, models/flava/model.py:283-298: projected by two GEMMs, then [cls | image | text]
        assembled by one kernel)."""
        X0, B, S, _, _, _, _ = self._embed(hidden, None)
        return self._infer(X0, B, S, want_attn=want_attn)

    def backward(self, save, dLAST, dXF):
        ws, st = self.s.ws, self.store
        d, B, S, Si, St = self.s.d, save.B, save.S, save.Si, save.St
        bf, f32 = torch.bfloat16, torch.float32
        cls = self.mod.cls_token
        has_cls = cls is not None
        G = self._backward(save, dLAST, dXF)
        if has_cls:
            ops.batch_sum(G, st.grad(cls), B, S * d, d)
        if self.image_proj is None:
            dH = G.view(B, S, d)[:, (1 if has_cls else 0):].clone()   # strided slice copy: plumbing
            return (dH,)
        dPi = ws.get("fmm.dPi", (B * Si, d), bf)
        dPt = ws.get("fmm.dPt", (B * St, d), bf)
        ops.split_tokens_cast(G, dPi, dPt, B, Si, St, d, has_cls)
        outs = []
        for dP, lin, key, n, din in ((dPi, self.image_proj, "fmm.Ib", B * Si, save.di),
                                     (dPt, self.text_proj, "fmm.Tb", B * St, save.dt)):
            Xb = save.get(key, (n, din), bf)
            ops.gemm(dP, Xb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(lin.weight),
                     splits=ops.wgrad_splits(d, din, n), accumulate=True)
            ops.colsum_bf16(dP, st.grad(lin.bias), n, d, d)
            dX = torch.empty((n, din), device=self.device, dtype=f32)
            ops.gemm(dP, st.shadow(lin.weight), b_mn=True, epilogue=ops.EPI_F32, out=dX)
            outs.append(dX)
        return (outs[0].view(B, Si, save.di), outs[1].view(B, St, save.dt))


class FirstTokenLinearFunction(torch.autograd.Function):
    """y = [tanh](linear(x[:, 0, :]))  (Pooler: modules/losses/flava.py:84-97; cls projections: model.py:244-246,
    261-263).  x fp32 [B, S, d].  Backward: weight / bias gradients by GEMM / column sum, dx scattered into row 0."""

    @staticmethod
    def forward(ctx, x, weight, bias, use_tanh):
        B, S, d = x.shape
        E = weight.shape[0]
        xf = x.contiguous().float()
        CLSb = torch.empty((B, d), device=x.device, dtype=torch.bfloat16)
        ops.gather_rows_cast(xf.view(B * S, d), CLSb, B, S, 0, d)
        wb = ops.cast_bf16(weight.detach().contiguous())
        out = torch.empty((B, E), device=x.device, dtype=torch.float32)
        ops.gemm(CLSb, wb, bias=bias.detach() if bias is not None else None, epilogue=ops.EPI_F32, out=out)
        if use_tanh:
            ops.tanh_(out)
        ctx.save_for_backward(CLSb, wb, out if use_tanh else None)
        ctx.shape, ctx.use_tanh, ctx.has_bias = (B, S, d, E), use_tanh, bias is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        CLSb, wb, y = ctx.saved_tensors
        B, S, d, E = ctx.shape
        dev = dout.device
        dof = dout.contiguous().float()
        if ctx.use_tanh:
            dpre = torch.empty((B, E), device=dev, dtype=torch.bfloat16)
            ops.tanh_bwd(dof, y, None, dpre)
        else:
            dpre = ops.cast_bf16(dof)
        dW = db = dx = None
        if ctx.needs_input_grad[1]:
            dW = torch.empty((E, d), device=dev, dtype=torch.float32)
            ops.gemm(dpre, CLSb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=dW)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = torch.zeros(E, device=dev, dtype=torch.float32)
            ops.colsum_bf16(dpre, db, B, E, E)
        if ctx.needs_input_grad[0]:
            dcls = torch.empty((B, d), device=dev, dtype=torch.float32)
            ops.gemm(dpre, wb, b_mn=True, epilogue=ops.EPI_F32, out=dcls)
            dx = torch.zeros((B, S, d), device=dev, dtype=torch.float32)
            ops.scatter_rows_add(dcls, dx.view(B * S, d), B, S, 0, d)
        return dx, dW, db, None


def first_token_linear(x: torch.Tensor, linear: nn.Linear, use_tanh: bool = False) -> torch.Tensor:
    return FirstTokenLinearFunction.apply(x, linear.weight, linear.bias, use_tanh)


def encoder_output(rt, data, diff, pooler: Optional[nn.Module]) -> TransformerOutput:
    """Training-mode TransformerOutput of one encoder call (pooler applied through FirstTokenLinearFunction).  data:
    the runtime's inputs that are not differentiated; the list that receives hidden_states is appended to them."""
    hidden: List[torch.Tensor] = []
    LAST, XF = run(rt, (*data, hidden), diff)
    B, S, d = hidden[0].shape
    last = LAST.view(B, S, d)
    hidden = list(hidden[:-1]) + [XF.view(B, S, d)]   # hidden_states[-1] is the differentiable output
    pooled = first_token_linear(last, pooler.dense, use_tanh=True) if pooler is not None else None
    return TransformerOutput(last_hidden_state=last, pooler_output=pooled, hidden_states=hidden, attentions=None)
