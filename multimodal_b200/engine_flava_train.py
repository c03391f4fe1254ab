"""Runtime of the FLAVA encoders (BASELINE.json config 3, forward and training step), one per encoder for both grad
modes: forward that keeps what the backward needs + the explicit backward schedule, behind torch.autograd Functions so
that the drop-in modules train with ``loss.backward()`` exactly like the reference's (models/flava/model.py:127-298
under autograd); under torch.no_grad() the same forward keeps nothing and returns the reference's ``TransformerOutput``
(every tensor allocated per call; ``attentions`` on request, recomputed from the packed QKV and the row LSE by one
extra kernel per layer: DESIGN.md §10).

The layer stack is the CLIP towers' ``engine.TransformerStack`` (same kernels, same fused schedule): the separate
query / key / value Linears are presented to it as one packed in-projection (``ParamStore.pack``), the MLP activation
is the exact-erf GELU epilogue pair, and the text tower's key-padding mask goes to the masked attention kernels
(forward and fused single-pass backward).  What is specific to FLAVA is on either side of the stack:

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

from types import SimpleNamespace
from typing import List, Optional, Sequence

import torch
from torch import nn

from . import ops
from ._lib import MMBError
from .engine import (ParamStore, TransformerStack, Workspace, _Shadows, act_code, patch_embed_bwd, patch_embed_fwd,
                     require_head_dim_64, run)
from .modules.layers.transformer import TransformerOutput


class FlavaTrainStack:
    """ParamStore (packed q/k/v order) + TransformerStack + final LayerNorm (+ pooler) of one FLAVA encoder."""

    def __init__(self, owner: nn.Module, encoder: nn.Module, layernorm: nn.Module, pooler: Optional[nn.Module],
                 prefix: str, extra: Sequence[nn.Module] = (), fp32_only: Sequence[nn.Parameter] = ()):
        layers = list(encoder.layer)
        l0 = layers[0]
        if not l0.norm_first:
            raise MMBError("only pre-norm (norm_first=True) FLAVA layers are on the accelerated path")
        d, H = l0.attention.dim_q, l0.attention.n_head
        require_head_dim_64(d, H)
        ff = l0.feedforward.model[0].weight.shape[0]
        params: List[nn.Parameter] = []
        for layer in layers:   # q / k / v weights, then biases, consecutive -> packable
            at = layer.attention
            params += [at.query.weight, at.key.weight, at.value.weight, at.query.bias, at.key.bias, at.value.bias]
        seen = {id(p) for p in params}
        for m in (owner, *extra):
            for p in m.parameters():
                if id(p) not in seen:
                    seen.add(id(p))
                    params.append(p)
        self.store = ParamStore(params, fp32_only)
        self.device = self.store.device
        st = self.store
        adapters = []
        for layer in layers:   # the attribute names TransformerStack reads (torch.nn.TransformerEncoderLayer layout)
            at, mlp = layer.attention, layer.feedforward.model
            attn = SimpleNamespace(in_proj_weight=st.pack([at.query.weight, at.key.weight, at.value.weight]),
                                   in_proj_bias=st.pack([at.query.bias, at.key.bias, at.value.bias], fp32=True),
                                   out_proj=at.output, num_heads=H)
            adapters.append(SimpleNamespace(self_attn=attn, norm1=layer.attention_layernorm,
                                            norm2=layer.feedforward_layernorm, linear1=mlp[0], linear2=mlp[-1]))
        self.ws = Workspace(self.device)   # scratch shared by all calls (stream-ordered)
        self.stack = TransformerStack(adapters, st, self.ws, d=d, heads=H, ff=ff,
                                      act=act_code(l0.feedforward.model[1]), prefix=prefix)
        self.sh = _Shadows(self.device)    # FLAVAModel's projections of the first token (project_first_token)
        self.layernorm, self.pooler, self.prefix = layernorm, pooler, prefix
        self.d, self.H, self.L = d, H, len(layers)

    def forward(self, X0: torch.Tensor, B: int, S: int, kmask: Optional[torch.Tensor], save: Workspace):
        """Returns ((LAST, XF), save): fp32 [B*S, d] each; LAST = layernorm(XF), XF = hidden_states[-1].  The list of
        hidden_states goes to `last_hidden`."""
        LAST, XF, self.last_hidden = self._run(X0, B, S, kmask, save)
        save.XF, save.B, save.S = XF, B, S
        return (LAST, XF), save

    def _run(self, X0, B, S, kmask, save: Optional[Workspace], attns=None):
        d, ln, pfx = self.d, self.layernorm, self.prefix
        M = B * S
        f32 = torch.float32
        stats = save if save is not None else self.ws
        hidden: List[torch.Tensor] = []
        XM, Y = self.stack.forward(X0, B, S, save, kmask=kmask, hidden=hidden, attns=attns)
        XF = torch.empty((M, d), device=self.device, dtype=f32)      # hidden_states[-1] (pre-LayerNorm)
        LAST = torch.empty((M, d), device=self.device, dtype=f32)    # layernorm(XF) == last_hidden_state
        ops.add_layernorm_fwd(XM, Y, XF, None, LAST, ln.weight, ln.bias, stats.get(f"{pfx}.mF", (M,), f32),
                              stats.get(f"{pfx}.rF", (M,), f32), M, d, ln.eps)
        hidden.append(XF.view(B, S, d))
        return LAST, XF, hidden

    def infer(self, X0: torch.Tensor, B: int, S: int, kmask: Optional[torch.Tensor] = None,
              want_attn: bool = False) -> TransformerOutput:
        """want_attn: also return every layer's attention probabilities fp32 [B, H, S, S] (`attentions`), recomputed
        from the packed QKV and the row LSE of the fused attention kernel (mmb_attention_probs)."""
        d, st = self.d, self.store
        attns: Optional[List[torch.Tensor]] = [] if want_attn else None
        LAST, _, hidden = self._run(X0, B, S, kmask, None, attns)
        pooled = None
        if self.pooler is not None:
            CLSb = self.ws.get(f"{self.prefix}.CLSb", (B, d), torch.bfloat16)
            ops.gather_rows_cast(LAST, CLSb, B, S, 0, d)
            pooled = torch.empty((B, d), device=self.device, dtype=torch.float32)
            ops.gemm(CLSb, st.shadow(self.pooler.dense.weight), bias=self.pooler.dense.bias, epilogue=ops.EPI_F32,
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

    def backward(self, save: Workspace, dLAST: Optional[torch.Tensor], dXF: Optional[torch.Tensor]) -> torch.Tensor:
        """Gradient w.r.t. X0 (fp32 [B*S, d], scratch: consume before the next backward of this encoder); parameter
        gradients are accumulated into the store's flat buffer."""
        d, ln, pfx, st = self.d, self.layernorm, self.prefix, self.store
        B, S = save.B, save.S
        M = B * S
        f32, bf = torch.float32, torch.bfloat16
        dLAST, dXF = _f32c(dLAST, (M, d)), _f32c(dXF, (M, d))
        G = self.ws.get(f"{pfx}.G", (M, d), f32)
        Gb = self.ws.get(f"{pfx}.Gb", (M, d), bf)
        if dLAST is None:   # only hidden_states[-1] was used downstream: LayerNorm backward of a zero gradient
            dLAST = torch.zeros((M, d), device=self.device, dtype=f32)
        ops.layernorm_bwd(save.XF, None, dLAST, save.get(f"{pfx}.mF", (M,), f32), save.get(f"{pfx}.rF", (M,), f32),
                          ln.weight, dXF, G, Gb, st.grad(ln.weight), st.grad(ln.bias), M, d,
                          gsum=self.stack.top_bias_grad())
        return self.stack.backward(G, Gb, B, S, top_bias_done=True, save=save)


def _f32c(t: Optional[torch.Tensor], shape) -> Optional[torch.Tensor]:
    if t is None:
        return None
    return t.contiguous().float().view(shape)


# One runtime per encoder: `forward(data, diff)` / `backward` under autograd (engine.run), `infer(...)` under
# torch.no_grad(): the same front end and stack without a save Workspace, then the pooler.
class FlavaImageTrainRuntime:
    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.ts = FlavaTrainStack(mod, mod.encoder, mod.layernorm, mod.pooler, "fimg")
        self.store = self.ts.store

    def _embed(self, pixel_values, image_patches_mask, save: Optional[Workspace]):
        emb, ts, st = self.mod.embeddings, self.ts, self.store
        conv = emb.patch_embeddings.projection
        st.refresh()
        return patch_embed_fwd(pixel_values, conv, st.shadow2d(conv.weight), emb.cls_token, emb.position_embeddings,
                               emb.mask_token, image_patches_mask, ts.ws, save if save is not None else ts.ws, "fimg")

    def forward(self, data, diff):
        pixel_values, image_patches_mask = data
        save = Workspace(self.ts.device)
        X0, B, S, save.P, save.pm = self._embed(pixel_values, image_patches_mask, save)
        return self.ts.forward(X0, B, S, None, save)

    def infer(self, pixel_values: torch.Tensor, image_patches_mask: Optional[torch.Tensor] = None,
              want_attn: bool = False) -> TransformerOutput:
        X0, B, S, _, _ = self._embed(pixel_values, image_patches_mask, None)   # X0 is returned as hidden_states[0]
        return self.ts.infer(X0, B, S, want_attn=want_attn)

    def backward(self, save, dLAST, dXF):
        emb, ts = self.mod.embeddings, self.ts
        G = ts.backward(save, dLAST, dXF)
        patch_embed_bwd(G, emb.patch_embeddings.projection, emb.cls_token, emb.position_embeddings, emb.mask_token,
                        save.pm, save.B, save.S, save.P, self.store, ts.ws, save, "fimg")
        return ()


class FlavaTextTrainRuntime:
    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.ts = FlavaTrainStack(mod, mod.encoder, mod.layernorm, mod.pooler, "ftxt",
                                  fp32_only=list(mod.embeddings.parameters()))
        self.store = self.ts.store

    def _embed(self, input_ids, attention_mask, token_type_ids, save: Optional[Workspace]):
        emb, ts, st = self.mod.embeddings, self.ts, self.store
        d = ts.d
        ids = input_ids.long().contiguous()
        B, S = ids.shape
        if S > emb.position_embeddings.weight.shape[0]:
            raise ValueError(f"sequence length {S} exceeds max_position_embeddings")
        st.refresh()
        X0 = torch.empty((B * S, d), device=ids.device, dtype=torch.float32)   # hidden_states[0]
        KM = (save if save is not None else ts.ws).get("ftxt.KM", (B * S,), torch.uint8)
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
        save = Workspace(self.ts.device)
        X0, B, S, KM, save.ids, save.tt, save.V = self._embed(*data, save)
        return self.ts.forward(X0, B, S, KM, save)

    def infer(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
              token_type_ids: Optional[torch.Tensor] = None, want_attn: bool = False) -> TransformerOutput:
        X0, B, S, KM, _, _, _ = self._embed(input_ids, attention_mask, token_type_ids, None)
        return self.ts.infer(X0, B, S, kmask=KM, want_attn=want_attn)

    def backward(self, save, dLAST, dXF):
        emb, ts, st = self.mod.embeddings, self.ts, self.store
        d, B, S = ts.d, save.B, save.S
        G = ts.backward(save, dLAST, dXF)
        word = emb.word_embeddings
        ops.bert_embed_ln_bwd(save.ids, save.tt, word.weight, emb.position_embeddings.weight,
                              emb.token_type_embeddings.weight, emb.layer_norm.weight, G, st.grad(word.weight),
                              st.grad(emb.position_embeddings.weight), st.grad(emb.token_type_embeddings.weight),
                              st.grad(emb.layer_norm.weight), st.grad(emb.layer_norm.bias), B, S, d, save.V,
                              emb.layer_norm.eps)
        if word.padding_idx is not None:   # nn.Embedding(padding_idx): that row receives no gradient
            ops.zero_(st.grad(word.weight)[word.padding_idx])
        return ()


class FlavaMMTrainRuntime:
    """[cls | image_to_mm(image_hidden) | text_to_mm(text_hidden)] -> stack.  The two projection Linears belong to
    FLAVAModel, not to the multimodal encoder; they live in this runtime's ParamStore (image_proj / text_proj None:
    the module was called directly with an already fused token sequence)."""

    def __init__(self, mod: nn.Module, image_proj: Optional[nn.Linear] = None, text_proj: Optional[nn.Linear] = None):
        self.mod, self.image_proj, self.text_proj = mod, image_proj, text_proj
        extra = [m for m in (image_proj, text_proj) if m is not None]
        self.ts = FlavaTrainStack(mod, mod.encoder, mod.layernorm, mod.pooler, "fmm", extra=extra)
        self.store = self.ts.store

    def _embed(self, diff, save: Optional[Workspace]):
        """-> (X0, B, S, Si, St, di, dt): Si = the fused sequence length and St = 0 for a direct call."""
        ts, st = self.ts, self.store
        d = ts.d
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
        keep = save if save is not None else ts.ws
        Ib = keep.get("fmm.Ib", (B * Si, di), bf)
        Tb = keep.get("fmm.Tb", (B * St, dt), bf)
        ops.cast_bf16(image_hidden.contiguous().float().view(-1), Ib.view(-1))
        ops.cast_bf16(text_hidden.contiguous().float().view(-1), Tb.view(-1))
        Pi = ts.ws.get("fmm.Pi", (B * Si, d), f32)
        Pt = ts.ws.get("fmm.Pt", (B * St, d), f32)
        ops.gemm(Ib, st.shadow(self.image_proj.weight), bias=self.image_proj.bias, epilogue=ops.EPI_F32, out=Pi)
        ops.gemm(Tb, st.shadow(self.text_proj.weight), bias=self.text_proj.bias, epilogue=ops.EPI_F32, out=Pt)
        S = Si + St + off
        X0 = torch.empty((B * S, d), device=image_hidden.device, dtype=f32)   # hidden_states[0]
        ops.concat_tokens(cls, Pi, Pt, X0, B, Si, St, d)
        return X0, B, S, Si, St, di, dt

    def forward(self, data, diff):
        save = Workspace(self.ts.device)
        X0, B, S, save.Si, save.St, save.di, save.dt = self._embed(diff, save)
        return self.ts.forward(X0, B, S, None, save)

    def infer(self, *hidden: torch.Tensor, want_attn: bool = False) -> TransformerOutput:
        """hidden: the fused token sequence fp32 [B, S, d] (direct call), or the image and text encoders' hidden
        states (FLAVAModel.encode_mm, models/flava/model.py:283-298: projected by two GEMMs, then [cls | image | text]
        assembled by one kernel)."""
        X0, B, S, _, _, _, _ = self._embed(hidden, None)
        return self.ts.infer(X0, B, S, want_attn=want_attn)

    def backward(self, save, dLAST, dXF):
        ts, st = self.ts, self.store
        d, B, S, Si, St = ts.d, save.B, save.S, save.Si, save.St
        bf, f32 = torch.bfloat16, torch.float32
        cls = self.mod.cls_token
        has_cls = cls is not None
        G = ts.backward(save, dLAST, dXF)
        if has_cls:
            ops.batch_sum(G, st.grad(cls), B, S * d, d)
        if self.image_proj is None:
            dH = G.view(B, S, d)[:, (1 if has_cls else 0):].clone()   # strided slice copy: plumbing
            return (dH,)
        dPi = ts.ws.get("fmm.dPi", (B * Si, d), bf)
        dPt = ts.ws.get("fmm.dPt", (B * St, d), bf)
        ops.split_tokens_cast(G, dPi, dPt, B, Si, St, d, has_cls)
        outs = []
        for dP, lin, key, n, din in ((dPi, self.image_proj, "fmm.Ib", B * Si, save.di),
                                     (dPt, self.text_proj, "fmm.Tb", B * St, save.dt)):
            Xb = save.get(key, (n, din), bf)
            ops.gemm(dP, Xb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(lin.weight),
                     splits=ops.wgrad_splits(d, din, n), accumulate=True)
            ops.colsum_bf16(dP, st.grad(lin.bias), n, d, d)
            dX = torch.empty((n, din), device=ts.device, dtype=f32)
            ops.gemm(dP, st.shadow(lin.weight), b_mn=True, epilogue=ops.EPI_F32, out=dX)
            outs.append(dX)
        return (outs[0].view(B, Si, save.di), outs[1].view(B, St, save.dt))


def run_encoder(rt, data, diff: Sequence[torch.Tensor] = ()):
    """-> (LAST [M,d], XF [M,d], hidden_states list) with LAST / XF attached to the autograd graph."""
    LAST, XF = run(rt, data, diff)
    hidden, rt.ts.last_hidden = rt.ts.last_hidden, None
    return LAST, XF, hidden


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
    """Training-mode TransformerOutput of one encoder call (pooler applied through FirstTokenLinearFunction)."""
    LAST, XF, hidden = run_encoder(rt, data, diff)
    B, S, d = hidden[0].shape
    last = LAST.view(B, S, d)
    hidden = list(hidden[:-1]) + [XF.view(B, S, d)]   # hidden_states[-1] is the differentiable output
    pooled = first_token_linear(last, pooler.dense, use_tanh=True) if pooler is not None else None
    return TransformerOutput(last_hidden_state=last, pooler_output=pooled, hidden_states=hidden, attentions=None)
