"""Host-side runtime of the dual-encoder path: parameter shadows, activation workspaces and the explicit
forward / backward schedules that drive the sm_90a kernels (multimodal_b200.ops).

Nothing here computes: every tensor op is a C-ABI kernel launch on the current CUDA stream.  The schedules follow
the reference call stack (SURVEY.md §3.1):
  torch/nn/modules/transformer.py:946-951 (pre-norm layer), torch/nn/functional.py:6478-6690 (MHA),
  models/clip/image_encoder.py:82-113, models/clip/text_encoder.py:113-134.
"""
from __future__ import annotations

import math
import os
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

import torch
from torch import nn

from . import ops
from ._lib import MMBError

_ALIGN = 64  # elements; keeps every shadow / grad slice 128 B aligned (TMA needs 16 B)

# bf16 operand shadows are re-cast when a parameter's autograd version counter (or storage) changes.  In-place writes
# through `.data` (`w.data.copy_()`, EMA updates, `module.weight.data.normal_()`) do NOT bump that counter, so every
# shadow key also carries this process-wide epoch: `invalidate_weight_caches()` (exported from the package root, and
# called by the drop-in modules' load_state_dict / _apply hooks) forces a re-cast on the next forward.
_WEIGHT_EPOCH = [0]


def invalidate_weight_caches() -> None:
    _WEIGHT_EPOCH[0] += 1


def weight_epoch() -> int:
    return _WEIGHT_EPOCH[0]


def watch_module(mod: nn.Module) -> None:
    """Invalidate the shadows whenever `mod` (or a parent calling into it) reloads or re-homes its parameters."""
    if getattr(mod, "_mmb_watched", False):
        return
    mod._mmb_watched = True
    mod.register_load_state_dict_post_hook(lambda module, incompatible: invalidate_weight_caches())


def _require_cuda(dev: torch.device) -> None:
    if dev.type != "cuda":
        raise MMBError("multimodal_b200 modules must live on a CUDA device (no CPU path); call .cuda() first")


class ParamStore:
    """Flat bf16 shadow (tensor-core operand copies) + flat fp32 gradient buffer for a list of parameters.
    fp32_only: parameters the kernels only ever read in fp32 (embedding tables); they go last and get no bf16 shadow."""

    def __init__(self, params: Sequence[nn.Parameter], fp32_only: Sequence[nn.Parameter] = ()):
        plain = {id(p) for p in fp32_only}
        self.params: List[nn.Parameter] = ([p for p in params if id(p) not in plain] +
                                           [p for p in params if id(p) in plain])
        if not self.params:
            raise MMBError("ParamStore: no parameters")
        dev = self.params[0].device
        _require_cuda(dev)
        self.device = dev
        self.off: Dict[int, int] = {}
        off, n_shadow = 0, None
        for p in self.params:
            if p.dtype != torch.float32:
                raise MMBError("parameters must be fp32 (bf16 operand copies are made internally)")
            if id(p) in plain and n_shadow is None:
                n_shadow = off
            self.off[id(p)] = off
            off += -(-p.numel() // _ALIGN) * _ALIGN
        self.total = off
        self.wb = torch.empty(off if n_shadow is None else n_shadow, device=dev, dtype=torch.bfloat16)
        self._g: Optional[torch.Tensor] = None
        self._seen: Dict[int, tuple] = {}
        self.master: Optional[torch.Tensor] = None  # set by flatten_()
        self._shadow_fresh = False
        self._epoch = _WEIGHT_EPOCH[0]
        self._shadowed = [p for p in self.params if self.off[id(p)] < self.wb.numel()]
        self._packs: List[list] = []   # [key tensor, parts, version seen]: fp32 concatenations kept current by refresh()
        self._keys: List[torch.Tensor] = []

    @property
    def g(self) -> torch.Tensor:
        """The fp32 gradient buffer, allocated on first use: a store that only serves no_grad forwards never holds it."""
        if self._g is None:
            self._g = torch.zeros(self.total, device=self.device, dtype=torch.float32)
        return self._g

    # -- views ------------------------------------------------------------------------------------------
    def shadow(self, p: nn.Parameter) -> torch.Tensor:
        o = self.off[id(p)]
        return self.wb[o:o + p.numel()].view(p.shape)

    def shadow2d(self, p: nn.Parameter) -> torch.Tensor:
        o = self.off[id(p)]
        return self.wb[o:o + p.numel()].view(p.shape[0], -1)

    def grad(self, p: nn.Parameter) -> torch.Tensor:
        o = self.off[id(p)]
        return self.g[o:o + p.numel()].view(p.shape)

    def grad2d(self, p: nn.Parameter) -> torch.Tensor:
        o = self.off[id(p)]
        return self.g[o:o + p.numel()].view(p.shape[0], -1)

    def pack(self, parts: Sequence[nn.Parameter], fp32: bool = False) -> torch.Tensor:
        """Present consecutive parameters as ONE tensor (rows concatenated): e.g. separate query / key / value Linears
        as the packed [3d, d] in-projection operand.  Returns a key tensor accepted by shadow() / grad() (views spanning
        all parts).  fp32=True: the key is a real fp32 concatenation, kept current by refresh(), usable as a kernel
        operand (biases); otherwise it is a shape-only placeholder."""
        offs = [self.off[id(p)] for p in parts]
        for a, b, p in zip(offs, offs[1:], parts):
            if b != a + p.numel():
                raise MMBError("ParamStore.pack: parts must be consecutive in the store with sizes that are multiples "
                               f"of {_ALIGN} elements")
        shape = (sum(p.shape[0] for p in parts),) + tuple(parts[0].shape[1:])
        if fp32:
            key = torch.empty(shape, device=self.device, dtype=torch.float32)
            self._packs.append([key, list(parts), None])
        else:
            key = torch.empty(shape, device="meta", dtype=torch.float32)
        self.off[id(key)] = offs[0]
        self._keys.append(key)   # keeps id(key) unique for the lifetime of the store
        return key

    def _refresh_packs(self, force: bool) -> None:
        for ent in self._packs:
            key, parts, seen = ent
            ver = tuple((p._version, p.data_ptr()) for p in parts) + (_WEIGHT_EPOCH[0],)
            if force or seen != ver:
                torch.cat([p.data.reshape(-1) for p in parts], out=key.view(-1))   # a few KB of biases: plumbing
                ent[2] = ver

    # -- maintenance ------------------------------------------------------------------------------------
    def flatten_(self) -> None:
        """Re-home every parameter into one flat fp32 master buffer (p.data and p.grad become views).  Enables the
        single-kernel fused optimizer / single NCCL all-reduce of multimodal_b200.train."""
        if self.master is not None:
            return
        self.master = torch.zeros(self.total, device=self.device, dtype=torch.float32)
        with torch.no_grad():
            for p in self.params:
                o = self.off[id(p)]
                self.master[o:o + p.numel()].copy_(p.data.reshape(-1))
                p.data = self.master[o:o + p.numel()].view(p.shape)
                p.grad = self.g[o:o + p.numel()].view(p.shape)
        self._shadow_fresh = False

    def refresh(self) -> None:
        """Make the bf16 shadows current (re-cast whatever changed since the last call)."""
        if self.master is not None:
            if not self._shadow_fresh or self._epoch != _WEIGHT_EPOCH[0]:
                ops.cast_bf16(self.master[:self.wb.numel()], self.wb)
                self._refresh_packs(True)
                self._shadow_fresh = True
                self._epoch = _WEIGHT_EPOCH[0]
            return
        for p in self._shadowed:
            if p.device != self.device:
                raise MMBError("parameter moved to another device after the runtime was created")
            key = (p._version, p.data_ptr(), _WEIGHT_EPOCH[0])
            if self._seen.get(id(p)) != key:
                src = p.data if p.data.is_contiguous() else p.data.contiguous()
                ops.cast_bf16(src.view(-1), self.wb[self.off[id(p)]:self.off[id(p)] + p.numel()])
                self._seen[id(p)] = key
        self._refresh_packs(False)

    def mark_dirty(self) -> None:
        self._shadow_fresh = False

    def zero_grads(self) -> None:
        ops.zero_(self.g)


class Workspace:
    """Named, lazily allocated, reused device buffers."""

    def __init__(self, device):
        self.device = device
        self.bufs: Dict[str, torch.Tensor] = {}
        self.X0: Optional[torch.Tensor] = None      # set by TransformerStack.forward when saving: layer-0 input
        self.kmask: Optional[torch.Tensor] = None   # ... and the key-padding mask / [B,S,S] mask / cross-attention
        self.mask3: Optional[torch.Tensor] = None   #     source that forward used
        self.enc: Optional[torch.Tensor] = None
        self.S_enc = 0
        self.dENC: Optional[torch.Tensor] = None    # set by backward: gradient w.r.t. the cross-attention source

    def get(self, name: str, shape, dtype) -> torch.Tensor:
        t = self.bufs.get(name)
        shape = tuple(int(s) for s in shape)
        if t is None or t.dtype != dtype or t.numel() < _numel(shape):
            t = torch.empty(_numel(shape), device=self.device, dtype=dtype)
            self.bufs[name] = t
        return t[:_numel(shape)].view(shape)

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.bufs.values())


def _numel(shape) -> int:
    n = 1
    for s in shape:
        n *= int(s)
    return n


class _Shadows:
    """bf16 operand copies of fp32 weights outside a ParamStore, re-cast when a parameter's version changes."""

    def __init__(self, device):
        self.device = device
        self.bufs: Dict[str, torch.Tensor] = {}
        self.seen: Dict[str, tuple] = {}

    def get(self, key: str, parts: Sequence[torch.Tensor]) -> torch.Tensor:
        """bf16 copy of cat(parts, dim=0) (each part [n_i, k])."""
        ver = (weight_epoch(),) + tuple((p._version, p.data_ptr()) for p in parts)
        buf = self.bufs.get(key)
        if buf is None:
            rows = sum(p.shape[0] for p in parts)
            buf = torch.empty((rows,) + tuple(parts[0].shape[1:]), device=self.device, dtype=torch.bfloat16)
            self.bufs[key] = buf
        if self.seen.get(key) != ver:
            r = 0
            for p in parts:
                src = p.data if p.data.is_contiguous() else p.data.contiguous()
                ops.cast_bf16(src.view(-1), buf[r:r + p.shape[0]].view(-1))
                r += p.shape[0]
            self.seen[key] = ver
        return buf

    def cat_f32(self, key: str, parts: Sequence[torch.Tensor]) -> torch.Tensor:
        ver = (weight_epoch(),) + tuple((p._version, p.data_ptr()) for p in parts)
        buf = self.bufs.get(key)
        if buf is None:
            buf = torch.empty(sum(p.numel() for p in parts), device=self.device, dtype=torch.float32)
            self.bufs[key] = buf
        if self.seen.get(key) != ver:
            r = 0
            for p in parts:
                buf[r:r + p.numel()].copy_(p.data.reshape(-1))   # 3 x d floats: plumbing
                r += p.numel()
            self.seen[key] = ver
        return buf


def act_code(act: nn.Module) -> int:
    """Kernel epilogue code of an MLP activation module."""
    from .modules.layers.activation import SiLU

    if isinstance(act, nn.GELU) and getattr(act, "approximate", "none") == "none":
        return ops.ACT_GELU_ERF
    if isinstance(act, SiLU):
        return ops.ACT_QUICK_GELU
    if isinstance(act, nn.ReLU):
        return ops.ACT_RELU
    raise MMBError(f"unsupported MLP activation {type(act).__name__} on the accelerated path (nn.GELU / SiLU / nn.ReLU)")


def scaled(scale: Optional[torch.Tensor], rows_per_scale: int) -> dict:
    """Keyword arguments that pass a stochastic-depth factor (fp32 [M / rows_per_scale] or None) to
    ops.add_layernorm_fwd / layernorm_bwd / cast_bf16: none without a factor, so an unscaled call is the call a stack
    without drop path makes."""
    return {} if scale is None else {"branch_scale": scale, "rows_per_scale": rows_per_scale}


def wants_grad(*mods: Optional[nn.Module]) -> bool:
    """True when the caller expects an autograd graph: grad mode on and some parameter of `mods` trainable."""
    if not torch.is_grad_enabled():
        return False
    return any(p.requires_grad for m in mods if m is not None for p in m.parameters())


def patch_embed_fwd(image: torch.Tensor, conv: nn.Module, wconv: torch.Tensor, cls: Optional[torch.Tensor],
                    pos: torch.Tensor, mask_token: Optional[torch.Tensor], image_patches_mask: Optional[torch.Tensor],
                    ws: Workspace, save: Workspace, prefix: str, keep: Optional[torch.Tensor] = None):
    """Patch front end of a ViT (patch_embedding.py:104-154, image_encoder.py:139-175): im2col + conv GEMM (+ bias), then
    [cls |] patch or mask token, + position embeddings, in one assembly kernel.  wconv: bf16 [d, 3*ps*ps] conv weight.
    keep (int32 [B, L], random patch dropping): only the kept patches are embedded, token off+j being patch keep[b, j].
    The im2col matrix goes to `save` (the conv weight gradient reads it), the rest of the scratch to `ws`.
    Returns (X0 fp32 [B*S, d], allocated per call; B, S = off + L (L = P without keep), P; the uint8 [B, P] patch mask
    or None)."""
    d, ps = conv.weight.shape[0], conv.weight.shape[2]
    image = image.contiguous().float()
    B, _, Hh, Ww = image.shape
    P = (Hh // ps) * (Ww // ps)
    L = P if keep is None else keep.shape[1]
    S = L + (1 if cls is not None else 0)
    K = 3 * ps * ps
    Kp = -(-K // 8) * 8   # row pitch: bf16 rows must be 16 B multiples for TMA (K = 588 -> 592 for 14x14 patches)
    bf = torch.bfloat16
    PATCH = save.get(f"{prefix}.PATCH", (B * L, Kp), bf)[:, :K]
    PO = ws.get(f"{prefix}.PO", (B * L, d), bf)
    X0 = torch.empty((B * S, d), device=image.device, dtype=torch.float32)
    if keep is None:
        ops.im2col(image, ps, PATCH)
    else:
        ops._im2col_gather(image, keep, ps, PATCH)
    if Kp != K:   # re-pitch the (tiny) conv weight shadow the same way
        wp = ws.get(f"{prefix}.WCONV", (d, Kp), bf)[:, :K]
        wp.copy_(wconv)
        wconv = wp
    ops.gemm(PATCH, wconv, bias=conv.bias, out=PO)
    pm = None
    if image_patches_mask is not None and mask_token is not None:
        pm = image_patches_mask.reshape(B, P).to(torch.uint8).contiguous()
    mt = mask_token if pm is not None else None
    if keep is None:
        ops.vit_assemble_fwd(PO, cls, pos, mt, pm, X0, B, S, d)
    else:
        ops._vit_assemble_gather_fwd(PO, cls, pos, mt, pm, keep, X0, P, d)
    return X0, B, S, P, pm


def patch_embed_bwd(G: torch.Tensor, conv: nn.Module, cls: Optional[torch.Tensor], pos: torch.Tensor,
                    mask_token: Optional[torch.Tensor], pm: Optional[torch.Tensor], B: int, S: int, P: int,
                    st: "ParamStore", ws: Workspace, save: Workspace, prefix: str,
                    keep: Optional[torch.Tensor] = None) -> None:
    """Parameter gradients of patch_embed_fwd from G = d X0 (fp32 [B*S, d]); keep as given to the forward."""
    d, ps = conv.weight.shape[0], conv.weight.shape[2]
    K = 3 * ps * ps
    rows = B * (P if keep is None else keep.shape[1])
    DP = ws.get(f"{prefix}.DP", (rows, d), torch.bfloat16)
    dmask = st.grad(mask_token) if pm is not None else None
    if keep is None:
        ops.batch_sum(G, st.grad(pos), B, S * d, S * d)
        if cls is not None:
            ops.batch_sum(G, st.grad(cls), B, S * d, d)
        ops.vit_assemble_bwd(G, pm, DP, dmask, B, S, d, cls is not None)
    else:
        ops._vit_assemble_gather_bwd(G, pm, keep, DP, dmask, st.grad(cls) if cls is not None else None, st.grad(pos),
                                    P, d, cls is not None)
    PATCH = save.get(f"{prefix}.PATCH", (rows, -(-K // 8) * 8), torch.bfloat16)[:, :K]
    ops.gemm(DP, PATCH, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad2d(conv.weight),
             splits=ops.wgrad_splits(d, K, rows), accumulate=True)
    if conv.bias is not None:
        ops.colsum_bf16(DP, st.grad(conv.bias), rows, d, d)


def require_head_dim_64(d: int, heads: int) -> None:
    if d % heads or d // heads != 64:
        raise MMBError(f"attention kernels support head_dim 64 only (got d={d}, heads={heads})")


class TransformerStack:
    """L pre-norm encoder / decoder layers (torch.nn.TransformerEncoderLayer parameter layout), QuickGELU or GELU MLP,
    head_dim 64 / 96 / 128 (a forward that saves for the backward: 64)."""

    # without a save Workspace, a buffer that is dead before its namesake is written shares that namesake's storage
    _SHARED = {"LN2": "LN1", "LNC": "LN1", "OC": "O"}

    def __init__(self, layers: Sequence[nn.Module], store: ParamStore, ws: Workspace, *, d: int, heads: int, ff: int,
                 act: int, prefix: str):
        self.layers = list(layers)
        self.store, self.ws = store, ws
        self.d, self.H, self.ff, self.act, self.prefix = d, heads, ff, act, prefix
        self.hd = d // heads
        if d % heads or self.hd not in (64, 96, 128):
            raise MMBError(f"unsupported head_dim {self.hd}")
        self.scale = 1.0 / math.sqrt(self.hd)
        self.L = len(self.layers)

    def _bufs(self, save):
        """buf(name, layer, shape, dtype): per-layer buffers in `save`, or without one the workspace's buffer of that
        name, looked up once per forward (every layer has the same shapes)."""
        if save is not None:
            return lambda name, l, shape, dt: save.get(f"{self.prefix}.{name}.{l}", shape, dt)
        got: Dict[str, torch.Tensor] = {}

        def buf(name, l, shape, dt):
            if name not in got:
                got[name] = self.ws.get(f"{self.prefix}.{self._SHARED.get(name, name)}.0", shape, dt)
            return got[name]
        return buf

    def forward(self, X0: torch.Tensor, B: int, S: int, save: Optional["Workspace"], *, causal: bool = False,
                kmask: Optional[torch.Tensor] = None, mask3: Optional[torch.Tensor] = None,
                enc: Optional[torch.Tensor] = None, S_enc: int = 0, scales=None,
                hidden: Optional[List[torch.Tensor]] = None, attns: Optional[List[torch.Tensor]] = None):
        """X0: fp32 [B*S, d] residual stream entering layer 0.  Returns (XM_last fp32, Y bf16): the final residual
        stream is XM_last + Y (the add is fused into whichever LayerNorm consumes it; with stochastic depth the caller
        scales that add by the last layer's feed-forward factor).
        save: the Workspace that receives the activations (and the arguments below) the backward reads, or None: a
        forward that keeps nothing runs in the stack's own workspace, one buffer per name for all layers.
        scales: stochastic depth (modules/layers/stochastic_depth.drop_path_scales): per layer the (attention,
        feed-forward) per-sample factors fp32 [B] or None; each scales its branch inside the residual add that
        follows it, and the backward scales the gradient entering the branch.  Not with cross-attention layers.
        kmask: optional uint8 [B*S] key-padding mask (1 = attend).  mask3: optional uint8 [B, S, S] mask (general
        attention kernels).  enc / S_enc: bf16 [B*S_enc, d_kv] cross-attention source for layers that carry a
        `cross_attn` block (TransformerDecoderLayer: modules/layers/transformer.py:354-377).
        hidden: list that receives each layer's input stream [B, S, d], X0 first (without `save`, allocated per call:
        they are returned to the user).  attns: list that receives each layer's attention probabilities fp32
        [B, H, S, S] (ops.attention_probs, recomputed from the packed QKV and the row LSE)."""
        if scales is not None and enc is not None:
            raise MMBError("stochastic depth is applied to encoder layers only (no cross-attention)")
        if save is None:
            self.ws.X0 = None   # this forward overwrites what a saving forward into the stack's own workspace kept
        else:
            if self.hd != 64:
                raise MMBError(f"training needs head_dim 64 in the layer stacks (got {self.hd}); the poolers may differ")
            save.X0, save.causal, save.kmask, save.mask3, save.enc, save.S_enc = X0, causal, kmask, mask3, enc, S_enc
            save.scales, save.rows_per_scale = scales, S
        st, d, ff, H = self.store, self.d, self.ff, self.H
        M = B * S
        bf, f32 = torch.bfloat16, torch.float32
        buf = self._bufs(save)
        Y = self.ws.get(f"{self.prefix}.Y", (M, d), bf)
        if hidden is not None:
            hidden.append(X0.view(B, S, d))
        XA, XM_prev = X0, None
        for l, layer in enumerate(self.layers):
            at = layer.self_attn
            s_attn = scales[l][0] if scales is not None else None
            s_prev_ff = scales[l - 1][1] if scales is not None and l > 0 else None
            LN1 = buf("LN1", l, (M, d), bf)
            QKV = buf("QKV", l, (M, 3 * d), bf)
            O = buf("O", l, (M, d), bf)
            LSE = buf("LSE", l, (B * H * S,), f32)
            XM = buf("XM", l, (M, d), f32)
            LN2 = buf("LN2", l, (M, d), bf)
            PRE = buf("PRE", l, (M, ff), bf)
            HACT = buf("HACT", l, (M, ff), bf)
            m1 = buf("m1", l, (M,), f32); r1 = buf("r1", l, (M,), f32)
            m2 = buf("m2", l, (M,), f32); r2 = buf("r2", l, (M,), f32)
            if l == 0:
                XA = X0
                ops.add_layernorm_fwd(XA, None, None, LN1, None, layer.norm1.weight, layer.norm1.bias, m1, r1, M, d,
                                      layer.norm1.eps)
            else:
                XA = (torch.empty((M, d), device=X0.device, dtype=f32) if save is None and hidden is not None
                      else buf("XA", l, (M, d), f32))
                ops.add_layernorm_fwd(XM_prev, Y, XA, LN1, None, layer.norm1.weight, layer.norm1.bias, m1, r1, M, d,
                                      layer.norm1.eps, **scaled(s_prev_ff, S))
                if hidden is not None:
                    hidden.append(XA.view(B, S, d))
            ops.gemm(LN1, st.shadow(at.in_proj_weight), bias=at.in_proj_bias, out=QKV)
            ops.self_attention(QKV, O, LSE, B, S, H, self.hd, causal, self.scale, kmask=kmask, mask=mask3)
            if attns is not None:
                P = torch.empty((B, H, S, S), device=X0.device, dtype=f32)
                ops.attention_probs(QKV, LSE, kmask, P, B, S, H, causal, self.scale)
                attns.append(P)
            ops.gemm(O, st.shadow(at.out_proj.weight), bias=at.out_proj.bias, out=Y)
            ca = getattr(layer, "cross_attn", None)
            if ca is not None and enc is not None:
                # x1 = x + self-attention (XM);  x2 = x1 + cross-attention(LN_c(x1), enc) (XC);  the MLP reads LN2(x2)
                lnc = layer.norm_cross
                Se = S_enc
                LNC = buf("LNC", l, (M, d), bf)
                QC = buf("QC", l, (M, d), bf)
                KVC = buf("KVC", l, (B * Se, 2 * d), bf)
                OC = buf("OC", l, (M, d), bf)
                XC = buf("XC", l, (M, d), f32)
                mc = buf("mc", l, (M,), f32); rc = buf("rc", l, (M,), f32)
                ops.add_layernorm_fwd(XA, Y, XM, LNC, None, lnc.weight, lnc.bias, mc, rc, M, d, lnc.eps)
                ops.gemm(LNC, st.shadow(ca.q_w), bias=ca.q_b, out=QC)
                ops.gemm(enc, st.shadow(ca.kv_w), bias=ca.kv_b, out=KVC)
                ops.attention_fwd_generic(QC, KVC[:, :d], KVC[:, d:], OC, B=B, Sq=S, Skv=Se, H=H, head_dim=self.hd,
                                          bsq=S * d, bsk=Se * 2 * d, bsv=Se * 2 * d, bso=S * d, scale=self.scale)
                ops.gemm(OC, st.shadow(ca.out_proj.weight), bias=ca.out_proj.bias, out=Y)
                ops.add_layernorm_fwd(XM, Y, XC, LN2, None, layer.norm2.weight, layer.norm2.bias, m2, r2, M, d,
                                      layer.norm2.eps)
                XM = XC
            else:
                ops.add_layernorm_fwd(XA, Y, XM, LN2, None, layer.norm2.weight, layer.norm2.bias, m2, r2, M, d,
                                      layer.norm2.eps, **scaled(s_attn, S))
            ops.gemm(LN2, st.shadow(layer.linear1.weight), bias=layer.linear1.bias, epilogue=ops.EPI_BF16_ACT, out=PRE,
                     out2=HACT, act=self.act)
            ops.gemm(HACT, st.shadow(layer.linear2.weight), bias=layer.linear2.bias, out=Y)
            XM_prev = XM
        return XM_prev, Y

    @staticmethod
    def top_scale(save: "Workspace"):
        """(factor or None, rows_per_scale) of the last layer's MLP branch: scales the add of XM_last + Y, and the
        gradient entering that branch at the start of the backward."""
        scales = getattr(save, "scales", None)
        return (scales[-1][1] if scales is not None else None), getattr(save, "rows_per_scale", 0)

    def top_bias_grad(self) -> torch.Tensor:
        """Gradient slot of the last layer's linear2.bias: the producer of the incoming Gb sums its columns into it."""
        return self.store.grad(self.layers[-1].linear2.bias)

    def backward(self, G: torch.Tensor, Gb: torch.Tensor, B: int, S: int, *, save: "Workspace", on_layer_done=None,
                 top_bias_done: bool = False) -> torch.Tensor:
        """G (fp32) / Gb (bf16 copy, times the last MLP branch's stochastic-depth factor when the forward had
        scales): gradient w.r.t. the final residual stream [B*S, d]; save: the Workspace the forward saved into.
        Returns G w.r.t. X0 (in place).  Parameter gradients are ACCUMULATED into the ParamStore's flat fp32 buffer.
        The bias gradients of linear2 / out_proj are column sums of Gb; they are produced by the LayerNorm-backward
        kernel that writes Gb (`gsum`), not by a separate pass (top_bias_done: the caller's kernel did the top one)."""
        X0, kmask, causal = save.X0, getattr(save, "kmask", None), getattr(save, "causal", False)
        mask3, enc, Se = getattr(save, "mask3", None), getattr(save, "enc", None), getattr(save, "S_enc", 0)
        scales = getattr(save, "scales", None)
        save.dENC = None
        if X0 is None:
            raise MMBError("backward called without a saved training forward")
        st, d, ff, H = self.store, self.d, self.ff, self.H
        M = B * S
        bf = torch.bfloat16
        T1 = self.ws.get(f"{self.prefix}.T1", (M, d), bf)
        T3 = self.ws.get(f"{self.prefix}.T3", (M, 3 * d), bf)
        sp = ops.wgrad_splits
        for l in range(self.L - 1, -1, -1):
            layer = self.layers[l]
            at = layer.self_attn
            f32 = torch.float32
            g = lambda n, shape, dt: save.get(f"{self.prefix}.{n}.{l}", shape, dt)  # noqa: E731
            LN1, QKV, O = g("LN1", (M, d), bf), g("QKV", (M, 3 * d), bf), g("O", (M, d), bf)
            LSE = g("LSE", (B * H * S,), f32)
            XM, LN2 = g("XM", (M, d), f32), g("LN2", (M, d), bf)
            ca = getattr(layer, "cross_attn", None) if enc is not None else None
            XMID = g("XC", (M, d), f32) if ca is not None else XM     # the stream the MLP branch was added to
            PRE, HACT = g("PRE", (M, ff), bf), g("HACT", (M, ff), bf)
            m1, r1, m2, r2 = g("m1", (M,), f32), g("r1", (M,), f32), g("m2", (M,), f32), g("r2", (M,), f32)
            XA = X0 if l == 0 else g("XA", (M, d), f32)
            # ---- MLP branch:  y = W2 act(W1 LN2(x) + b1) + b2 ----
            ops.gemm(Gb, HACT, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(layer.linear2.weight),
                     splits=sp(d, ff, M), accumulate=True)
            if l == self.L - 1 and not top_bias_done:
                ops.colsum_bf16(Gb, st.grad(layer.linear2.bias), M, d, d)
            dPRE = HACT  # overwrite: act output is dead once its wgrad has been issued (same stream)
            fuse = os.environ.get("MMB_FUSE_COLSUM_GEMM", "1") == "1"
            ops.gemm(Gb, st.shadow(layer.linear2.weight), b_mn=True, epilogue=ops.EPI_BF16_DACT, aux=PRE, out=dPRE,
                     act=self.act, colsum=st.grad(layer.linear1.bias) if fuse else None)   # db1 = colsum(dPRE), fused into the epilogue
            ops.gemm(dPRE, LN2, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(layer.linear1.weight),
                     splits=sp(ff, d, M), accumulate=True)
            if not fuse:
                ops.colsum_bf16(dPRE, st.grad(layer.linear1.bias), M, ff, ff)
            ops.gemm(dPRE, st.shadow(layer.linear1.weight), b_mn=True, out=T1)
            ops.layernorm_bwd(XMID, T1, None, m2, r2, layer.norm2.weight, G, G, Gb, st.grad(layer.norm2.weight),
                              st.grad(layer.norm2.bias), M, d,
                              gsum=st.grad(ca.out_proj.bias if ca is not None else at.out_proj.bias),
                              **scaled(scales[l][0] if scales is not None else None, S))
            if ca is not None:
                # ---- cross-attention branch:  x2 = x1 + Wo_c Attn(Wq LN_c(x1), Wkv enc) ----
                lnc = layer.norm_cross
                dkv = enc.shape[1]
                LNC, QC, OC = g("LNC", (M, d), bf), g("QC", (M, d), bf), g("OC", (M, d), bf)
                KVC = g("KVC", (B * Se, 2 * d), bf)
                mc, rc = g("mc", (M,), f32), g("rc", (M,), f32)
                ops.gemm(Gb, OC, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(ca.out_proj.weight),
                         splits=sp(d, d, M), accumulate=True)
                ops.gemm(Gb, st.shadow(ca.out_proj.weight), b_mn=True, out=T1)      # d OC
                dQC = self.ws.get(f"{self.prefix}.dQC", (M, d), bf)
                dKVC = self.ws.get(f"{self.prefix}.dKVC", (B * Se, 2 * d), bf)
                ops.attention_bwd_generic(QC, KVC[:, :d], KVC[:, d:], T1, dKVC[:, :d], dKVC[:, d:], dq=dQC, B=B, Sq=S,
                                          Skv=Se, H=H, head_dim=self.hd, bsq=S * d, bsk=Se * 2 * d, bsv=Se * 2 * d, bso=S * d,
                                          scale=self.scale)
                ops.gemm(dQC, LNC, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(ca.q_w), splits=sp(d, d, M),
                         accumulate=True)
                ops.colsum_bf16(dQC, st.grad(ca.q_b), M, d, d)
                ops.gemm(dKVC, enc, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(ca.kv_w),
                         splits=sp(2 * d, dkv, B * Se), accumulate=True)
                ops.colsum_bf16(dKVC, st.grad(ca.kv_b), B * Se, 2 * d, 2 * d)
                if save.dENC is None:   # gradient w.r.t. the cross-attention source, summed over the layers
                    save.dENC = torch.empty((B * Se, dkv), device=G.device, dtype=f32)
                    ops.gemm(dKVC, st.shadow(ca.kv_w), b_mn=True, epilogue=ops.EPI_F32, out=save.dENC)
                else:
                    ops.gemm(dKVC, st.shadow(ca.kv_w), b_mn=True, epilogue=ops.EPI_F32, out=save.dENC, accumulate=True)
                ops.gemm(dQC, st.shadow(ca.q_w), b_mn=True, out=T1)                  # d LN_c(x1)
                ops.layernorm_bwd(XM, T1, None, mc, rc, lnc.weight, G, G, Gb, st.grad(lnc.weight), st.grad(lnc.bias), M, d,
                                  gsum=st.grad(at.out_proj.bias))
            # ---- attention branch ----
            ops.gemm(Gb, O, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(at.out_proj.weight),
                     splits=sp(d, d, M), accumulate=True)
            ops.gemm(Gb, st.shadow(at.out_proj.weight), b_mn=True, out=T1)  # dO
            ops.self_attention(QKV, O, LSE, B, S, H, self.hd, causal, self.scale, kmask=kmask, mask=mask3, dout=T1,
                               dqkv=T3)
            ops.gemm(T3, LN1, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(at.in_proj_weight),
                     splits=sp(3 * d, d, M), accumulate=True)
            ops.colsum_bf16(T3, st.grad(at.in_proj_bias), M, 3 * d, 3 * d)
            ops.gemm(T3, st.shadow(at.in_proj_weight), b_mn=True, out=T1)
            ops.layernorm_bwd(XA, T1, None, m1, r1, layer.norm1.weight, G, G, Gb, st.grad(layer.norm1.weight),
                              st.grad(layer.norm1.bias), M, d,
                              gsum=st.grad(self.layers[l - 1].linear2.bias) if l > 0 else None,
                              **scaled(scales[l - 1][1] if scales is not None and l > 0 else None, S))
            if on_layer_done is not None:
                on_layer_done(l)  # all parameter gradients of layer l are final (data-parallel all-reduce hook)
        return G


def _attention_parts(at: nn.Module):
    """(separate q / k / v Linears or None when already packed, output Linear, head count) of a TorchMultimodal
    attention module: packed `input_proj` (MultiHeadSelfAttention), `q_proj` / `k_proj` / `v_proj`
    (MultiHeadAttentionWithCache) or FLAVA's `query` / `key` / `value` / `output` (MultiHeadAttention)."""
    if hasattr(at, "input_proj"):
        return None, at.output_proj, at.num_heads
    if hasattr(at, "q_proj"):
        return (at.q_proj, at.k_proj, at.v_proj), at.output_proj, at.num_heads
    return (at.query, at.key, at.value), at.output, at.n_head


def as_f32(t: Optional[torch.Tensor], shape) -> Optional[torch.Tensor]:
    return None if t is None else t.contiguous().float().view(shape)


class ModuleStack:
    """ParamStore + TransformerStack over a list of TorchMultimodal pre-norm encoder / decoder layers
    (modules/layers/transformer.py, models/flava/transformer.py), plus the final residual add and the gradient entering
    the stack's backward.  The store holds every parameter of `owner` and `extra` (modules outside the owner whose
    parameters its runtime uses); the separate q / k / v (and cross-attention k / v) projections go first, weights then
    biases, so that they can be packed into one operand."""

    def __init__(self, owner: nn.Module, layers, prefix: str, extra: Sequence[nn.Module] = (),
                 fp32_only: Sequence[nn.Parameter] = ()):
        layers = list(layers)
        l0 = layers[0]
        if not l0.norm_first:
            raise MMBError("only pre-norm (norm_first=True) layers are on the accelerated path")
        params: List[nn.Parameter] = []
        for layer in layers:
            qkv = _attention_parts(layer.attention)[0]
            if qkv is not None:
                params += [p.weight for p in qkv] + [p.bias for p in qkv]
            ca = getattr(layer, "cross_attention", None)
            if ca is not None:
                params += [ca.k_proj.weight, ca.v_proj.weight, ca.k_proj.bias, ca.v_proj.bias]
        seen = {id(p) for p in params}
        for m in (owner, *extra):
            for p in m.parameters():
                if id(p) not in seen:
                    seen.add(id(p))
                    params.append(p)
        self.store = st = ParamStore(params, fp32_only)
        self.device = st.device
        self.d = l0.attention_layernorm.normalized_shape[0]
        self.ws = Workspace(self.device)   # scratch shared by all calls (stream-ordered)
        adapters = []
        for layer in layers:   # the attribute names TransformerStack reads (torch.nn.TransformerEncoderLayer layout)
            mlp = layer.feedforward.model
            qkv, out_proj, heads = _attention_parts(layer.attention)
            if qkv is None:
                w, b = layer.attention.input_proj.weight, layer.attention.input_proj.bias
            else:
                w, b = st.pack([p.weight for p in qkv]), st.pack([p.bias for p in qkv], fp32=True)
            attn = SimpleNamespace(in_proj_weight=w, in_proj_bias=b, out_proj=out_proj, num_heads=heads)
            ad = SimpleNamespace(self_attn=attn, norm1=layer.attention_layernorm, norm2=layer.feedforward_layernorm,
                                 linear1=mlp[0], linear2=mlp[-1])
            ca = getattr(layer, "cross_attention", None)
            if ca is not None:
                ad.cross_attn = SimpleNamespace(q_w=ca.q_proj.weight, q_b=ca.q_proj.bias,
                                                kv_w=st.pack([ca.k_proj.weight, ca.v_proj.weight]),
                                                kv_b=st.pack([ca.k_proj.bias, ca.v_proj.bias], fp32=True),
                                                out_proj=ca.output_proj)
                ad.norm_cross = layer.cross_attention_layernorm
            adapters.append(ad)
        self.stack = TransformerStack(adapters, st, self.ws, d=self.d, heads=_attention_parts(l0.attention)[2],
                                      ff=l0.feedforward.model[0].weight.shape[0], act=act_code(l0.feedforward.model[1]),
                                      prefix=prefix)
        self.prefix = prefix
        self.layers = layers     # the modules themselves: their StochasticDepth (drop_path_rate), if any

    def finish(self, XM, Y, B: int, S: int, ln: Optional[nn.Module], save: Optional[Workspace], scales,
               LASTb: Optional[torch.Tensor] = None):
        """XF = XM + Y (the residual stream after the last layer; Y times the last MLP branch's stochastic-depth
        factor when `scales` has one); LAST = ln(XF) when a final LayerNorm exists, and its bf16 copy into LASTb if
        given.  XF / LAST are returned to the caller: allocated per call."""
        d, pfx, M = self.d, self.prefix, B * S
        f32 = torch.float32
        stats = save if save is not None else self.ws
        XF = torch.empty((M, d), device=self.device, dtype=f32)
        LAST = torch.empty((M, d), device=self.device, dtype=f32) if ln is not None else None
        aff = ln if ln is not None else self.stack.layers[0].norm1   # affine terms unused when nothing is normalised
        ops.add_layernorm_fwd(XM, Y, XF, LASTb, LAST, aff.weight, aff.bias,
                              stats.get(f"{pfx}.mF", (M,), f32) if ln is not None else None,
                              stats.get(f"{pfx}.rF", (M,), f32) if ln is not None else None, M, d, aff.eps,
                              **scaled(scales[-1][1] if scales is not None else None, S))
        if save is not None:
            save.XF = XF
        return XF, LAST

    def start_backward(self, save: Workspace, M: int, ln: Optional[nn.Module], dLAST, dXF):
        """(G fp32, Gb bf16, top_bias_done): gradient w.r.t. XF entering the stack's backward; Gb is the gradient
        entering the last MLP branch (scaled by its stochastic-depth factor, if any).  With a final LayerNorm and a
        gradient of LAST or XF, the LayerNorm backward adds both (a missing dLAST counts as zero)."""
        d, pfx, st = self.d, self.prefix, self.store
        f32, bf = torch.float32, torch.bfloat16
        G = self.ws.get(f"{pfx}.G", (M, d), f32)
        Gb = self.ws.get(f"{pfx}.Gb", (M, d), bf)
        scale, rows = self.stack.top_scale(save)
        if ln is not None and (dLAST is not None or dXF is not None):
            if dLAST is None:   # only XF was used downstream
                dLAST = torch.zeros((M, d), device=self.device, dtype=f32)
            ops.layernorm_bwd(save.XF, None, dLAST, save.get(f"{pfx}.mF", (M,), f32), save.get(f"{pfx}.rF", (M,), f32),
                              ln.weight, dXF, G, Gb, st.grad(ln.weight), st.grad(ln.bias), M, d,
                              gsum=self.stack.top_bias_grad(), **scaled(scale, rows))
            return G, Gb, True
        if dXF is None:
            ops.zero_(G)
        else:
            G.copy_(dXF.view(M, d))      # the stack's backward works in place on G
        ops.cast_bf16(G, Gb, **scaled(scale, rows))
        return G, Gb, False


class ViTTower:
    """CLIPViTEncoder runtime (models/clip/image_encoder.py:82-113).  Output: the embeddings fp32 [B, E]."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.store = ParamStore(list(mod.parameters()))
        self.ws = Workspace(self.store.device)
        d = mod.conv.weight.shape[0]
        layer0 = mod.encoder.layers[0]
        self.d, self.ps = d, mod.conv.weight.shape[2]
        self.E = mod.projection.shape[1]
        require_head_dim_64(d, layer0.self_attn.num_heads)
        self.stack = TransformerStack(mod.encoder.layers, self.store, self.ws, d=d, heads=layer0.self_attn.num_heads,
                                      ff=layer0.linear1.weight.shape[0], act=ops.ACT_QUICK_GELU, prefix="img")

    def _forward(self, image: torch.Tensor, save: Optional[Workspace], out: Optional[torch.Tensor] = None):
        """out (optional): fp32 [B, E] destination of the embeddings (e.g. a row block of a larger buffer)."""
        mod, st, ws, d = self.mod, self.store, self.ws, self.d
        keep = save if save is not None else ws
        if image.dtype != torch.float32:
            image = image.float()
        image = image.contiguous()
        B, _, Himg, Wimg = image.shape
        ps = self.ps
        P = (Himg // ps) * (Wimg // ps)
        S = P + 1
        K = 3 * ps * ps
        bf, f32 = torch.bfloat16, torch.float32
        st.refresh()
        Kp = -(-K // 8) * 8   # row pitch: bf16 rows must be 16 B multiples for TMA (K = 588 -> 592 for 14x14 patches)
        PATCH = keep.get("img.PATCH", (B * P, Kp), bf)[:, :K]
        PO = keep.get("img.PO", (B * P, d), bf)
        X0 = keep.get("img.X0", (B * S, d), f32)
        m0 = keep.get("img.m0", (B * S,), f32); r0 = keep.get("img.r0", (B * S,), f32)
        ops.im2col(image, ps, PATCH)
        wconv = st.shadow2d(mod.conv.weight)
        if Kp != K:  # re-pitch the (tiny) conv weight shadow the same way
            wpad = ws.get("img.WCONV", (d, Kp), bf)[:, :K]
            wpad.copy_(wconv)
            wconv = wpad
        ops.gemm(PATCH, wconv, out=PO)
        ops.vit_embed_ln_fwd(PO, mod.cls_token_embedding, mod.positional_embedding, mod.ln_pre.weight, mod.ln_pre.bias,
                             X0, m0, r0, B, S, d, mod.ln_pre.eps)
        XM, Y = self.stack.forward(X0, B, S, save)
        XSEL = keep.get("img.XSEL", (B, d), f32)
        LNP = keep.get("img.LNP", (B, d), bf)
        mP = keep.get("img.mP", (B,), f32); rP = keep.get("img.rP", (B,), f32)
        ops.add_layernorm_fwd(XM, Y, XSEL, LNP, None, mod.ln_post.weight, mod.ln_post.bias, mP, rP, B, d, mod.ln_post.eps,
                              row_idx=None, rows_per_group=S)
        EMB = out if out is not None else torch.empty((B, self.E), device=image.device, dtype=f32)
        ops.gemm(LNP, st.shadow(mod.projection), b_mn=True, epilogue=ops.EPI_F32, out=EMB)
        if save is not None:
            save.B, save.S, save.P = B, S, P
        return EMB

    def forward(self, data, diff, save: Optional[Workspace] = None):
        """data: (image,).  save: the Workspace that keeps what the backward reads (default: a new one)."""
        save = Workspace(self.store.device) if save is None else save
        return (self._forward(*data, save),), save

    def infer(self, image: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self._forward(image, None, out)

    def backward(self, save: Workspace, dEMB: torch.Tensor, on_layer_done=None):
        """on_layer_done(l): called once every parameter gradient of layer l is final (data-parallel all-reduce)."""
        mod, st, ws, d = self.mod, self.store, self.ws, self.d
        B, S, P = save.B, save.S, save.P
        bf, f32 = torch.bfloat16, torch.float32
        M = B * S
        dEb = ops.cast_bf16(dEMB.contiguous().float())
        LNP, XSEL = save.get("img.LNP", (B, d), bf), save.get("img.XSEL", (B, d), f32)
        ops.gemm(LNP, dEb, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(mod.projection), accumulate=True)
        dLNP = ws.get("img.dLNP", (B, d), f32)
        ops.gemm(dEb, st.shadow(mod.projection), epilogue=ops.EPI_F32, out=dLNP)
        G = ws.get("img.G", (M, d), f32)
        Gb = ws.get("img.Gb", (M, d), bf)
        ops.zero_(G); ops.zero_(Gb)
        ops.layernorm_bwd(XSEL, None, dLNP, save.get("img.mP", (B,), f32), save.get("img.rP", (B,), f32),
                          mod.ln_post.weight, None, G, Gb, st.grad(mod.ln_post.weight), st.grad(mod.ln_post.bias), B, d,
                          row_idx=None, rows_per_group=S, gsum=self.stack.top_bias_grad())
        self.stack.backward(G, Gb, B, S, save=save, on_layer_done=on_layer_done, top_bias_done=True)
        PO = save.get("img.PO", (B * P, d), bf)
        DP = ws.get("img.DP", (B * P, d), bf)
        ops.vit_embed_ln_bwd(PO, mod.cls_token_embedding, mod.positional_embedding, G, save.get("img.m0", (M,), f32),
                             save.get("img.r0", (M,), f32), mod.ln_pre.weight, G, DP, st.grad(mod.ln_pre.weight),
                             st.grad(mod.ln_pre.bias), B, S, d)
        ops.batch_sum(G, st.grad(mod.positional_embedding), B, S * d, S * d)
        ops.batch_sum(G, st.grad(mod.cls_token_embedding), B, S * d, d)
        K = 3 * self.ps * self.ps
        PATCH = save.get("img.PATCH", (B * P, -(-K // 8) * 8), bf)[:, :K]
        ops.gemm(DP, PATCH, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad2d(mod.conv.weight),
                 splits=ops.wgrad_splits(d, PATCH.shape[1], B * P), accumulate=True)
        return ()


class TextTower:
    """CLIPTextEncoder runtime (models/clip/text_encoder.py:113-134).  Output: the embeddings fp32 [B, E]."""

    def __init__(self, mod: nn.Module):
        self.mod = mod
        self.store = ParamStore(list(mod.parameters()))
        self.ws = Workspace(self.store.device)
        layer0 = mod.encoder.layers[0]
        self.d = mod.width
        self.E = mod.projection.weight.shape[0]
        require_head_dim_64(self.d, layer0.self_attn.num_heads)
        self.stack = TransformerStack(mod.encoder.layers, self.store, self.ws, d=self.d,
                                      heads=layer0.self_attn.num_heads, ff=layer0.linear1.weight.shape[0],
                                      act=ops.ACT_QUICK_GELU, prefix="txt")

    def _forward(self, text: torch.Tensor, save: Optional[Workspace], return_hidden_state: bool = False,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
        mod, st, ws, d = self.mod, self.store, self.ws, self.d
        keep = save if save is not None else ws
        if text.dtype != torch.int64:
            text = text.long()
        text = text.contiguous()
        B, S = text.shape
        bf, f32 = torch.bfloat16, torch.float32
        st.refresh()
        X0 = keep.get("txt.X0", (B * S, d), f32)
        V = mod.token_embedding.weight.shape[0]
        ops.text_embed_fwd(text, mod.token_embedding.weight, mod.positional_embedding, X0, B, S, d, V)
        XM, Y = self.stack.forward(X0, B, S, save, causal=True)
        if return_hidden_state:
            HS = torch.empty((B, S, d), device=text.device, dtype=f32)
            ops.add_layernorm_fwd(XM, Y, None, None, HS, mod.ln_final.weight, mod.ln_final.bias, None, None, B * S, d,
                                  mod.ln_final.eps)
            return HS
        IDX = keep.get("txt.IDX", (B,), torch.int32)
        ops.argmax_tokens(text, IDX, B, S)
        XSEL = keep.get("txt.XSEL", (B, d), f32)
        LNF = keep.get("txt.LNF", (B, d), bf)
        mF = keep.get("txt.mF", (B,), f32); rF = keep.get("txt.rF", (B,), f32)
        ops.add_layernorm_fwd(XM, Y, XSEL, LNF, None, mod.ln_final.weight, mod.ln_final.bias, mF, rF, B, d,
                              mod.ln_final.eps, row_idx=IDX, rows_per_group=S)
        EMB = out if out is not None else torch.empty((B, self.E), device=text.device, dtype=f32)
        ops.gemm(LNF, st.shadow(mod.projection.weight), epilogue=ops.EPI_F32, out=EMB)
        if save is not None:
            save.B, save.S, save.tokens = B, S, text
        return EMB

    def forward(self, data, diff, save: Optional[Workspace] = None):
        """data: (text,).  save: the Workspace that keeps what the backward reads (default: a new one)."""
        save = Workspace(self.store.device) if save is None else save
        return (self._forward(*data, save),), save

    def infer(self, text: torch.Tensor, return_hidden_state: bool = False,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The embeddings, or with return_hidden_state the ln_final-ed hidden states fp32 [B, S, width]."""
        return self._forward(text, None, return_hidden_state, out)

    def backward(self, save: Workspace, dEMB: torch.Tensor, on_layer_done=None):
        mod, st, ws, d = self.mod, self.store, self.ws, self.d
        B, S = save.B, save.S
        bf, f32 = torch.bfloat16, torch.float32
        M = B * S
        dEb = ops.cast_bf16(dEMB.contiguous().float())
        LNF, XSEL = save.get("txt.LNF", (B, d), bf), save.get("txt.XSEL", (B, d), f32)
        ops.gemm(dEb, LNF, a_mn=True, b_mn=True, epilogue=ops.EPI_F32, out=st.grad(mod.projection.weight), accumulate=True)
        dLNF = ws.get("txt.dLNF", (B, d), f32)
        ops.gemm(dEb, st.shadow(mod.projection.weight), b_mn=True, epilogue=ops.EPI_F32, out=dLNF)
        G = ws.get("txt.G", (M, d), f32)
        Gb = ws.get("txt.Gb", (M, d), bf)
        ops.zero_(G); ops.zero_(Gb)
        IDX = save.get("txt.IDX", (B,), torch.int32)
        ops.layernorm_bwd(XSEL, None, dLNF, save.get("txt.mF", (B,), f32), save.get("txt.rF", (B,), f32),
                          mod.ln_final.weight, None, G, Gb, st.grad(mod.ln_final.weight), st.grad(mod.ln_final.bias), B,
                          d, row_idx=IDX, rows_per_group=S, gsum=self.stack.top_bias_grad())
        self.stack.backward(G, Gb, B, S, save=save, on_layer_done=on_layer_done, top_bias_done=True)
        ops.batch_sum(G, st.grad(mod.positional_embedding), B, S * d, S * d)
        ops.text_embed_bwd(save.tokens, G, st.grad(mod.token_embedding.weight), B, S, d)
        return ()


class RuntimeFunction(torch.autograd.Function):
    """One training forward of a runtime that keeps its activations.  inputs: (runtime, data, n_diff, *diff_inputs,
    *parameters).  rt.forward(data, diff) -> (outputs, save); rt.backward(save, *d outputs) -> gradients of diff."""

    @staticmethod
    def forward(ctx, rt, data, n_diff, *tensors):
        ctx.set_materialize_grads(False)   # an unused output arrives as None in backward, not as a zero tensor
        outs, save = rt.forward(data, tensors[:n_diff])
        ctx.rt, ctx.save, ctx.n_diff = rt, save, n_diff
        ctx.need = ctx.needs_input_grad[3 + n_diff:]
        return tuple(outs)

    @staticmethod
    def backward(ctx, *douts):
        rt, save = ctx.rt, ctx.save
        if save is None:
            raise MMBError("this forward was already back-propagated (its activations are freed)")
        st = rt.store
        flat = st.master is not None
        if not flat:
            st.zero_grads()
        in_grads = rt.backward(save, *douts)
        ctx.save = None
        if flat:  # p.grad are views of the flat buffer: gradients were accumulated in place
            # `optimizer.zero_grad(set_to_none=True)` (torch's default) or `p.grad = None` severs those views; re-attach
            # them, otherwise gradients would pile up invisibly in the flat buffer while the optimizer skips the parameter
            for p in st.params:
                want = st.grad(p)
                if p.grad is None or p.grad.data_ptr() != want.data_ptr():
                    p.grad = want
            return (None, None, None, *in_grads) + (None,) * len(st.params)
        g = st.g.clone()
        grads = []
        for p, need in zip(st.params, ctx.need):
            o = st.off[id(p)]
            grads.append(g[o:o + p.numel()].view(p.shape) if need else None)
        return (None, None, None, *in_grads, *grads)


def run(rt, data, diff: Sequence[torch.Tensor] = ()):
    return RuntimeFunction.apply(rt, data, len(diff), *diff, *rt.store.params)


class _RuntimeOwner(nn.Module):
    """Lazily (re)builds the module's fused runtime when the module moves or its parameters are replaced.  One runtime
    serves both grad modes: forward + explicit backward under autograd (`run`), and `infer` under torch.no_grad()."""

    _runtime_cls = None

    def _runtime(self, *extra: Optional[nn.Module]):
        """`extra`: modules outside this one whose parameters its fused front end owns (the multimodal projections)."""
        mods = [m for m in extra if m is not None]
        ids = [(id(p), p.device) for m in (self, *mods) for p in m.parameters()]
        if getattr(self, "_rt", None) is None or self._rt_ids != ids:
            object.__setattr__(self, "_rt", type(self)._runtime_cls(self, *extra))
            object.__setattr__(self, "_rt_ids", ids)
            watch_module(self)
        return self._rt
