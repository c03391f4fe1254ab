"""Typed Python wrappers over the C ABI (include/mmb200.h).

PyTorch is used here for device memory and streams only: every function takes CUDA tensors, checks dtype /
contiguity / device, and launches hand-written sm_90a kernels on ``torch.cuda.current_stream()``.  A CPU
tensor, a missing library or a non-zero status raises — there is no eager / CPU fallback.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib
from ._lib import MMBError

EPI_BF16, EPI_BF16_ACT, EPI_BF16_DACT, EPI_F32 = 0, 1, 2, 3
ACT_QUICK_GELU, ACT_GELU_ERF, ACT_RELU = 0, 1, 2

_NULL = ctypes.c_void_p(0)

# When set to a list, every GEMM launch is bracketed by CUDA events on the launching stream and appended as
# (algorithmic_flops, (a_mn, b_mn, epilogue), (start_event, end_event)) — used by bench.py for the live roofline.
GEMM_TIMING = None
# Same for the other kernel families of the step: (family, algorithmic work, unit, (start_event, end_event)) with
# family in {"attn_fwd", "attn_bwd", "ln_fwd", "ln_bwd"}; work in flops (attention) or bytes (LayerNorm passes).
FAMILY_TIMING = None


class _timed:
    """Brackets one launch with CUDA events on the current stream when FAMILY_TIMING is armed (bench.py only)."""

    __slots__ = ("fam", "work", "unit", "ev")

    def __init__(self, fam, work, unit):
        self.fam, self.work, self.unit, self.ev = fam, work, unit, None

    def __enter__(self):
        if FAMILY_TIMING is not None:
            self.ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self.ev[0].record()
        return self

    def __exit__(self, *exc):
        if self.ev is not None and exc[0] is None:
            self.ev[1].record()
            FAMILY_TIMING.append((self.fam, float(self.work), self.unit, self.ev))
        return False


def _p(t: Optional[torch.Tensor]):
    return _NULL if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise MMBError(f"{name}: expected a CUDA tensor (multimodal_b200 has no CPU path), got device {t.device}")
    if t.dtype != dtype:
        raise MMBError(f"{name}: expected dtype {dtype}, got {t.dtype}")


def _rowmajor(t: torch.Tensor, name: str):
    if t.dim() != 2 or t.stride(1) != 1:
        raise MMBError(f"{name}: expected a row-major 2-D tensor, got shape {tuple(t.shape)} stride {t.stride()}")


def gemm(A, B, *, a_mn=False, b_mn=False, epilogue=EPI_BF16, out=None, out2=None, bias=None, aux=None, alpha=1.0,
         act=ACT_QUICK_GELU, splits=1, accumulate=False, colsum=None):
    """D = alpha * op(A) @ op(B)^T (+bias).  A: [M,K] (a_mn: stored [K,M]); B: [N,K] (b_mn: stored [K,N])."""
    _chk(A, torch.bfloat16, "A"); _chk(B, torch.bfloat16, "B"); _rowmajor(A, "A"); _rowmajor(B, "B")
    M, K = (A.shape[1], A.shape[0]) if a_mn else (A.shape[0], A.shape[1])
    N, Kb = (B.shape[1], B.shape[0]) if b_mn else (B.shape[0], B.shape[1])
    if K != Kb:
        raise MMBError(f"gemm: contraction mismatch {K} vs {Kb}")
    odt = torch.float32 if epilogue == EPI_F32 else torch.bfloat16
    if out is None:
        out = torch.empty((M, N), device=A.device, dtype=odt)
    _chk(out, odt, "out"); _rowmajor(out, "out")
    if tuple(out.shape) != (M, N):
        raise MMBError(f"gemm: out shape {tuple(out.shape)} != {(M, N)}")
    if epilogue == EPI_BF16_ACT:
        if out2 is None:
            out2 = torch.empty((M, N), device=A.device, dtype=torch.bfloat16)
        _chk(out2, torch.bfloat16, "out2"); _rowmajor(out2, "out2")
    if bias is not None:
        _chk(bias, torch.float32, "bias")
    if aux is not None:
        _chk(aux, torch.bfloat16, "aux"); _rowmajor(aux, "aux")
    ev = None
    if GEMM_TIMING is not None:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    rc = _lib.lib().mmb_gemm_bf16(_p(A), A.stride(0), int(a_mn), _p(B), B.stride(0), int(b_mn), _p(out), out.stride(0),
                                  _p(out2), out2.stride(0) if out2 is not None else 0, M, N, K, epilogue, act,
                                  float(alpha), _p(bias), _p(aux), aux.stride(0) if aux is not None else 0,
                                  int(splits), int(accumulate), _p(colsum), _stream())
    _lib.check(rc, "mmb_gemm_bf16")
    if ev is not None:
        ev[1].record()
        GEMM_TIMING.append((2.0 * M * N * K, (int(a_mn), int(b_mn), epilogue), ev))
    return (out, out2) if epilogue == EPI_BF16_ACT else out


_CLUSTERS = {}


def _clusters_on_current_device() -> int:
    dev = torch.cuda.current_device()
    if dev not in _CLUSTERS:
        _CLUSTERS[dev] = torch.cuda.get_device_properties(dev).multi_processor_count // 2
    return _CLUSTERS[dev]


def wgrad_splits(out_rows: int, out_cols: int, k: int, n_units: Optional[int] = None) -> int:
    """Split-K factor for a weight-gradient GEMM so that the output's 256 x 128 blocks fill the machine (a 2-CTA
    cluster computes a 256 x 256 tile, two such blocks).  The count is kept at 256 x 128 so that every weight gradient
    keeps its split count, and with it its fp32 summation order: a changed split count reassociates the sum, and Adam's
    normalised update turns that into visibly different weights within a step.  n_units = 2-CTA clusters the GPU
    holds at once (default: half the current device's SM count, e.g. 66 on an H100 SXM, 57 on an H100 PCIe)."""
    if n_units is None:
        n_units = _clusters_on_current_device()
    tiles = ((out_rows + 255) // 256) * ((out_cols + 127) // 128)
    kb = (k + 63) // 64
    if tiles >= 2 * n_units:
        return 1
    best, best_eff = 1, 0.0
    for s in range(1, min(kb, 64) + 1):
        if kb // s < 8:  # keep each split's main loop long enough to amortise the prologue
            break
        waves = -(-tiles * s // n_units)
        eff = tiles * s / (waves * n_units)
        if eff >= 0.9:  # smallest split that fills >= 90% of the last wave: every extra split adds reduce-add traffic
            return s
        if eff > best_eff + 1e-9:
            best, best_eff = s, eff
    return best


def cast_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None, branch_scale: Optional[torch.Tensor] = None,
              rows_per_scale: int = 0) -> torch.Tensor:
    """bf16 copy of src; with branch_scale (fp32 [rows / rows_per_scale], stochastic depth), row r of the 2-D src is
    multiplied by branch_scale[r // rows_per_scale] first."""
    _chk(src, torch.float32, "src")
    if not src.is_contiguous():
        raise MMBError("cast_bf16: src must be contiguous")
    if out is None:
        out = torch.empty(src.shape, device=src.device, dtype=torch.bfloat16)
    _chk(out, torch.bfloat16, "out")
    if branch_scale is None:
        _lib.check(_lib.lib().mmb_cast_f32_to_bf16(_p(src), _p(out), src.numel(), _stream()), "mmb_cast_f32_to_bf16")
        return out
    if src.dim() != 2 or out.numel() != src.numel():
        raise MMBError("cast_bf16: a branch_scale needs a 2-D src [rows, d] and an out of the same size")
    _check_scale(branch_scale, src.shape[0], rows_per_scale)
    _lib.check(_lib.lib().mmb_cast_f32_to_bf16_scaled(_p(src), _p(out), src.numel(), _p(branch_scale),
                                                      rows_per_scale * src.shape[1], _stream()),
               "mmb_cast_f32_to_bf16_scaled")
    return out


def _check_scale(scale: torch.Tensor, M: int, rows_per_scale: int) -> None:
    """Per-sample stochastic-depth factors: contiguous fp32 with one entry per rows_per_scale rows of M."""
    _chk(scale, torch.float32, "branch_scale")
    if rows_per_scale <= 0 or M % rows_per_scale or not scale.is_contiguous() or scale.numel() != M // rows_per_scale:
        raise MMBError(f"branch_scale: expected a contiguous fp32 tensor of {M} / rows_per_scale = {rows_per_scale} "
                       f"entries, got shape {tuple(scale.shape)}")


def cast_f32(src: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _chk(src, torch.bfloat16, "src"); _chk(out, torch.float32, "out")
    if not (src.is_contiguous() and out.is_contiguous()) or src.numel() != out.numel():
        raise MMBError("cast_f32: contiguous tensors of equal size expected")
    _lib.check(_lib.lib().mmb_cast_bf16_to_f32(_p(src), _p(out), src.numel(), _stream()), "mmb_cast_bf16_to_f32")
    return out


def im2col(img: torch.Tensor, ps: int, out: torch.Tensor) -> torch.Tensor:
    _chk(img, torch.float32, "img"); _chk(out, torch.bfloat16, "out")
    B, C, H, W = img.shape
    _rowmajor(out, "out")
    _lib.check(_lib.lib().mmb_im2col_patches(_p(img), _p(out), out.stride(0), B, H, W, ps, _stream()), "mmb_im2col_patches")
    return out


# Patch dropping (csrc/patch_drop.cu): called by engine.patch_embed_fwd / patch_embed_bwd only; their kernel contracts
# are held in tests/test_gpu_patch_drop.py.
def _check_keep(keep: torch.Tensor) -> torch.Tensor:
    _chk(keep, torch.int32, "keep")
    if keep.dim() != 2 or not keep.is_contiguous():
        raise MMBError(f"keep: expected a contiguous int32 [B, L] tensor, got shape {tuple(keep.shape)}")
    return keep


def _im2col_gather(img: torch.Tensor, keep: torch.Tensor, ps: int, out: torch.Tensor) -> torch.Tensor:
    """im2col of the kept patches: out row b*L+j = patch keep[b, j] of image b (keep int32 [B, L])."""
    _chk(img, torch.float32, "img"); _chk(out, torch.bfloat16, "out"); _check_keep(keep)
    B, C, H, W = img.shape
    _rowmajor(out, "out")
    if keep.shape[0] != B or out.shape[0] != keep.numel():
        raise MMBError(f"im2col_gather: keep {tuple(keep.shape)} / out {tuple(out.shape)} do not match batch {B}")
    _lib.check(_lib.lib().mmb_im2col_patches_gather(_p(img), _p(keep), _p(out), out.stride(0), B, H, W, ps,
                                                    keep.shape[1], _stream()), "mmb_im2col_patches_gather")
    return out


def add_layernorm_fwd(x_in, y, x_out, ln_bf16, ln_f32, gamma, beta, mean, rstd, M, d, eps, row_idx=None,
                      rows_per_group=0, branch_scale=None, rows_per_scale=0):
    """x_out = x_in + y, LayerNorm of it.  branch_scale (fp32 [M / rows_per_scale], stochastic depth): row m adds
    branch_scale[m // rows_per_scale] * y instead (not with a row gather)."""
    nbytes = M * d * (4 + (2 if y is not None else 0) + (4 if x_out is not None else 0) +
                      (2 if ln_bf16 is not None else 0) + (4 if ln_f32 is not None else 0))
    if branch_scale is not None:
        if rows_per_group > 0 or y is None:
            raise MMBError("add_layernorm_fwd: a branch_scale needs y and excludes the row gather")
        _check_scale(branch_scale, M, rows_per_scale)
        with _timed("ln_fwd", nbytes + 4 * (M // rows_per_scale), "B"):
            _lib.check(_lib.lib().mmb_add_layernorm_fwd_scaled(_p(x_in), _p(y), _p(x_out), _p(ln_bf16), _p(ln_f32),
                                                               _p(gamma), _p(beta), _p(mean), _p(rstd), _p(branch_scale),
                                                               rows_per_scale, M, d, float(eps), _stream()),
                       "mmb_add_layernorm_fwd_scaled")
        return
    with _timed("ln_fwd", nbytes, "B"):
        _lib.check(_lib.lib().mmb_add_layernorm_fwd(_p(x_in), _p(y), _p(x_out), _p(ln_bf16), _p(ln_f32), _p(gamma),
                                                    _p(beta), _p(mean), _p(rstd), _p(row_idx), rows_per_group, M, d,
                                                    float(eps), _stream()), "mmb_add_layernorm_fwd")


def vit_embed_ln_fwd(patch_out, cls, pos, gamma, beta, x0, mean, rstd, B, S, d, eps):
    _lib.check(_lib.lib().mmb_vit_embed_ln_fwd(_p(patch_out), _p(cls), _p(pos), _p(gamma), _p(beta), _p(x0), _p(mean),
                                               _p(rstd), B, S, d, float(eps), _stream()), "mmb_vit_embed_ln_fwd")


def layernorm_bwd(x, dy_bf16, dy_f32, mean, rstd, gamma, g_in, g_out, g_bf16, dgamma, dbeta, M, d, row_idx=None,
                  rows_per_group=0, gsum=None, branch_scale=None, rows_per_scale=0):
    """LayerNorm backward + residual-gradient add.  branch_scale (fp32 [M / rows_per_scale], stochastic depth of the
    branch that consumes g_bf16): g_bf16 = bf16(branch_scale[m // rows_per_scale] * g_out) and gsum sums it; g_out is
    unscaled (not with a row scatter)."""
    nbytes = M * d * (4 + (2 if dy_bf16 is not None else 4) + (4 if g_in is not None else 0) +
                      (4 if g_out is not None else 0) + (2 if g_bf16 is not None else 0))
    if branch_scale is not None:
        if rows_per_group > 0 or g_bf16 is None:
            raise MMBError("layernorm_bwd: a branch_scale needs g_bf16 and excludes the row scatter")
        _check_scale(branch_scale, M, rows_per_scale)
        with _timed("ln_bwd", nbytes + 4 * (M // rows_per_scale), "B"):
            _lib.check(_lib.lib().mmb_layernorm_bwd_scaled(_p(x), _p(dy_bf16), _p(dy_f32), _p(mean), _p(rstd),
                                                           _p(gamma), _p(g_in), _p(g_out), _p(g_bf16), _p(dgamma),
                                                           _p(dbeta), _p(branch_scale), rows_per_scale, M, d, _p(gsum),
                                                           _stream()), "mmb_layernorm_bwd_scaled")
        return
    with _timed("ln_bwd", nbytes, "B"):
        _lib.check(_lib.lib().mmb_layernorm_bwd(_p(x), _p(dy_bf16), _p(dy_f32), _p(mean), _p(rstd), _p(gamma), _p(g_in),
                                                _p(g_out), _p(g_bf16), _p(dgamma), _p(dbeta), _p(row_idx),
                                                rows_per_group, M, d, _p(gsum), _stream()), "mmb_layernorm_bwd")


def vit_embed_ln_bwd(patch_out, cls, pos, dy_f32, mean, rstd, gamma, dt_f32, dpatch_bf16, dgamma, dbeta, B, S, d):
    _lib.check(_lib.lib().mmb_vit_embed_ln_bwd(_p(patch_out), _p(cls), _p(pos), _p(dy_f32), _p(mean), _p(rstd), _p(gamma),
                                               _p(dt_f32), _p(dpatch_bf16), _p(dgamma), _p(dbeta), B, S, d, _stream()),
               "mmb_vit_embed_ln_bwd")


def batch_sum(inp, out, Bn, ld, n):
    _lib.check(_lib.lib().mmb_batch_sum(_p(inp), _p(out), Bn, ld, n, _stream()), "mmb_batch_sum")


def colsum_bf16(x, out, M, N, ld):
    _lib.check(_lib.lib().mmb_colsum_bf16(_p(x), _p(out), M, N, ld, _stream()), "mmb_colsum_bf16")


def text_embed_fwd(tokens, emb, pos, x, B, S, d, V):
    _chk(tokens, torch.int64, "tokens")
    _lib.check(_lib.lib().mmb_text_embed_fwd(_p(tokens), _p(emb), _p(pos), _p(x), B, S, d, V, _stream()), "mmb_text_embed_fwd")


def text_embed_bwd(tokens, g, demb, B, S, d):
    _lib.check(_lib.lib().mmb_text_embed_bwd(_p(tokens), _p(g), _p(demb), B, S, d, _stream()), "mmb_text_embed_bwd")


def argmax_tokens(tokens, idx, B, S):
    _chk(tokens, torch.int64, "tokens"); _chk(idx, torch.int32, "idx")
    _lib.check(_lib.lib().mmb_argmax_tokens(_p(tokens), _p(idx), B, S, _stream()), "mmb_argmax_tokens")


def l2norm_fwd(x, y, y_bf16, inv_norm, B, E, eps=1e-12):
    _lib.check(_lib.lib().mmb_l2norm_fwd(_p(x), _p(y), _p(y_bf16), _p(inv_norm), B, E, float(eps), _stream()), "mmb_l2norm_fwd")


def l2norm_bwd(dy, y, inv_norm, dx, dx_bf16, B, E):
    _lib.check(_lib.lib().mmb_l2norm_bwd(_p(dy), _p(y), _p(inv_norm), _p(dx), _p(dx_bf16), B, E, _stream()), "mmb_l2norm_bwd")


def adamw_step(p, g, m, v, p_bf16, n, lr, beta1, beta2, eps, wd, step, grad_scale=1.0, zero_grad=True):
    _lib.check(_lib.lib().mmb_adamw_step(_p(p), _p(g), _p(m), _p(v), _p(p_bf16), n, lr, beta1, beta2, eps, wd, step,
                                         grad_scale, int(zero_grad), _stream()), "mmb_adamw_step")


def anyprecision_adamw_step(p, g, m, v, comp, p_bf16, lr, beta1, beta2, eps, wd, step, grad_scale=1.0, zero_grad=False):
    """One AnyPrecisionAdamW update of a flat fp32 tensor; m / v / comp may be fp32 or bf16 (comp=None: no Kahan)."""
    _chk(p, torch.float32, "p"); _chk(g, torch.float32, "g")
    code = {torch.float32: 0, torch.bfloat16: 1}
    for t, name in ((m, "exp_avg"), (v, "exp_avg_sq"), (comp, "compensation")):
        if t is not None and (not t.is_cuda or t.dtype not in code or t.numel() != p.numel()):
            raise MMBError(f"anyprecision_adamw_step: {name} must be a CUDA fp32/bf16 tensor of the parameter's size")
    _lib.check(_lib.lib().mmb_anyprecision_adamw_step(
        _p(p), _p(g), _p(m), code[m.dtype], _p(v), code[v.dtype], _p(comp), code[comp.dtype] if comp is not None else 0,
        _p(p_bf16), p.numel(), float(lr), float(beta1), float(beta2), float(eps), float(wd), int(step), float(grad_scale),
        int(zero_grad), _stream()), "mmb_anyprecision_adamw_step")


def act_fwd(x: torch.Tensor, kind: int) -> torch.Tensor:
    _chk(x, torch.float32, "x")
    if not x.is_contiguous():
        raise MMBError("act_fwd: x must be contiguous")
    y = torch.empty_like(x)
    _lib.check(_lib.lib().mmb_act_fwd(_p(x), _p(y), x.numel(), int(kind), _stream()), "mmb_act_fwd")
    return y


def zero_(t: torch.Tensor):
    if not t.is_cuda or not t.is_contiguous():
        raise MMBError("zero_: expected a contiguous CUDA tensor")
    _lib.check(_lib.lib().mmb_memset_async(_p(t), 0, t.numel() * t.element_size(), _stream()), "mmb_memset_async")
    return t


def attention_fwd(qkv, out, lse, B, S, H, causal, scale):
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    with _timed("attn_fwd", 4.0 * S * S * 64 * H * B * (0.5 if causal else 1.0), "F"):
        _lib.check(_lib.lib().mmb_attention_fwd(_p(qkv), _p(out), _p(lse), B, S, H, 64, int(causal), float(scale),
                                                _stream()), "mmb_attention_fwd")


def attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, scale):
    with _timed("attn_bwd", 10.0 * S * S * 64 * H * B * (0.5 if causal else 1.0), "F"):   # 2.5 x forward
        _lib.check(_lib.lib().mmb_attention_bwd(_p(qkv), _p(out), _p(dout), _p(lse), _p(dqkv), B, S, H, 64, int(causal),
                                                float(scale), _stream()), "mmb_attention_bwd")
        _lib.LAUNCHES += _lib.lib().mmb_attention_bwd_launches(S) - 1   # two kernels for the two-pass variants


def contrastive_ce_stats(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, row_loss, lse_out,
                         dscale_accum, logits_out=None, row_w=None):
    _chk(sims, torch.float32, "sims")
    _lib.check(_lib.lib().mmb_contrastive_ce_stats(_p(sims), sims.stride(0), _p(logit_scale), rows, N, label_offset,
                                                   float(smoothing), float(loss_weight), _p(row_loss), _p(lse_out),
                                                   _p(dscale_accum), _p(logits_out),
                                                   logits_out.stride(0) if logits_out is not None else 0, _p(row_w),
                                                   _stream()), "mmb_contrastive_ce_stats")


def contrastive_ce_grad(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, lse_row, lse_col, col_lo,
                        col_hi, dsims_bf16, dsims_f32, row_w=None, col_w=None):
    _chk(sims, torch.float32, "sims")
    d = dsims_bf16 if dsims_bf16 is not None else dsims_f32
    if dsims_bf16 is not None and dsims_f32 is not None and dsims_bf16.stride(0) != dsims_f32.stride(0):
        raise MMBError("contrastive_ce_grad: dsims_bf16 and dsims_f32 must share the leading dimension")
    _lib.check(_lib.lib().mmb_contrastive_ce_grad(_p(sims), sims.stride(0), _p(logit_scale), rows, N, label_offset,
                                                  float(smoothing), float(loss_weight), _p(lse_row), _p(lse_col),
                                                  int(col_lo), int(col_hi), _p(dsims_bf16), _p(dsims_f32), d.stride(0),
                                                  _p(row_w), _p(col_w), _stream()), "mmb_contrastive_ce_grad")


def gemm_ce_num_parts(N: int) -> int:
    return int(_lib.lib().mmb_gemm_ce_num_parts(int(N)))


def gemm_ce_stats(A, B, log_scale, label0, part, part0, xlabel):
    """Fused similarity GEMM + online-softmax statistics (logits never written): see include/mmb200.h."""
    _chk(A, torch.bfloat16, "A"); _chk(B, torch.bfloat16, "B"); _rowmajor(A, "A"); _rowmajor(B, "B")
    _chk(part, torch.float32, "part"); _chk(xlabel, torch.float32, "xlabel")
    M, K = A.shape
    N = B.shape[0]
    if B.shape[1] != K or part.dim() != 3 or part.shape[0] != M or part.shape[2] != 4 or not part.is_contiguous():
        raise MMBError("gemm_ce_stats: expected B [N,K] and a contiguous part buffer [M, parts, 4]")
    _lib.check(_lib.lib().mmb_gemm_ce_stats(_p(A), A.stride(0), _p(B), B.stride(0), M, N, K, _p(log_scale), int(label0),
                                            _p(part), part.shape[1], int(part0), _p(xlabel), _stream()), "mmb_gemm_ce_stats")


def linear_cross_entropy(hidden_bf16, weight_bf16, labels_i32, ignore_index, accum, row_loss=None):
    """Fused Linear(no bias) -> CrossEntropy(ignore_index): accum[0] += sum of kept rows' losses, accum[1] += count.
    The [M, V] logits are never written (mmb_gemm_ce_stats_labels + mmb_ce_labels_reduce)."""
    _chk(hidden_bf16, torch.bfloat16, "hidden"); _chk(weight_bf16, torch.bfloat16, "weight")
    _rowmajor(hidden_bf16, "hidden"); _rowmajor(weight_bf16, "weight")
    _chk(labels_i32, torch.int32, "labels"); _chk(accum, torch.float32, "accum")
    M, K = hidden_bf16.shape
    V = weight_bf16.shape[0]
    if weight_bf16.shape[1] != K or labels_i32.numel() != M or not labels_i32.is_contiguous():
        raise MMBError("linear_cross_entropy: expected weight [V, K] and contiguous int32 labels [M]")
    npar = gemm_ce_num_parts(V)
    part = torch.empty((M, npar, 4), device=hidden_bf16.device, dtype=torch.float32)
    xlabel = torch.zeros(M, device=hidden_bf16.device, dtype=torch.float32)
    zero = torch.zeros(1, device=hidden_bf16.device, dtype=torch.float32)      # log(temperature) = 0
    _lib.check(_lib.lib().mmb_gemm_ce_stats_labels(_p(hidden_bf16), hidden_bf16.stride(0), _p(weight_bf16),
                                                   weight_bf16.stride(0), M, V, K, _p(zero), _p(labels_i32), _p(part), npar, 0,
                                                   _p(xlabel), _stream()), "mmb_gemm_ce_stats_labels")
    _lib.check(_lib.lib().mmb_ce_labels_reduce(_p(part), npar, npar, _p(xlabel), _p(labels_i32), int(ignore_index), M,
                                               _p(row_loss), _p(accum), _stream()), "mmb_ce_labels_reduce")


def ce_stats_reduce(part, n_parts, xlabel, rows, n_total, smoothing, loss_weight, row_w, row_loss, lse_out, dscale_accum):
    _lib.check(_lib.lib().mmb_ce_stats_reduce(_p(part), part.shape[1], int(n_parts), _p(xlabel), rows, n_total,
                                              float(smoothing), float(loss_weight), _p(row_w), _p(row_loss), _p(lse_out),
                                              _p(dscale_accum), _stream()), "mmb_ce_stats_reduce")


def gemm_ce_grad(A, B, log_scale, label0, n_total, rows_total, smoothing, loss_weight, lse_row, row_w, lse_col, col_w,
                 col_lo, col_hi, dsims):
    """Recomputes the logits tile by tile and writes d loss / d sims (bf16) straight from the accumulators."""
    _chk(A, torch.bfloat16, "A"); _chk(B, torch.bfloat16, "B"); _rowmajor(A, "A"); _rowmajor(B, "B")
    _chk(dsims, torch.bfloat16, "dsims"); _rowmajor(dsims, "dsims")
    M, K = A.shape
    N = B.shape[0]
    if tuple(dsims.shape) != (M, N):
        raise MMBError(f"gemm_ce_grad: dsims shape {tuple(dsims.shape)} != {(M, N)}")
    _lib.check(_lib.lib().mmb_gemm_ce_grad(_p(A), A.stride(0), _p(B), B.stride(0), M, N, K, _p(log_scale), int(label0),
                                           int(n_total), int(rows_total), float(smoothing), float(loss_weight), _p(lse_row),
                                           _p(row_w), _p(lse_col), _p(col_w), int(col_lo), int(col_hi), _p(dsims),
                                           dsims.stride(0), _stream()), "mmb_gemm_ce_grad")


def sum_scale(inp, n, scale, out, accumulate=False):
    _lib.check(_lib.lib().mmb_sum_scale(_p(inp), n, float(scale), _p(out), int(accumulate), _stream()), "mmb_sum_scale")


def matmul_f32(A, B, *, ta=False, tb=False, out=None, alpha=1.0, accumulate=False):
    """fp32 SIMT matmul (tiny / unaligned shapes).  C = alpha * op(A) @ op(B); ta: A stored [K,M]; tb: B stored [N,K]."""
    _chk(A, torch.float32, "A"); _chk(B, torch.float32, "B"); _rowmajor(A, "A"); _rowmajor(B, "B")
    M, K = (A.shape[1], A.shape[0]) if ta else (A.shape[0], A.shape[1])
    N, Kb = (B.shape[0], B.shape[1]) if tb else (B.shape[1], B.shape[0])
    if K != Kb:
        raise MMBError(f"matmul_f32: contraction mismatch {K} vs {Kb}")
    if out is None:
        out = torch.empty((M, N), device=A.device, dtype=torch.float32)
    _lib.check(_lib.lib().mmb_matmul_f32(_p(A), A.stride(0), int(ta), _p(B), B.stride(0), int(tb), _p(out), out.stride(0),
                                         M, N, K, float(alpha), int(accumulate), _stream()), "mmb_matmul_f32")
    return out


# ---- FLAVA forward helpers -----------------------------------------------------------------------------------------
def attention_fwd_kmask(qkv, out, lse, kmask, B, S, H, causal, scale):
    _chk(qkv, torch.bfloat16, "qkv"); _chk(kmask, torch.uint8, "kmask")
    _lib.check(_lib.lib().mmb_attention_fwd_kmask(_p(qkv), _p(out), _p(lse), _p(kmask), B, S, H, 64, int(causal),
                                                  float(scale), _stream()), "mmb_attention_fwd_kmask")


def attention_probs(qkv, lse, kmask, probs, B, S, H, causal, scale):
    _chk(qkv, torch.bfloat16, "qkv"); _chk(lse, torch.float32, "lse"); _chk(probs, torch.float32, "probs")
    _lib.check(_lib.lib().mmb_attention_probs(_p(qkv), _p(lse), _p(kmask), _p(probs), B, S, H, int(causal), float(scale),
                                              _stream()), "mmb_attention_probs")


def bert_embed_ln_fwd(ids, type_ids, word, pos, type_emb, gamma, beta, x, kmask_out, pad_id, B, S, d, V, eps):
    _chk(ids, torch.int64, "ids")
    _lib.check(_lib.lib().mmb_bert_embed_ln_fwd(_p(ids), _p(type_ids), _p(word), _p(pos), _p(type_emb), _p(gamma), _p(beta),
                                                _p(x), _p(kmask_out), int(pad_id), B, S, d, V, float(eps), _stream()),
               "mmb_bert_embed_ln_fwd")


def vit_assemble_fwd(patch_out, cls, pos, mask_token, patch_mask, x, B, S, d):
    _lib.check(_lib.lib().mmb_vit_assemble_fwd(_p(patch_out), _p(cls), _p(pos), _p(mask_token), _p(patch_mask), _p(x), B, S,
                                               d, _stream()), "mmb_vit_assemble_fwd")


def _vit_assemble_gather_fwd(patch_out, cls, pos, mask_token, patch_mask, keep, x, P, d):
    """x [B*(off+L), d] from the kept patches' projections patch_out [B*L, d] (keep int32 [B, L], P patches)."""
    _check_keep(keep)
    B, L = keep.shape
    _lib.check(_lib.lib().mmb_vit_assemble_gather_fwd(_p(patch_out), _p(cls), _p(pos), _p(mask_token), _p(patch_mask),
                                                      _p(keep), _p(x), B, L, P, d, _stream()),
               "mmb_vit_assemble_gather_fwd")


def gather_rows_cast(x, out, B, rows_per_group, row, d):
    _lib.check(_lib.lib().mmb_gather_rows_cast(_p(x), _p(out), B, rows_per_group, row, d, _stream()), "mmb_gather_rows_cast")


def gather_rows_idx_cast(x, idx, out, d):
    """out[m, :] = bf16(x2d[idx[m], :]); x fp32 viewed as rows of `d` elements with row pitch x.stride(-2)."""
    _chk(x, torch.float32, "x"); _chk(idx, torch.int64, "idx"); _chk(out, torch.bfloat16, "out")
    if x.stride(-1) != 1 or not idx.is_contiguous() or not out.is_contiguous():
        raise MMBError("gather_rows_idx_cast: expected unit inner stride, contiguous idx / out")
    _lib.check(_lib.lib().mmb_gather_rows_idx_cast(_p(x), x.stride(-2), _p(idx), _p(out), idx.numel(), d, _stream()),
               "mmb_gather_rows_idx_cast")
    return out


def tanh_(x):
    _chk(x, torch.float32, "x")
    _lib.check(_lib.lib().mmb_tanh_inplace(_p(x), x.numel(), _stream()), "mmb_tanh_inplace")
    return x


def concat_tokens(cls, a, b, out, B, Sa, Sb, d):
    _lib.check(_lib.lib().mmb_concat_tokens(_p(cls), _p(a), _p(b), _p(out), B, Sa, Sb, d, _stream()), "mmb_concat_tokens")


# ---- CoCa forward helpers ---------------------------------------------------------------------------------------
def coca_text_embed_fwd(ids, emb, cls, pos, x, B, S, d, V):
    _chk(ids, torch.int64, "ids")
    _lib.check(_lib.lib().mmb_coca_text_embed_fwd(_p(ids), _p(emb), _p(cls), _p(pos), _p(x), B, S, d, V, _stream()),
               "mmb_coca_text_embed_fwd")


def self_attention(qkv, out, lse, B, S, H, head_dim, causal, scale, *, kmask=None, mask=None, dout=None, dqkv=None):
    """Self-attention on a packed [B*S, 3*H*head_dim] QKV buffer: the forward, or with dout / dqkv its backward.  The
    one place that picks the kernel, so a forward and its backward, in any grad mode, always run the same one:
      kmask (uint8 [B*S] key-padding mask)      -> the key-masked fused kernels (head_dim 64 only);
      mask (uint8 [B, S, S]) or head_dim != 64  -> the general kernels (lse unused);
      otherwise                                 -> the fused kernels."""
    if kmask is not None and mask is not None:
        raise MMBError("self_attention: pass either a key-padding mask or a [B, S, S] mask, not both")
    if kmask is not None and head_dim != 64:
        raise MMBError(f"self_attention: the key-padding-mask kernels support head_dim 64 only (got {head_dim}); "
                       "pass the mask as a [B, S, S] mask instead")
    if kmask is not None:
        if dout is None:
            attention_fwd_kmask(qkv, out, lse, kmask, B, S, H, causal, scale)
        else:
            attention_bwd_kmask(qkv, out, dout, lse, dqkv, kmask, B, S, H, causal, scale)
    elif mask is not None or head_dim != 64:
        d = H * head_dim
        kw = dict(B=B, Sq=S, Skv=S, H=H, head_dim=head_dim, bsq=S * 3 * d, bsk=S * 3 * d, bsv=S * 3 * d, bso=S * d,
                  scale=scale, mask=mask, mask_bs=S * S if mask is not None else 0,
                  mask_qs=S if mask is not None else 0, causal=causal)
        if dout is None:
            attention_fwd_generic(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], out, **kw)
        else:
            attention_bwd_generic(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], dout, dqkv[:, d:2 * d], dqkv[:, 2 * d:],
                                  dq=dqkv[:, :d], **kw)
    elif dout is None:
        attention_fwd(qkv, out, lse, B, S, H, causal, scale)
    else:
        attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, scale)


def attention_fwd_generic(q, k, v, out, *, B, Sq, Skv, H, head_dim, bsq, bsk, bsv, bso, scale, mask=None, mask_bs=0,
                          mask_qs=0, causal=False):
    """q/k/v/out: 2-D bf16 views [rows, >= H*head_dim] (row-major, possibly column slices of a wider matrix)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        _chk(t, torch.bfloat16, n); _rowmajor(t, n)
    if mask is not None:
        _chk(mask, torch.uint8, "mask")
    _lib.check(_lib.lib().mmb_attention_fwd_generic(_p(q), q.stride(0), int(bsq), _p(k), k.stride(0), int(bsk), _p(v),
                                                    v.stride(0), int(bsv), _p(out), out.stride(0), int(bso), _p(mask),
                                                    int(mask_bs), int(mask_qs), B, Sq, Skv, H, head_dim, int(causal),
                                                    float(scale), _stream()), "mmb_attention_fwd_generic")


# Longest query the split-KV decode kernel takes (one m16 tile); longer queries run attention_fwd_generic.
DECODE_MAX_SQ = 16


def decode_attention_wins(B: int, H: int, Sq: int, Skv: int) -> bool:
    """Whether attention_fwd_decode beats attention_fwd_generic at this shape (scripts/decode_bench.py, DESIGN.md §9):
    at every Sq <= 16 except short caches over many (batch, head) pairs, where both launch one CTA per pair and the
    general kernel's wider CTAs win (Skv 77, B 64, H 12: 24-26 us against 34-40 us at head_dim 64)."""
    return Sq <= DECODE_MAX_SQ and not (Skv <= 128 and B * H >= 264)


def attention_fwd_decode(q, k, v, out, *, B, Sq, Skv, H, head_dim, bsq, bsk, bsv, bso, scale, mask=None, mask_bs=0,
                         mask_qs=0, causal=False):
    """attention_fwd_generic's contract for Sq <= DECODE_MAX_SQ, on the split-KV decode kernel."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        _chk(t, torch.bfloat16, n); _rowmajor(t, n)
    if mask is not None:
        _chk(mask, torch.uint8, "mask")
    _lib.check(_lib.lib().mmb_attention_fwd_decode(_p(q), q.stride(0), int(bsq), _p(k), k.stride(0), int(bsk), _p(v),
                                                   v.stride(0), int(bsv), _p(out), out.stride(0), int(bso), _p(mask),
                                                   int(mask_bs), int(mask_qs), B, Sq, Skv, H, head_dim, int(causal),
                                                   float(scale), _stream()), "mmb_attention_fwd_decode")


def attention_decode_splits(B: int, H: int, Skv: int) -> int:
    return int(_lib.lib().mmb_attention_decode_splits(int(B), int(H), int(Skv)))


def kv_cache_append(past, new_rows, out, out_bf16, *, B, H, Sp, Sn, head_dim):
    """cat(past, new) along the sequence into row-major [B, Sp + Sn, H*head_dim] buffers.  past: [B, H, Sp, head_dim]
    fp32 / bf16 with unit inner stride (or None when Sp = 0); new_rows: bf16 2-D view [B*Sn, >= H*head_dim]; out: fp32
    or bf16, out_bf16: bf16 (either may be None)."""
    _chk(new_rows, torch.bfloat16, "new_rows"); _rowmajor(new_rows, "new_rows")
    if past is not None:
        if past.dtype not in (torch.float32, torch.bfloat16) or not past.is_cuda or past.stride(-1) != 1:
            raise MMBError("kv_cache_append: past must be a CUDA fp32 / bf16 tensor with unit stride along head_dim")
        if tuple(past.shape) != (B, H, Sp, head_dim):
            raise MMBError(f"kv_cache_append: past shape {tuple(past.shape)} != {(B, H, Sp, head_dim)}")
    for t, n in ((out, "out"), (out_bf16, "out_bf16")):
        if t is not None and (not t.is_cuda or not t.is_contiguous() or t.numel() != B * (Sp + Sn) * H * head_dim):
            raise MMBError(f"kv_cache_append: {n} must be a contiguous CUDA tensor of B * (Sp + Sn) * H * head_dim elements")
    if out is not None and out.dtype not in (torch.float32, torch.bfloat16):
        raise MMBError(f"kv_cache_append: out dtype {out.dtype} is not fp32 / bf16")
    if out_bf16 is not None:
        _chk(out_bf16, torch.bfloat16, "out_bf16")
    ps = past.stride() if past is not None else (0, 0, 0, 1)
    _lib.check(_lib.lib().mmb_kv_cache_append(_p(past), int(past is not None and past.dtype == torch.float32), ps[0],
                                              ps[1], ps[2], _p(new_rows), new_rows.stride(0), _p(out),
                                              int(out is not None and out.dtype == torch.float32), _p(out_bf16), B, H, Sp,
                                              Sn, head_dim, _stream()), "mmb_kv_cache_append")


def ce_labels(logits, labels, label_stride, ignore_index, M, V, row_loss, accum):
    _chk(logits, torch.float32, "logits"); _chk(labels, torch.int64, "labels"); _rowmajor(logits, "logits")
    _lib.check(_lib.lib().mmb_ce_labels(_p(logits), logits.stride(0), _p(labels), int(label_stride), int(ignore_index), M,
                                        V, _p(row_loss), _p(accum), _stream()), "mmb_ce_labels")


# ---- FLAVA / CoCa backward helpers ------------------------------------------------------------------------------
def attention_bwd_kmask(qkv, out, dout, lse, dqkv, kmask, B, S, H, causal, scale):
    _chk(qkv, torch.bfloat16, "qkv"); _chk(kmask, torch.uint8, "kmask")
    with _timed("attn_bwd", 10.0 * S * S * 64 * H * B, "F"):
        _lib.check(_lib.lib().mmb_attention_bwd_kmask(_p(qkv), _p(out), _p(dout), _p(lse), _p(dqkv), _p(kmask), B, S, H, 64,
                                                      int(causal), float(scale), _stream()), "mmb_attention_bwd_kmask")
        _lib.LAUNCHES += _lib.lib().mmb_attention_bwd_launches(S) - 1


def bert_embed_ln_bwd(ids, type_ids, word, pos, type_emb, gamma, dy, dword, dpos, dtype_emb, dgamma, dbeta, B, S, d, V, eps):
    _chk(ids, torch.int64, "ids"); _chk(dy, torch.float32, "dy")
    _lib.check(_lib.lib().mmb_bert_embed_ln_bwd(_p(ids), _p(type_ids), _p(word), _p(pos), _p(type_emb), _p(gamma), _p(dy),
                                                _p(dword), _p(dpos), _p(dtype_emb), _p(dgamma), _p(dbeta), B, S, d, V,
                                                float(eps), _stream()), "mmb_bert_embed_ln_bwd")


def vit_assemble_bwd(g, patch_mask, dpatch, dmask_token, B, S, d, has_cls=True):
    _chk(g, torch.float32, "g"); _chk(dpatch, torch.bfloat16, "dpatch")
    _lib.check(_lib.lib().mmb_vit_assemble_bwd(_p(g), _p(patch_mask), _p(dpatch), _p(dmask_token), B, S, d, int(has_cls),
                                               _stream()), "mmb_vit_assemble_bwd")


def _vit_assemble_gather_bwd(g, patch_mask, keep, dpatch, dmask_token, dcls, dpos, P, d, has_cls=True):
    """Backward of vit_assemble_gather_fwd; dmask_token / dcls / dpos are added into (+=), each may be None."""
    _chk(g, torch.float32, "g"); _chk(dpatch, torch.bfloat16, "dpatch"); _check_keep(keep)
    B, L = keep.shape
    _lib.check(_lib.lib().mmb_vit_assemble_gather_bwd(_p(g), _p(patch_mask), _p(keep), _p(dpatch), _p(dmask_token),
                                                      _p(dcls), _p(dpos), B, L, P, d, int(has_cls), _stream()),
               "mmb_vit_assemble_gather_bwd")


def split_tokens_cast(g, a, b, B, Sa, Sb, d, has_cls=True):
    _chk(g, torch.float32, "g")
    _lib.check(_lib.lib().mmb_split_tokens_cast(_p(g), _p(a), _p(b), B, Sa, Sb, d, int(has_cls), _stream()),
               "mmb_split_tokens_cast")


def tanh_bwd(dy, y, dx=None, dx_bf16=None):
    _chk(dy, torch.float32, "dy"); _chk(y, torch.float32, "y")
    if not (dy.is_contiguous() and y.is_contiguous()) or dy.numel() != y.numel():
        raise MMBError("tanh_bwd: contiguous tensors of equal size expected")
    _lib.check(_lib.lib().mmb_tanh_bwd(_p(dy), _p(y), _p(dx), _p(dx_bf16), y.numel(), _stream()), "mmb_tanh_bwd")


def scatter_rows_add(src, dst, B, rows_per_group, row, d):
    _chk(src, torch.float32, "src"); _chk(dst, torch.float32, "dst")
    _lib.check(_lib.lib().mmb_scatter_rows_add(_p(src), _p(dst), B, rows_per_group, row, d, _stream()),
               "mmb_scatter_rows_add")


def scatter_rows_idx_add(src, idx, dst, d):
    """dst2d[idx[m], :] += src[m, :]; dst fp32 viewed as rows of `d` elements with row pitch dst.stride(-2)."""
    _chk(src, torch.float32, "src"); _chk(idx, torch.int64, "idx"); _chk(dst, torch.float32, "dst")
    if not src.is_contiguous() or not idx.is_contiguous() or dst.stride(-1) != 1:
        raise MMBError("scatter_rows_idx_add: contiguous src / idx and unit inner stride of dst expected")
    _lib.check(_lib.lib().mmb_scatter_rows_idx_add(_p(src), _p(idx), _p(dst), dst.stride(-2), idx.numel(), d, _stream()),
               "mmb_scatter_rows_idx_add")


def ce_labels_bwd(logits, labels, label_stride, ignore_index, M, V, accum, grad_scale, dlogits, gscale=None):
    """gscale: optional fp32 device scalar multiplied into grad_scale (the incoming d loss; no host read-back)."""
    _chk(logits, torch.float32, "logits"); _chk(labels, torch.int64, "labels"); _chk(dlogits, torch.bfloat16, "dlogits")
    _rowmajor(logits, "logits"); _rowmajor(dlogits, "dlogits")
    if gscale is not None:
        _chk(gscale, torch.float32, "gscale")
    _lib.check(_lib.lib().mmb_ce_labels_bwd(_p(logits), logits.stride(0), _p(labels), int(label_stride), int(ignore_index),
                                            M, V, _p(accum), float(grad_scale), _p(gscale), _p(dlogits), dlogits.stride(0),
                                            _stream()), "mmb_ce_labels_bwd")


def act_bwd(dy, pre, dx, kind):
    _chk(dy, torch.bfloat16, "dy"); _chk(pre, torch.bfloat16, "pre"); _chk(dx, torch.bfloat16, "dx")
    if not (dy.is_contiguous() and pre.is_contiguous() and dx.is_contiguous()) or not (dy.numel() == pre.numel() == dx.numel()):
        raise MMBError("act_bwd: contiguous bf16 tensors of equal size expected")
    _lib.check(_lib.lib().mmb_act_bwd(_p(dy), _p(pre), _p(dx), dy.numel(), int(kind), _stream()), "mmb_act_bwd")


def attention_bwd_generic(q, k, v, dout, dk, dv, *, B, Sq, Skv, H, head_dim, bsq, bsk, bsv, bso, scale, dq=None,
                          dq_f32=None, mask=None, mask_bs=0, mask_qs=0, causal=False):
    """Backward of attention_fwd_generic.  q/k/v/dout and dq/dk/dv: 2-D bf16 views (dq/dk/dv with the row / batch strides
    of q/k/v).  dq_f32: fp32 [Sq, >= H*head_dim], zeroed by the caller, for batch-shared queries (bsq = 0)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (dout, "dout"), (dk, "dk"), (dv, "dv")):
        _chk(t, torch.bfloat16, n); _rowmajor(t, n)
    if dk.stride(0) != k.stride(0) or dv.stride(0) != v.stride(0) or (dq is not None and dq.stride(0) != q.stride(0)):
        raise MMBError("attention_bwd_generic: dq / dk / dv must have the row strides of q / k / v")
    if dq is not None:
        _chk(dq, torch.bfloat16, "dq"); _rowmajor(dq, "dq")
    if dq_f32 is not None:
        _chk(dq_f32, torch.float32, "dq_f32"); _rowmajor(dq_f32, "dq_f32")
    if mask is not None:
        _chk(mask, torch.uint8, "mask")
    scratch = torch.empty(2 * B * H * Sq, device=q.device, dtype=torch.float32)
    _lib.check(_lib.lib().mmb_attention_bwd_generic(
        _p(q), q.stride(0), int(bsq), _p(k), k.stride(0), int(bsk), _p(v), v.stride(0), int(bsv), _p(dout), dout.stride(0),
        int(bso), _p(mask), int(mask_bs), int(mask_qs), _p(dq), _p(dq_f32), dq_f32.stride(0) if dq_f32 is not None else 0,
        _p(dk), _p(dv), _p(scratch), B, Sq, Skv, H, head_dim, int(causal), float(scale), _stream()),
        "mmb_attention_bwd_generic")


# ---- GPU input pipeline (image transform) -----------------------------------------------------------------------
def clip_image_transform_max_taps() -> int:
    return int(_lib.lib().mmb_clip_image_transform_max_taps())


def clip_image_transform(src_ptrs, geom, out, mean, std):
    """src_ptrs int64 [n] (device pointers of HWC uint8 images), geom int32 [n, 12] (include/mmb200.h), out fp32
    [n, 3, S, S]; mean / std: 3 Python floats each."""
    _chk(src_ptrs, torch.int64, "src_ptrs"); _chk(geom, torch.int32, "geom"); _chk(out, torch.float32, "out")
    n, _, S, S2 = out.shape
    if S != S2 or tuple(geom.shape) != (n, 12) or src_ptrs.numel() != n or not (geom.is_contiguous() and out.is_contiguous()):
        raise MMBError("clip_image_transform: expected geom [n, 12], src_ptrs [n], out [n, 3, S, S] (contiguous)")
    table = torch.empty((n, 2, S, 2 + clip_image_transform_max_taps()), device=out.device, dtype=torch.int32)
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    _lib.check(_lib.lib().mmb_clip_image_transform(_p(src_ptrs), _p(geom), _p(table), _p(out), n, S,
                                                   ctypes.cast(m3, ctypes.c_void_p), ctypes.cast(s3, ctypes.c_void_p),
                                                   _stream()), "mmb_clip_image_transform")
    return out
