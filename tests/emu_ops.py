"""TEST INFRASTRUCTURE ONLY: torch (CPU) emulation of the C-ABI kernels' CONTRACTS, as documented in include/mmb200.h.

Purpose: the host-side schedules (engine.py / engine_flava_train.py: which buffer goes to which kernel, in which order,
which gradient slot accumulates what) are plain Python and can be checked without a GPU by swapping `multimodal_b200.ops`
entry points for these functions (``install(monkeypatch)``) and comparing the result with autograd over the oracle.
The emulation keeps the kernels' storage types (bf16 tensors are rounded exactly where the kernels round) and fp32
arithmetic; it is never imported by the package and is not a fallback — the product raises without the CUDA library.
"""
import math

import torch

BF, F32 = torch.bfloat16, torch.float32
EPI_BF16, EPI_BF16_ACT, EPI_BF16_DACT, EPI_F32 = 0, 1, 2, 3


def _act(x, kind):
    return x * torch.sigmoid(1.702 * x) if kind == 0 else torch.nn.functional.gelu(x)


def _act_grad(x, kind):
    if kind == 0:
        s = torch.sigmoid(1.702 * x)
        return s * (1 + 1.702 * x * (1 - s))
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def gemm(A, B, *, a_mn=False, b_mn=False, epilogue=EPI_BF16, out=None, out2=None, bias=None, aux=None, alpha=1.0,
         act=0, splits=1, accumulate=False, colsum=None):
    assert A.dtype == BF and B.dtype == BF
    Af = A.float().t() if a_mn else A.float()
    Bf = B.float().t() if b_mn else B.float()
    assert Af.shape[1] == Bf.shape[1], (Af.shape, Bf.shape)
    acc = alpha * (Af @ Bf.t())
    M, N = acc.shape
    assert not (accumulate and epilogue != EPI_F32) and not (bias is not None and epilogue == EPI_BF16_DACT)
    assert colsum is None or epilogue in (EPI_BF16, EPI_BF16_DACT)
    if bias is not None:
        assert bias.dtype == F32 and bias.numel() == N
        acc = acc + bias.detach().view(1, N)
    odt = F32 if epilogue == EPI_F32 else BF
    if out is None:
        out = torch.empty((M, N), dtype=odt)
    assert out.dtype == odt and tuple(out.shape) == (M, N), (out.dtype, out.shape, (M, N))
    if epilogue == EPI_F32:
        out.copy_(out + acc if accumulate else acc)
        return out
    if epilogue == EPI_BF16:
        out.copy_(acc.to(BF))
        if colsum is not None:
            colsum.add_(out.float().sum(0))
        return out
    if epilogue == EPI_BF16_ACT:
        if out2 is None:
            out2 = torch.empty((M, N), dtype=BF)
        out.copy_(acc.to(BF))
        out2.copy_(_act(out.float(), act).to(BF))
        return out, out2
    assert epilogue == EPI_BF16_DACT and aux is not None and aux.dtype == BF
    res = (acc * _act_grad(aux.float(), act)).to(BF)
    out.copy_(res)
    if colsum is not None:
        colsum.add_(res.float().sum(0))
    return out


def cast_bf16(src, out=None):
    assert src.dtype == F32
    if out is None:
        out = torch.empty(src.shape, dtype=BF)
    out.copy_(src.detach().to(BF).view(out.shape))
    return out


def zero_(t):
    t.zero_()
    return t


def im2col(img, ps, out):
    B, C, H, W = img.shape
    cols = torch.nn.functional.unfold(img, kernel_size=ps, stride=ps)      # [B, C*ps*ps, P]
    out.copy_(cols.transpose(1, 2).reshape(-1, C * ps * ps).to(BF))
    return out


def _ln_rows(x, gamma, beta, eps):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    return (x - mean) * rstd * gamma.detach() + beta.detach(), mean.squeeze(-1), rstd.squeeze(-1)


def add_layernorm_fwd(x_in, y, x_out, ln_bf16, ln_f32, gamma, beta, mean, rstd, M, d, eps, row_idx=None,
                      rows_per_group=0):
    if rows_per_group > 0:
        phys = torch.arange(M) * rows_per_group + (row_idx.long() if row_idx is not None else 0)
    else:
        phys = torch.arange(M)
    x = torch.zeros(M, d)
    if x_in is not None:
        x = x + x_in.detach().reshape(-1, d)[phys]
    if y is not None:
        x = x + y.reshape(-1, d)[phys].float()
    out, m, r = _ln_rows(x, gamma, beta, eps)
    if x_out is not None:
        x_out.view(-1, d)[:M].copy_(x)
    if ln_bf16 is not None:
        ln_bf16.view(-1, d)[:M].copy_(out.to(BF))
    if ln_f32 is not None:
        ln_f32.view(-1, d)[:M].copy_(out)
    if mean is not None:
        mean.copy_(m)
    if rstd is not None:
        rstd.copy_(r)


def layernorm_bwd(x, dy_bf16, dy_f32, mean, rstd, gamma, g_in, g_out, g_bf16, dgamma, dbeta, M, d, row_idx=None,
                  rows_per_group=0, gsum=None):
    assert (dy_bf16 is None) != (dy_f32 is None)
    if rows_per_group > 0:
        phys = torch.arange(M) * rows_per_group + (row_idx.long() if row_idx is not None else 0)
    else:
        phys = torch.arange(M)
    xx = x.detach().reshape(-1, d)[:M]
    dy = (dy_bf16.float() if dy_bf16 is not None else dy_f32).reshape(-1, d)[:M]
    h = (xx - mean.view(M, 1)) * rstd.view(M, 1)
    if dgamma is not None:
        dgamma.add_((dy * h).sum(0))
    if dbeta is not None:
        dbeta.add_(dy.sum(0))
    dyg = dy * gamma.detach()
    dx = rstd.view(M, 1) * (dyg - dyg.mean(-1, keepdim=True) - h * (dyg * h).mean(-1, keepdim=True))
    if g_in is not None:
        dx = dx + g_in.reshape(-1, d)[phys]
    if g_out is not None:
        g_out.view(-1, d)[phys] = dx
    if g_bf16 is not None:
        gb = dx.to(BF)
        g_bf16.view(-1, d)[phys] = gb
        if gsum is not None:
            gsum.add_(gb.float().sum(0))


def batch_sum(inp, out, Bn, ld, n):
    flat = inp.detach().reshape(-1)
    rows = torch.stack([flat[b * ld:b * ld + n] for b in range(Bn)])
    out.view(-1)[:n].add_(rows.sum(0))


def colsum_bf16(x, out, M, N, ld):
    assert x.dtype == BF
    out.view(-1)[:N].add_(x.reshape(-1, ld)[:M, :N].float().sum(0))


def _attn(qkv, B, S, H, causal, scale, kmask):
    d = H * 64
    q, k, v = (t.reshape(B, S, H, 64).transpose(1, 2) for t in qkv.float().view(B, S, 3 * d).split(d, dim=-1))
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        s = s + torch.full((S, S), float("-inf")).triu(1)
    if kmask is not None:
        s = s.masked_fill(~kmask.view(B, 1, 1, S).bool(), float("-inf"))
    return q, k, v, s


def _softmax_rows(s):
    """softmax over the keys; a row with no visible key (all -inf) gets p = 0, with a zero gradient, as the kernels
    give it O = 0 and no backward contribution (include/mmb200.h)."""
    vis = (s > float("-inf")).any(-1, keepdim=True)
    return torch.softmax(torch.where(vis, s, torch.zeros_like(s)), -1) * vis


def attention_fwd(qkv, out, lse, B, S, H, causal, scale, kmask=None):
    q, k, v, s = _attn(qkv, B, S, H, causal, scale, kmask)
    out.copy_((_softmax_rows(s) @ v).transpose(1, 2).reshape(B * S, H * 64).to(BF))
    if lse is not None:
        lse.copy_(torch.logsumexp(s, -1).reshape(-1))


def attention_fwd_kmask(qkv, out, lse, kmask, B, S, H, causal, scale):
    attention_fwd(qkv, out, lse, B, S, H, causal, scale, kmask)


def attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, scale, kmask=None):
    qf = qkv.float().requires_grad_(True)
    with torch.enable_grad():
        _, _, v, s = _attn(qf, B, S, H, causal, scale, kmask)
        o = (_softmax_rows(s) @ v).transpose(1, 2).reshape(B * S, H * 64)
        o.backward(dout.float())
    dqkv.copy_(qf.grad.to(BF))


def attention_bwd_kmask(qkv, out, dout, lse, dqkv, kmask, B, S, H, causal, scale):
    attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, scale, kmask)


def attention_probs(qkv, lse, kmask, probs, B, S, H, causal, scale):
    """exp(q.k * scale - lse) from the lse the forward wrote; 0 where the key is masked, causal-future or the row empty."""
    _, _, _, s = _attn(qkv, B, S, H, causal, scale, kmask)
    vis = s > float("-inf")
    probs.copy_(torch.where(vis, torch.exp(s - lse.view(B, H, S, 1)), torch.zeros_like(s)))


def vit_assemble_fwd(patch_out, cls, pos, mask_token, patch_mask, x, B, S, d):
    off = 1 if cls is not None else 0
    P = S - off
    e = patch_out.float().view(B, P, d)
    if patch_mask is not None and mask_token is not None:
        e = torch.where(patch_mask.view(B, P, 1).bool(), mask_token.detach().view(1, 1, d).expand(B, P, d), e)
    if cls is not None:
        e = torch.cat([cls.detach().view(1, 1, d).expand(B, 1, d), e], 1)
    x.view(B, S, d).copy_(e + pos.detach().view(1, S, d))


def vit_assemble_bwd(g, patch_mask, dpatch, dmask_token, B, S, d, has_cls=True):
    off = 1 if has_cls else 0
    P = S - off
    gp = g.view(B, S, d)[:, off:]
    if patch_mask is not None:
        m = patch_mask.view(B, P, 1).bool()
        if dmask_token is not None:
            dmask_token.view(-1).add_((gp * m).sum((0, 1)))
        gp = torch.where(m, torch.zeros_like(gp), gp)
    dpatch.copy_(gp.reshape(B * P, d).to(BF))


def bert_embed_ln_fwd(ids, type_ids, word, pos, type_emb, gamma, beta, x, kmask_out, pad_id, B, S, d, V, eps):
    tt = type_ids if type_ids is not None else torch.zeros_like(ids)
    e = word.detach()[ids] + pos.detach()[:S][None] + type_emb.detach()[tt]
    out, _, _ = _ln_rows(e, gamma, beta, eps)
    x.view(B, S, d).copy_(out)
    if kmask_out is not None:
        kmask_out.copy_((ids != pad_id).to(torch.uint8).view(-1))


def bert_embed_ln_bwd(ids, type_ids, word, pos, type_emb, gamma, dy, dword, dpos, dtype_emb, dgamma, dbeta, B, S, d, V, eps):
    tt = type_ids if type_ids is not None else torch.zeros_like(ids)
    w, p, t, g = (z.detach().clone().requires_grad_(True) for z in (word, pos, type_emb, gamma))
    b = torch.zeros(d, requires_grad=True)
    with torch.enable_grad():
        out = torch.nn.functional.layer_norm(w[ids] + p[:S][None] + t[tt], (d,), g, b, eps)
        out.backward(dy.view(B, S, d))
    for dst, src in ((dword, w), (dpos, p), (dtype_emb, t), (dgamma, g), (dbeta, b)):
        if dst is not None:
            dst.add_(src.grad)


def concat_tokens(cls, a, b, out, B, Sa, Sb, d):
    parts = []
    if cls is not None:
        parts.append(cls.detach().view(1, 1, d).expand(B, 1, d))
    # the kernel reads a and b as compact [B*Sa, d] / [B*Sb, d] rows (b is not read when Sb == 0)
    assert a.is_contiguous() and a.numel() == B * Sa * d, (tuple(a.shape), B, Sa, d)
    parts.append(a.detach().view(B, Sa, d))
    if Sb:
        assert b.is_contiguous() and b.numel() == B * Sb * d, (tuple(b.shape), B, Sb, d)
        parts.append(b.detach().view(B, Sb, d))
    out.view(B, -1, d).copy_(torch.cat(parts, 1))


def split_tokens_cast(g, a, b, B, Sa, Sb, d, has_cls=True):
    off = 1 if has_cls else 0
    gv = g.view(B, off + Sa + Sb, d)
    if a is not None and Sa:
        a.copy_(gv[:, off:off + Sa].reshape(-1, d).to(BF))
    if b is not None and Sb:
        b.copy_(gv[:, off + Sa:].reshape(-1, d).to(BF))


def gather_rows_cast(x, out, B, rows_per_group, row, d):
    out.copy_(x.detach().view(B, rows_per_group, d)[:, row].to(BF))


def tanh_(x):
    return x.tanh_()


def tanh_bwd(dy, y, dx=None, dx_bf16=None):
    v = dy * (1 - y * y)
    if dx is not None:
        dx.copy_(v)
    if dx_bf16 is not None:
        dx_bf16.copy_(v.to(BF))


def scatter_rows_add(src, dst, B, rows_per_group, row, d):
    dst.view(B, rows_per_group, d)[:, row] += src


def gather_rows_idx_cast(x, idx, out, d):
    ld = x.stride(-2)
    flat = x.detach().as_strided((int(idx.max().item()) + 1 if idx.numel() else 0, d), (ld, 1))
    out.copy_(flat[idx].to(BF))
    return out


def scatter_rows_idx_add(src, idx, dst, d):
    rows = int(idx.max().item()) + 1 if idx.numel() else 0
    torch.as_strided(dst, (rows, d), (dst.stride(-2), 1)).index_add_(0, idx, src)


def ce_labels(logits, labels, label_stride, ignore_index, M, V, row_loss, accum):
    lab = labels.view(-1)[::label_stride][:M]
    keep = lab != ignore_index
    lg = logits.detach()[:M, :V]
    nll = torch.logsumexp(lg, -1) - lg.gather(1, lab.clamp_min(0).view(-1, 1)).squeeze(1)
    nll = torch.where(keep, nll, torch.zeros_like(nll))
    if row_loss is not None:
        row_loss.copy_(nll)
    accum[0] += nll.sum()
    accum[1] += keep.sum()


def ce_labels_bwd(logits, labels, label_stride, ignore_index, M, V, accum, grad_scale, dlogits, gscale=None):
    lab = labels.view(-1)[::label_stride][:M]
    keep = lab != ignore_index
    p = torch.softmax(logits.detach()[:M, :V], -1)
    p[torch.arange(M)[keep], lab[keep]] -= 1
    w = grad_scale * (float(gscale[0]) if gscale is not None else 1.0) / (max(float(accum[1]), 1.0) if accum is not None else 1.0)
    dlogits.copy_((w * p * keep.view(-1, 1)).to(BF))


def act_bwd(dy, pre, dx, kind):
    dx.copy_((dy.float() * _act_grad(pre.float(), kind)).to(BF))


def cast_f32(src, out):
    out.copy_(src.float())
    return out


def act_fwd(x, kind):
    return _act(x.detach(), kind)


def sum_scale(inp, n, scale, out, accumulate=False):
    s = inp.detach().reshape(-1)[:n].sum() * scale
    out.view(-1)[:1].copy_((out.view(-1)[0] + s if accumulate else s).view(1))


def matmul_f32(A, B, *, ta=False, tb=False, out=None, alpha=1.0, accumulate=False):
    r = alpha * ((A.t() if ta else A) @ (B.t() if tb else B))
    if out is None:
        return r
    out.copy_(out + r if accumulate else r)
    return out


def _gen_scores(q, k, v, B, Sq, Skv, H, hd, bsq, scale, mask, causal):
    """Scores [B, H, Sq, Skv] (-inf where masked) and V [B, H, Skv, hd] of the general attention."""
    qh = (q.reshape(1, Sq, H, hd).expand(B, Sq, H, hd) if bsq == 0 else q.reshape(B, Sq, H, hd)).transpose(1, 2)
    kh, vh = k.reshape(B, Skv, H, hd).transpose(1, 2), v.reshape(B, Skv, H, hd).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) * scale
    if causal:
        s = s + torch.full((Sq, Skv), float("-inf")).triu(1)
    if mask is not None:
        mk = mask.bool()
        mk = mk.view(B, 1, Sq, Skv) if mk.numel() == B * Sq * Skv else mk.view(B, 1, 1, Skv)
        s = s.masked_fill(~mk, float("-inf"))
    return s, vh


def _gen_attn(q, k, v, B, Sq, Skv, H, hd, bsq, scale, mask, causal):
    s, vh = _gen_scores(q, k, v, B, Sq, Skv, H, hd, bsq, scale, mask, causal)
    return (_softmax_rows(s) @ vh).transpose(1, 2).reshape(B * Sq, H * hd)


def attention_fwd_generic(q, k, v, out, *, B, Sq, Skv, H, head_dim, bsq, bsk, bsv, bso, scale, mask=None, mask_bs=0,
                          mask_qs=0, causal=False):
    out.copy_(_gen_attn(q.float(), k.float(), v.float(), B, Sq, Skv, H, head_dim, bsq, scale, mask, causal).to(BF))


def attention_bwd_generic(q, k, v, dout, dk, dv, *, B, Sq, Skv, H, head_dim, bsq, bsk, bsv, bso, scale, dq=None,
                          dq_f32=None, mask=None, mask_bs=0, mask_qs=0, causal=False):
    qf, kf, vf = (t.float().clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        _gen_attn(qf, kf, vf, B, Sq, Skv, H, head_dim, bsq, scale, mask, causal).backward(dout.float())
    dk.copy_(kf.grad.to(BF))
    dv.copy_(vf.grad.to(BF))
    if dq is not None:
        dq.copy_(qf.grad.to(BF))
    if dq_f32 is not None:
        dq_f32[:, :H * head_dim] += qf.grad


def coca_text_embed_fwd(ids, emb, cls, pos, x, B, S, d, V):
    e = emb.detach()[ids]
    if cls is not None:
        e = torch.cat([e, cls.detach().reshape(1, 1, d).expand(B, 1, d)], 1)
    x.view(B, S, d).copy_(e + pos.detach().reshape(1, -1, d)[:, :S])


def l2norm_fwd(x, y, y_bf16, inv_norm, B, E, eps=1e-12):
    inv = 1.0 / x.detach().norm(dim=1).clamp_min(eps)
    y.copy_(x.detach() * inv[:, None])
    if y_bf16 is not None:
        y_bf16.copy_(y.to(BF))
    if inv_norm is not None:
        inv_norm.copy_(inv)


def l2norm_bwd(dy, y, inv_norm, dx, dx_bf16, B, E):
    r = inv_norm[:, None] * (dy - y * (y * dy).sum(1, keepdim=True))
    if dx is not None:
        dx.copy_(r)
    if dx_bf16 is not None:
        dx_bf16.copy_(r.to(BF))


def vit_embed_ln_fwd(patch_out, cls, pos, gamma, beta, x0, mean, rstd, B, S, d, eps):
    t = torch.cat([cls.detach().reshape(1, 1, d).expand(B, 1, d), patch_out.float().view(B, S - 1, d)], 1) + pos.detach().reshape(1, S, d)
    out, m, r = _ln_rows(t.reshape(B * S, d), gamma, beta, eps)
    x0.view(B * S, d).copy_(out)
    mean.copy_(m)
    rstd.copy_(r)


def vit_embed_ln_bwd(patch_out, cls, pos, dy_f32, mean, rstd, gamma, dt_f32, dpatch_bf16, dgamma, dbeta, B, S, d):
    t = (torch.cat([cls.detach().reshape(1, 1, d).expand(B, 1, d), patch_out.float().view(B, S - 1, d)], 1)
         + pos.detach().reshape(1, S, d)).reshape(B * S, d)
    dy = dy_f32.reshape(B * S, d).clone()
    h = (t - mean.view(-1, 1)) * rstd.view(-1, 1)
    dgamma.add_((dy * h).sum(0))
    dbeta.add_(dy.sum(0))
    dyg = dy * gamma.detach()
    dx = rstd.view(-1, 1) * (dyg - dyg.mean(-1, keepdim=True) - h * (dyg * h).mean(-1, keepdim=True))
    dt_f32.view(B * S, d).copy_(dx)
    dpatch_bf16.view(B, S - 1, d).copy_(dx.view(B, S, d)[:, 1:].to(BF))


def text_embed_fwd(tokens, emb, pos, x, B, S, d, V):
    x.view(B, S, d).copy_(emb.detach()[tokens] + pos.detach().reshape(1, S, d))


def text_embed_bwd(tokens, g, demb, B, S, d):
    demb.index_add_(0, tokens.reshape(-1), g.reshape(B * S, d))


def argmax_tokens(tokens, idx, B, S):
    idx.copy_(tokens.argmax(-1).to(torch.int32))


_LOG2E32 = torch.tensor(1.4426950408889634, dtype=F32)
_LN2_32 = torch.tensor(0.6931471805599453, dtype=F32)


def _temperature(log_scale):
    return torch.exp(log_scale.detach().reshape(-1)[:1].float())


def contrastive_ce_stats(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, row_loss, lse_out,
                         dscale_accum, logits_out=None, row_w=None):
    T = _temperature(logit_scale)
    l = T * sims[:rows, :N].float()
    ar = torch.arange(rows)
    lab = label_offset + ar
    mx = l.amax(1, keepdim=True)
    lse = mx.squeeze(1) + torch.log(torch.exp(l - mx).sum(1))
    xl = l[ar, lab]
    mean = l.sum(1) / N
    loss = (1 - smoothing) * (lse - xl) + smoothing * (lse - mean)
    wrow = row_w[:rows].float() if row_w is not None else torch.full((rows,), 1.0 / rows)
    if row_loss is not None:
        row_loss[:rows] = loss * wrow * rows if row_w is not None else loss
    if lse_out is not None:
        lse_out[:rows] = lse
    if logits_out is not None:
        logits_out[:rows, :N] = l
    if dscale_accum is not None:
        gl = torch.exp(l - lse[:, None]) - torch.tensor(smoothing, dtype=F32) / N
        gl[ar, lab] -= 1 - smoothing
        dscale_accum.view(-1)[:1] += ((gl * l).sum(1) * loss_weight * wrow).sum()


def contrastive_ce_grad(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, lse_row, lse_col, col_lo,
                        col_hi, dsims_bf16, dsims_f32, row_w=None, col_w=None):
    T = _temperature(logit_scale)
    l = T * sims[:rows, :N].float()
    ar = torch.arange(rows)
    t = torch.full((rows, N), smoothing / N, dtype=F32)
    t[ar, label_offset + ar] += 1 - smoothing
    gs = loss_weight * T * (row_w[:rows].float() if row_w is not None else torch.full((rows,), 1.0 / rows))
    g = gs[:, None] * (torch.exp(l - lse_row[:rows, None]) - t)
    lo, hi = max(col_lo, 0), min(col_hi, N)
    if lse_col is not None and hi > lo:
        j = slice(lo, hi)
        wc = loss_weight * T * (col_w[j].float() if col_w is not None else torch.full((hi - lo,), 1.0 / rows))
        add = wc * (torch.exp(l[:, j] - lse_col[j]) - t[:, j])
        g[:, j] += torch.where(wc != 0, add, torch.zeros_like(add))   # zero-weight rows may carry a non-finite LSE
    if dsims_bf16 is not None:
        dsims_bf16[:rows, :N] = g.to(BF)
    if dsims_f32 is not None:
        dsims_f32[:rows, :N] = g


def _merge_lanes(a, b):
    """One __shfl_xor level of the EPI_CE_STATS quad merge: (m2, se, sex, sx) of two lanes, m2 in log2 units."""
    (m, se, sex, sx), (mo, seo, sexo, sxo) = a, b
    mn = torch.maximum(m, mo)
    f = torch.where(m == float("-inf"), torch.zeros_like(m), torch.exp2(m - mn))
    fo = torch.where(mo == float("-inf"), torch.zeros_like(mo), torch.exp2(mo - mn))
    return mn, se * f + seo * fo, sex * f + sexo * fo, sx + sxo


def _ce_stats_epilogue(acc, T, lab, part, part0, xlabel):
    """EPI_CE_STATS over one launch's fp32 accumulators acc [M, N]: per 128-column part, lane tq of a quad reduces the
    32 columns c with (c % 8) // 2 == tq (max, then sum 2^(a T2 - m2), sum 2^(...) x, sum x with x = a T), the four
    lanes merge as lanes 0+1 and 2+3, then the two pairs; part p gets {m2 ln2, se, sex, sx}.  xlabel[r] = x[r, lab[r]]
    where lab[r] is a column of this launch."""
    M, N = acc.shape
    P = (N + 127) // 128
    T2 = T * _LOG2E32
    a = torch.zeros(M, P * 128)
    a[:, :N] = acc
    ok = torch.zeros(M, P * 128, dtype=torch.bool)
    ok[:, :N] = True
    a, ok = a.view(M, P, 16, 4, 2), ok.view(M, P, 16, 4, 2)     # column 128 p + 8 j + 2 tq + e
    x = a * T
    m2 = torch.where(ok, a, torch.full_like(a, float("-inf"))).amax((2, 4), keepdim=True) * T2
    pe = torch.where(ok, torch.exp2(a * T2 - torch.where(m2 == float("-inf"), torch.zeros_like(m2), m2)),
                     torch.zeros_like(a))
    zx = torch.where(ok, x, torch.zeros_like(x))
    lane = (m2[:, :, 0, :, 0], pe.sum((2, 4)), (pe * zx).sum((2, 4)), zx.sum((2, 4)))     # [M, P, 4 lanes] each
    q = [tuple(t[..., k] for t in lane) for k in range(4)]
    m, se, sex, sx = _merge_lanes(_merge_lanes(q[0], q[1]), _merge_lanes(q[2], q[3]))
    part[:M, part0:part0 + P] = torch.stack([m * _LN2_32, se, sex, sx], -1)
    r = torch.arange(M)
    hit = (lab >= 0) & (lab < N)
    xlabel[r[hit]] = (acc[r[hit], lab[hit]] * T)


def gemm_ce_stats(A, B, log_scale, label0, part, part0, xlabel):
    acc = A.float() @ B.float().t()
    _ce_stats_epilogue(acc, _temperature(log_scale), label0 + torch.arange(A.shape[0]), part, part0, xlabel)


def ce_stats_reduce(part, n_parts, xlabel, rows, n_total, smoothing, loss_weight, row_w, row_loss, lse_out,
                    dscale_accum):
    m, y, z, w = part[:rows, :n_parts].float().unbind(-1)
    ok = y > 0
    mx = torch.where(ok, m, torch.full_like(m, float("-inf"))).amax(1, keepdim=True)
    f = torch.where(ok, torch.exp(m - mx), torch.zeros_like(m))
    se = torch.where(ok, y * f, torch.zeros_like(y)).sum(1)
    sex = torch.where(ok, z * f, torch.zeros_like(z)).sum(1)
    lse = mx.squeeze(1) + torch.log(se)
    xl = xlabel[:rows].float()
    mean = w.sum(1) / n_total
    loss = (1 - smoothing) * (lse - xl) + smoothing * (lse - mean)
    wrow = row_w[:rows].float() if row_w is not None else torch.full((rows,), 1.0 / rows)
    if row_loss is not None:
        row_loss[:rows] = loss * wrow * rows if row_w is not None else loss
    if lse_out is not None:
        lse_out[:rows] = lse
    if dscale_accum is not None:
        dscale_accum.view(-1)[:1] += ((sex / se - (1 - smoothing) * xl - smoothing * mean) * loss_weight * wrow).sum()


def gemm_ce_grad(A, B, log_scale, label0, n_total, rows_total, smoothing, loss_weight, lse_row, row_w, lse_col, col_w,
                 col_lo, col_hi, dsims):
    from multimodal_b200._lib import MMBError

    M, N = A.shape[0], B.shape[0]
    if N % 8:
        raise MMBError("gemm_ce_grad: a bf16 output needs N % 8 == 0")
    assert tuple(dsims.shape) == (M, N) and dsims.dtype == BF
    acc = A.float() @ B.float().t()
    T = _temperature(log_scale)
    T2 = T * _LOG2E32
    r = torch.arange(M)
    t = (torch.tensor(smoothing, dtype=F32) / float(n_total)).expand(M, N).clone()
    lab = label0 + r
    hit = (lab >= 0) & (lab < N)
    t[r[hit], lab[hit]] += 1 - smoothing
    gs = torch.tensor(loss_weight, dtype=F32) / float(rows_total)
    gsT = T * (loss_weight * row_w[:M].float() if row_w is not None else gs.expand(M))
    g = gsT[:, None] * (torch.exp2(acc * T2 - (lse_row[:M] * _LOG2E32)[:, None]) - t)
    lo, hi = max(col_lo, 0), min(col_hi, N)
    if lse_col is not None and hi > lo:
        j = slice(lo, hi)
        wc = (loss_weight * T * col_w[j].float()) if col_w is not None else (T * gs).expand(hi - lo)
        add = wc * (torch.exp2(acc[:, j] * T2 - lse_col[j] * _LOG2E32) - t[:, j])
        g[:, j] += torch.where(wc != 0, add, torch.zeros_like(add))
    dsims.copy_(g.to(BF))


def linear_cross_entropy(hidden_bf16, weight_bf16, labels_i32, ignore_index, accum, row_loss=None):
    M, V = hidden_bf16.shape[0], weight_bf16.shape[0]
    P = (V + 127) // 128
    part = torch.zeros(M, P, 4)
    xlabel = torch.zeros(M)
    lab = labels_i32.reshape(-1).long()
    _ce_stats_epilogue(hidden_bf16.float() @ weight_bf16.float().t(), torch.ones(1), lab, part, 0, xlabel)
    m, y = part[..., 0], part[..., 1]
    mx = m.amax(1, keepdim=True)
    loss = mx.squeeze(1) + torch.log((y * torch.exp(m - mx)).sum(1)) - xlabel
    keep = lab != ignore_index
    loss = torch.where(keep, loss, torch.zeros_like(loss))
    if row_loss is not None:
        row_loss[:M] = loss
    accum.view(-1)[0] += loss.sum()
    accum.view(-1)[1] += keep.sum()


_real_wgrad_splits = None


def wgrad_splits(out_rows, out_cols, k, n_units=None):
    """No device to ask for its SM count: the split-K factor an H100 SXM (66 2-CTA clusters) would get.  The emulated
    GEMM's result does not depend on it."""
    return _real_wgrad_splits(out_rows, out_cols, k, 66 if n_units is None else n_units)


NAMES = [n for n, f in list(globals().items()) if callable(f) and not n.startswith("_") and n not in ("install",)]


def install(monkeypatch):
    """Swap the kernel wrappers of multimodal_b200.ops for the emulation and lift the CUDA-device guard."""
    from multimodal_b200 import engine, ops

    global _real_wgrad_splits
    _real_wgrad_splits = ops.wgrad_splits
    for n in NAMES:
        if hasattr(ops, n):
            monkeypatch.setattr(ops, n, globals()[n])
    monkeypatch.setattr(engine, "_require_cuda", lambda dev: None)
