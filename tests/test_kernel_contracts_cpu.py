"""The kernel contracts of tests/kernel_contract_cases.py on the CPU: the emulation the schedule tests install
(tests/emu_ops.py, tests/emu_decode_ops.py) against the float64 references at CPU-sized cases, a guard that every
kernel has a contract check, deliberately broken emulations that the checks must reject, and the zero-size calls of the
column / batch sums, which return before any CUDA call."""
import ctypes
import inspect
import types

import pytest
import torch

import emu_ops
import kernel_contract_cases as KC

_CPU_CASES = [(op, c) for op, cases in KC.CASES.items() for c in cases if not c.get("gpu")]


@pytest.mark.parametrize("op,case", _CPU_CASES, ids=[f"{op}[{KC.case_id(c)}]" for op, c in _CPU_CASES])
def test_emulation_meets_float64_contract(op, case):
    KC.CHECKS[op](KC.emulation(), "cpu", case)


# ---- coverage guard ----------------------------------------------------------------------------------------------------
# Public wrappers of multimodal_b200.ops without an entry in CASES, each with the test file that covers it.
ALLOWLIST = {
    "self_attention": "test_attention_router_cpu.py",
    "clip_image_transform": "test_gpu_clip_transform.py",
    "clip_image_transform_max_taps": "test_clip_transform_cpu.py",
    "adamw_step": "test_gpu_optim.py",
    "anyprecision_adamw_step": "test_gpu_optim.py",
    # pure host helpers
    "wgrad_splits": "test_abi_cpu.py",
    "gemm_ce_num_parts": "test_kernel_contracts_cpu.py",   # asserted by check_gemm_ce_stats
    "attention_decode_splits": "test_gpu_decoder_cache.py",
    "decode_attention_wins": "test_decoder_cache_cpu.py",
}


def test_every_emulated_kernel_has_a_contract_check():
    import emu_decode_ops

    emulated = set(emu_ops.NAMES) | {"attention_fwd_decode", "kv_cache_append"}
    assert {n for n in vars(emu_decode_ops) if n in ("attention_fwd_decode", "kv_cache_append")} == \
        {"attention_fwd_decode", "kv_cache_append"}
    missing = sorted(n for n in emulated if n not in KC.CASES and n not in ALLOWLIST)
    assert not missing, f"emulated kernels without a contract check: {missing}"


def test_every_ops_wrapper_has_a_contract_check_or_a_named_test():
    import os

    from multimodal_b200 import ops

    public = {n for n, f in vars(ops).items()
              if inspect.isfunction(f) and f.__module__ == ops.__name__ and not n.startswith("_")}
    missing = sorted(public - set(KC.CASES) - set(ALLOWLIST))
    assert not missing, f"ops wrappers with neither a contract check nor an allowlist entry: {missing}"
    assert not set(ALLOWLIST) & set(KC.CASES)
    assert set(ALLOWLIST) <= public, sorted(set(ALLOWLIST) - public)
    here = os.path.dirname(os.path.abspath(__file__))
    for name, f in ALLOWLIST.items():
        assert os.path.isfile(os.path.join(here, f)), f"{name}: {f} does not exist"
    for op in KC.CASES:
        assert hasattr(ops, op), op


# ---- mutation check: broken emulations must fail their contract --------------------------------------------------------
def _truncating_cast_bf16(src, out=None):
    b = src.contiguous().view(torch.int32) & -65536          # round toward zero
    out.copy_(torch.where(torch.isnan(src), src, b.view(torch.float32)).to(torch.bfloat16))
    return out


def _ln_bwd_skips_last_row(x, dy_bf16, dy_f32, mean, rstd, gamma, g_in, g_out, g_bf16, dgamma, dbeta, M, d, row_idx=None,
                           rows_per_group=0, gsum=None):
    emu_ops.layernorm_bwd(x, dy_bf16, dy_f32, mean[:M - 1], rstd[:M - 1], gamma, g_in, g_out, g_bf16, dgamma, dbeta,
                          M - 1, d, row_idx=None if row_idx is None else row_idx[:M - 1], rows_per_group=rows_per_group,
                          gsum=gsum)


def _ln_fwd_ignores_rows_per_group(*args, row_idx=None, rows_per_group=0):
    emu_ops.add_layernorm_fwd(*args)


def _colsum_assigns(x, out, M, N, ld):
    out.view(-1)[:N].zero_()
    emu_ops.colsum_bf16(x, out, M, N, ld)


def _act_fwd_quick_for_gelu(x, kind):
    return emu_ops.act_fwd(x, 0)


def _ce_counts_all_rows(logits, labels, label_stride, ignore_index, M, V, row_loss, accum):
    emu_ops.ce_labels(logits, labels, label_stride, ignore_index, M, V, row_loss, accum)
    lab = labels.view(-1)[::label_stride][:M]
    accum[1] += (lab == ignore_index).sum()


def _text_embed_bwd_last_duplicate(tokens, g, demb, B, S, d):
    flat, rows = tokens.reshape(-1), g.reshape(B * S, d)
    last = {}
    for r, t in enumerate(flat.tolist()):
        last[t] = r
    for t, r in last.items():
        demb[t] += rows[r]


def _colsum_drops_partial_block(x, out, M, N, ld):
    full = N // 256 * 256
    out.view(-1)[:full].add_(x.reshape(-1, ld)[:M, :full].float().sum(0))


def _l2norm_truncating_bf16(x, y, y_bf16, inv_norm, B, E, eps=1e-12):
    emu_ops.l2norm_fwd(x, y, None, inv_norm, B, E, eps)
    _truncating_cast_bf16(y, y_bf16)


def _batch_sum_skips_last(inp, out, Bn, ld, n):
    emu_ops.batch_sum(inp, out, Bn - 1, ld, n)


def _online_attn_fwd(qkv, out, lse, B, S, H, causal, scale, kmask=None, *, rescale=True, drop_block=None, diag=0,
                     kmask_last_block=True):
    """The kernels' online softmax over 64-key blocks (running max m, sum l, O in fp32, P rounded to bf16 for PV), with
    the defects the mutants below switch on."""
    inf = float("inf")
    km = kmask
    if km is not None and not kmask_last_block:
        km = km.clone().view(B, S)
        km[:, (S - 1) // 64 * 64:] = 1
    _, _, v, s = emu_ops._attn(qkv, B, S, H, False, scale, km)
    if causal:
        s = s + torch.full((S, S), -inf).triu(1 + diag)
    m = torch.full((B, H, S, 1), -inf)
    l = torch.zeros(B, H, S, 1)
    o = torch.zeros(B, H, S, 64)
    for j0 in range(0, S, 64):
        sb = s[..., j0:j0 + 64].clone()
        if drop_block is not None and j0 == 64 * drop_block:
            sb[:, :, 128:] = -inf
        mn = torch.maximum(m, sb.amax(-1, keepdim=True))
        base = torch.where(mn == -inf, torch.zeros_like(mn), mn)
        c = torch.exp(m - base)
        e = torch.exp(sb - base)
        l = l * c + e.sum(-1, keepdim=True)
        o = (o * c if rescale else o) + e.to(torch.bfloat16).float() @ v[..., j0:j0 + 64, :]
        m = mn
    out.copy_((o / torch.where(l > 0, l, torch.ones_like(l))).transpose(1, 2).reshape(B * S, H * 64).to(torch.bfloat16))
    lse.copy_(torch.where(l > 0, m + torch.log(l), torch.full_like(l, -inf)).reshape(-1))


def _fwd_no_rescale(qkv, out, lse, B, S, H, causal, scale):
    _online_attn_fwd(qkv, out, lse, B, S, H, causal, scale, rescale=False)


def _fwd_drops_block_past_first_tile(qkv, out, lse, B, S, H, causal, scale):
    _online_attn_fwd(qkv, out, lse, B, S, H, causal, scale, drop_block=1)


def _fwd_causal_off_by_one(qkv, out, lse, B, S, H, causal, scale):
    _online_attn_fwd(qkv, out, lse, B, S, H, causal, scale, diag=1)


def _fwd_kmask_ignored_in_last_block(qkv, out, lse, kmask, B, S, H, causal, scale):
    _online_attn_fwd(qkv, out, lse, B, S, H, causal, scale, kmask, kmask_last_block=False)


def _bwd_dkdv_skip_last_partial_tile(qkv, out, dout, lse, dqkv, B, S, H, causal, scale):
    emu_ops.attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, scale)
    if S % 128:   # dK / dV without the query rows of the last, partial 128-row tile (their dO and dS set to zero)
        d = dout.clone().view(B, S, -1)
        d[:, S // 128 * 128:] = 0
        part = torch.empty_like(dqkv)
        emu_ops.attention_bwd(qkv, out, d.view(B * S, -1), lse, part, B, S, H, causal, scale)
        dqkv[:, H * 64:] = part[:, H * 64:]


def _dq_f32_assigned(*args, dq_f32=None, **kw):
    if dq_f32 is not None:
        dq_f32.zero_()
    emu_ops.attention_bwd_generic(*args, dq_f32=dq_f32, **kw)


def _decode_combine_unscaled(q, k, v, out, *, B, Sq, Skv, H, head_dim, bsq, bsk, bsv, bso, scale, mask=None, mask_bs=0,
                             mask_qs=0, causal=False):
    """The decode kernel's schedule: each key split keeps its own running max m_s, sum l_s and unnormalised O_s; the
    combine adds them without rescaling each to the common max, O = sum O_s / sum l_s."""
    from multimodal_b200 import _lib

    full = None if mask is None else torch.as_strided(mask, (B, Sq, Skv), (mask_bs, mask_qs, 1)).contiguous()
    s, vh = emu_ops._gen_scores(q.float(), k.float(), v.float(), B, Sq, Skv, H, head_dim, bsq, scale, full, causal)
    n = _lib.lib().mmb_attention_decode_splits(B, H, Skv)
    per = -(-(-(-Skv // 64)) // n) * 64
    o = torch.zeros(B, H, Sq, head_dim)
    l = torch.zeros(B, H, Sq, 1)
    for j0 in range(0, Skv, per):
        sb = s[..., j0:j0 + per]
        m = sb.amax(-1, keepdim=True)
        e = torch.exp(sb - torch.where(m == float("-inf"), torch.zeros_like(m), m))
        o = o + e.to(torch.bfloat16).float() @ vh[..., j0:j0 + per, :]
        l = l + e.sum(-1, keepdim=True)
    r = o / torch.where(l > 0, l, torch.ones_like(l))
    out.copy_(r.transpose(1, 2).reshape(B * Sq, H * head_dim).to(torch.bfloat16))


def _probs_next_row_lse(qkv, lse, kmask, probs, B, S, H, causal, scale):
    l = lse.view(B, H, S)
    emu_ops.attention_probs(qkv, torch.cat([l[..., 1:], l[..., -1:]], -1).reshape(-1), kmask, probs, B, S, H, causal,
                            scale)


def _reduce_without_rescale(part, n_parts, xlabel, rows, n_total, smoothing, loss_weight, row_w, row_loss, lse_out,
                            dscale_accum):
    """ce_stats_reduce adding every part's sums as they are, without rescaling them to the row's common maximum."""
    q = part.clone()
    mx = q[:rows, :n_parts, 0].amax(1, keepdim=True)
    q[:rows, :n_parts, 0] = mx
    emu_ops.ce_stats_reduce(q, n_parts, xlabel, rows, n_total, smoothing, loss_weight, row_w, row_loss, lse_out,
                            dscale_accum)


def _grad_smoothing_over_launch_n(A, B, log_scale, label0, n_total, *rest):
    emu_ops.gemm_ce_grad(A, B, log_scale, label0, B.shape[0], *rest)


def _grad_transposed_range_inclusive(A, B, log_scale, label0, n_total, rows_total, smoothing, loss_weight, lse_row,
                                     row_w, lse_col, col_w, col_lo, col_hi, dsims):
    emu_ops.gemm_ce_grad(A, B, log_scale, label0, n_total, rows_total, smoothing, loss_weight, lse_row, row_w, lse_col,
                         col_w, col_lo, col_hi + 1, dsims)


def _grad_transposed_row_weights(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, lse_row, lse_col,
                                 col_lo, col_hi, dsims_bf16, dsims_f32, row_w=None, col_w=None):
    """contrastive_ce_grad weighting the transposed term of element (i, j) with row i's weight instead of column j's."""
    g = torch.zeros(rows, N)
    emu_ops.contrastive_ce_grad(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, lse_row, None, 0, 0,
                                None, g, row_w, None)
    if lse_col is not None and col_hi > col_lo and row_w is not None:
        T = torch.exp(logit_scale.reshape(-1)[:1])
        j = slice(col_lo, col_hi)
        t = torch.full((rows, N), smoothing / N)
        t[torch.arange(rows), label_offset + torch.arange(rows)] += 1 - smoothing
        wc = (loss_weight * T * row_w[:rows])[:, None]
        add = wc * (torch.exp(T * sims[:rows, j] - lse_col[j]) - t[:, j])
        g[:, j] += torch.where(wc != 0, add, torch.zeros_like(add))
    elif lse_col is not None:
        emu_ops.contrastive_ce_grad(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, lse_row, lse_col,
                                    col_lo, col_hi, None, g, row_w, col_w)
    if dsims_bf16 is not None:
        dsims_bf16[:rows, :N] = g.to(torch.bfloat16)
    if dsims_f32 is not None:
        dsims_f32[:rows, :N] = g


def _stats_xlabel_at_row(A, B, log_scale, label0, part, part0, xlabel):
    """gemm_ce_stats taking row r's label at this launch's column r instead of label0 + r."""
    x = xlabel.clone()
    emu_ops.gemm_ce_stats(A, B, log_scale, label0, part, part0, x)
    emu_ops.gemm_ce_stats(A, B, log_scale, 0, part.clone(), part0, xlabel)


def _stats_drops_second_half(A, B, log_scale, label0, part, part0, xlabel):
    """gemm_ce_stats leaving the second 128-column part of a partial last tile unwritten."""
    N = B.shape[0]
    keep = part.clone()
    emu_ops.gemm_ce_stats(A, B, log_scale, label0, part, part0, xlabel)
    if N % 256 > 128:
        p = part0 + 2 * (N // 256) + 1
        part[:, p] = keep[:, p]


def _stats_dscale_unweighted(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, row_loss, lse_out,
                             dscale_accum, logits_out=None, row_w=None):
    """contrastive_ce_stats weighting every row's d loss / d log_scale share by 1 / rows whatever row_w says."""
    emu_ops.contrastive_ce_stats(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, row_loss, lse_out,
                                 None, logits_out, row_w)
    emu_ops.contrastive_ce_stats(sims, logit_scale, rows, N, label_offset, smoothing, loss_weight, None, None,
                                 dscale_accum, None, None)


def _linear_ce_counts_ignored(hidden, weight, labels, ignore_index, accum, row_loss=None):
    emu_ops.linear_cross_entropy(hidden, weight, labels, ignore_index, accum, row_loss)
    accum[1] += (labels == ignore_index).sum()


def _gemm_k(A, kw):
    return A.shape[0] if kw.get("a_mn") else A.shape[1]


def _gemm_bias_every_split(A, B, **kw):
    out = emu_ops.gemm(A, B, **kw)
    if kw["epilogue"] == emu_ops.EPI_F32 and kw.get("bias") is not None:
        out += (KC._gemm_splits(_gemm_k(A, kw), kw.get("splits", 1), "f32") - 1) * kw["bias"]
    return out


def _gemm_act_of_fp32_pre(A, B, **kw):
    res = emu_ops.gemm(A, B, **kw)
    if kw["epilogue"] == emu_ops.EPI_BF16_ACT:
        pre = emu_ops.gemm(A, B, **dict(kw, epilogue=emu_ops.EPI_F32, out=None, out2=None))
        res[1].copy_(emu_ops._act(pre, kw.get("act", 0)).to(torch.bfloat16))
    return res


def _gemm_colsum_unrounded(A, B, *, colsum=None, **kw):
    res = emu_ops.gemm(A, B, **kw)
    if colsum is not None:
        pre = emu_ops.gemm(A, B, **dict(kw, epilogue=emu_ops.EPI_F32, out=None, aux=None))
        if kw["epilogue"] == emu_ops.EPI_BF16_DACT:
            pre = pre * emu_ops._act_grad(kw["aux"].float(), kw.get("act", 0))
        colsum.add_(pre.sum(0))
    return res


def _gemm_colsum_assigns(A, B, *, colsum=None, **kw):
    if colsum is not None:
        colsum.zero_()
    return emu_ops.gemm(A, B, colsum=colsum, **kw)


def _gemm_drops_partial_k_block(A, B, **kw):
    k0 = _gemm_k(A, kw) // 64 * 64
    A = A[:k0] if kw.get("a_mn") else A[:, :k0]
    B = B[:k0] if kw.get("b_mn") else B[:, :k0]
    return emu_ops.gemm(A, B, **kw)


def _gemm_dact_ignores_alpha(A, B, **kw):
    if kw["epilogue"] == emu_ops.EPI_BF16_DACT:
        kw["alpha"] = 1.0
    return emu_ops.gemm(A, B, **kw)


def _gemm_splitk_ignores_accumulate(A, B, **kw):
    if kw["epilogue"] == emu_ops.EPI_F32 and KC._gemm_splits(_gemm_k(A, kw), kw.get("splits", 1), "f32") > 1:
        kw["accumulate"] = False
    return emu_ops.gemm(A, B, **kw)


def _gemm_writes_row_padding(A, B, *, out=None, **kw):
    res = emu_ops.gemm(A, B, out=out, **kw)
    if out is not None and out.stride(0) > out.shape[1]:
        rows = torch.as_strided(out, (out.shape[0], out.stride(0)), out.stride(), out.storage_offset())
        rows[:, out.shape[1]:] = 0
    return res


MUTANTS = {
    "gemm adds the bias in every split": ("gemm", "gemm", _gemm_bias_every_split),
    "gemm applies the activation to the fp32 pre-activation": ("gemm", "gemm", _gemm_act_of_fp32_pre),
    "gemm column sums over the unrounded output": ("gemm", "gemm", _gemm_colsum_unrounded),
    "gemm column sums assigned instead of accumulated": ("gemm", "gemm", _gemm_colsum_assigns),
    "gemm drops the last partial k-block": ("gemm", "gemm", _gemm_drops_partial_k_block),
    "gemm act' epilogue ignores alpha": ("gemm", "gemm", _gemm_dact_ignores_alpha),
    "split-K gemm ignores accumulate": ("gemm", "gemm", _gemm_splitk_ignores_accumulate),
    "gemm writes the padding columns between N and ld": ("gemm", "gemm", _gemm_writes_row_padding),
    "cast truncates instead of rounding": ("cast_bf16", "cast_bf16", _truncating_cast_bf16),
    "LayerNorm backward skips the last row": ("layernorm_bwd", "layernorm_bwd", _ln_bwd_skips_last_row),
    "rows_per_group ignored": ("add_layernorm_fwd", "add_layernorm_fwd", _ln_fwd_ignores_rows_per_group),
    "+= replaced by =": ("colsum_bf16", "colsum_bf16", _colsum_assigns),
    "GELU swapped for QuickGELU": ("act_fwd", "act_fwd", _act_fwd_quick_for_gelu),
    "ignored-row count taken from all rows": ("ce_labels", "ce_labels", _ce_counts_all_rows),
    "text_embed_bwd keeps only the last duplicate": ("text_embed_bwd", "text_embed_bwd", _text_embed_bwd_last_duplicate),
    "colsum drops the last partial 256-column block": ("colsum_bf16", "colsum_bf16", _colsum_drops_partial_block),
    "bf16 output of fp32 math rounds toward zero": ("l2norm_fwd", "l2norm_fwd", _l2norm_truncating_bf16),
    "batch_sum drops the last batch row": ("batch_sum", "batch_sum", _batch_sum_skips_last),
    "online softmax does not rescale O when the running max moves": ("attention_fwd", "attention_fwd", _fwd_no_rescale),
    "one 64-key block dropped for query rows past the first 128-row tile":
        ("attention_fwd", "attention_fwd", _fwd_drops_block_past_first_tile),
    "causal diagonal off by one": ("attention_fwd", "attention_fwd", _fwd_causal_off_by_one),
    "key mask ignored in the last partial key block":
        ("attention_fwd_kmask", "attention_fwd_kmask", _fwd_kmask_ignored_in_last_block),
    "dK / dV skip the query rows of the last partial 128-row tile":
        ("attention_bwd", "attention_bwd", _bwd_dkdv_skip_last_partial_tile),
    "dq_f32 assigned instead of accumulated": ("attention_bwd_generic", "attention_bwd_generic", _dq_f32_assigned),
    "decode splits combined without rescaling to the common max":
        ("attention_fwd_decode", "attention_fwd_decode", _decode_combine_unscaled),
    "attention_probs uses the lse of the next row": ("attention_probs", "attention_probs", _probs_next_row_lse),
    "ce_stats_reduce sums the parts without rescaling them to the common max":
        ("ce_stats_reduce", "ce_stats_reduce", _reduce_without_rescale),
    "smoothing term divided by the launch's N instead of n_total":
        ("gemm_ce_grad", "gemm_ce_grad", _grad_smoothing_over_launch_n),
    "transposed term applied on [col_lo, col_hi]": ("gemm_ce_grad", "gemm_ce_grad", _grad_transposed_range_inclusive),
    "transposed term weighted by row_w instead of col_w":
        ("contrastive_ce_grad", "contrastive_ce_grad", _grad_transposed_row_weights),
    "gemm_ce_stats writes xlabel at column r instead of label0 + r":
        ("gemm_ce_stats", "gemm_ce_stats", _stats_xlabel_at_row),
    "gemm_ce_stats drops the second 128-column part of a partial tile":
        ("gemm_ce_stats", "gemm_ce_stats", _stats_drops_second_half),
    "contrastive_ce_stats ignores row_w in dscale": ("contrastive_ce_stats", "contrastive_ce_stats", _stats_dscale_unweighted),
    "linear_cross_entropy counts ignored rows": ("linear_cross_entropy", "linear_cross_entropy", _linear_ce_counts_ignored),
}


@pytest.mark.parametrize("what", list(MUTANTS))
def test_broken_emulation_fails_its_contract(what):
    op, name, broken = MUTANTS[what]
    impl = types.SimpleNamespace(**vars(KC.emulation()))
    setattr(impl, name, broken)
    cases = [c for c in KC.CASES[op] if not c.get("gpu")]
    caught = 0
    for case in cases:
        try:
            KC.CHECKS[op](impl, "cpu", case)
        except AssertionError:
            caught += 1
    assert caught > 0, f"no CPU case of {op} rejects the mutant '{what}'"


def test_online_softmax_restatement_meets_the_contract():
    """The blockwise restatement the attention mutants are built on passes every CPU case when no defect is on, so
    each mutant fails for its defect alone."""
    impl = types.SimpleNamespace(**vars(KC.emulation()))
    impl.attention_fwd = lambda *a: _online_attn_fwd(*a)
    impl.attention_fwd_kmask = lambda qkv, out, lse, kmask, *a: _online_attn_fwd(qkv, out, lse, *a, kmask)
    for op in ("attention_fwd", "attention_fwd_kmask"):
        for case in KC.CASES[op]:
            if not case.get("gpu"):
                KC.CHECKS[op](impl, "cpu", case)


def test_attention_cases_sit_where_they_say():
    """The general cases lie on the side of the resident / streamed switch the case list names, and every decode
    case runs the number of key splits it was built for."""
    from multimodal_b200 import _lib

    lib = _lib.lib()
    for c in KC.CASES["attention_fwd_generic"]:
        assert lib.mmb_attention_generic_streamed(c["Sq"], c["Skv"], c["hd"]) == KC._STREAMED[(c["Sq"], c["Skv"], c["hd"])], c
    assert set(KC._STREAMED.values()) == {0, 1}
    for c in KC.CASES["attention_fwd_decode"]:
        assert lib.mmb_attention_decode_splits(c["B"], c["H"], c["Skv"]) == c.get("splits", 1), c


def test_gemm_cases_sit_where_they_say():
    """The persistent-loop GEMM cases give every CTA (2-CTA cluster) of a 132-SM H100 at least 3 tiles, and some CTA
    a partial-N tile right after a full one (tile t runs on unit t mod units, n_blk = t mod n_tiles within a split);
    together they cover every instantiation in both variants."""
    seen = set()
    for c in KC.CASES["gemm"]:
        if not c.get("persist"):
            continue
        clu = c["gemm_mode"] == 1
        units = KC.H100_SMS // 2 if clu else KC.H100_SMS
        m_tiles, n_tiles = KC._cdiv(c["M"], 256 if clu else 128), KC._cdiv(c["N"], 256)
        tiles = m_tiles * n_tiles * KC._gemm_splits(c["K"], c.get("splits", 1), c["epi"])
        assert tiles // units >= 3, c
        assert c["N"] % 256 and n_tiles > 1, c
        n_blk = lambda t: t % (m_tiles * n_tiles) % n_tiles  # noqa: E731
        assert any(n_blk(t) < n_tiles - 1 and n_blk(t + units) == n_tiles - 1 for t in range(tiles - units)), c
        seen.add((KC._gemm_kind_key(c), c["gemm_mode"]))
    assert seen == {(KC._gemm_kind_key(k), m) for k in KC.GEMM_KINDS for m in (0, 1)}


def test_gemm_cases_cover_every_instantiation_on_the_cpu():
    """The CPU cases reach every instantiation, so each emulation mutant meets the epilogue it breaks."""
    cpu = {KC._gemm_kind_key(c) for c in KC.CASES["gemm"] if not c.get("gpu")}
    assert cpu == {KC._gemm_kind_key(k) for k in KC.GEMM_KINDS}


@pytest.mark.parametrize("epilogue,accumulate,bias", [(0, 1, False), (1, 1, False), (2, 1, False), (2, 0, True)],
                         ids=["bf16_accumulate", "act_accumulate", "dact_accumulate", "dact_bias"])
def test_gemm_refuses_accumulate_and_bias_its_epilogue_would_ignore(epilogue, accumulate, bias):
    """mmb_gemm_bf16 returns MMB_ERR_ARG before touching any pointer: only EPI_F32 adds into D0, and
    EPI_BF16_DACT has no bias term (D0 = bf16(alpha acc act'(aux)))."""
    from multimodal_b200 import _lib

    null = ctypes.c_void_p(0)
    host = (ctypes.c_float * 64)()        # a real address that the refused call never reads
    b = ctypes.cast(host, ctypes.c_void_p) if bias else null
    rc = _lib.lib().mmb_gemm_bf16(null, 8, 0, null, 8, int(epilogue == 2), null, 8, null, 8, 8, 8, 8, epilogue, 0,
                                  ctypes.c_float(1.0), b, null, 8, 1, accumulate, null, null)
    assert rc == -22, rc     # MMB_ERR_ARG


# ---- zero-size calls ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn,args", [
    ("mmb_colsum_bf16", (0, 8, 8)),       # M = 0
    ("mmb_colsum_bf16", (5, 0, 8)),       # N = 0
    ("mmb_colsum_bf16", (0, 0, 0)),
    ("mmb_batch_sum", (0, 8, 8)),         # Bn = 0
    ("mmb_batch_sum", (3, 8, 0)),         # n = 0
    ("mmb_batch_sum", (0, 0, 0)),
])
def test_zero_size_sums_return_ok_without_touching_memory(fn, args):
    from multimodal_b200 import _lib

    null = ctypes.c_void_p(0)
    f = getattr(_lib.lib(), fn)
    if fn == "mmb_colsum_bf16":
        M, N, ld = args
        rc = f(null, null, M, N, ld, null)
    else:
        Bn, ld, n = args
        rc = f(null, null, Bn, ld, n, null)
    assert rc == 0, rc
