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
    "attention_probs": "test_gpu_attention_long.py",
    "clip_image_transform": "test_gpu_clip_transform.py",
    "clip_image_transform_max_taps": "test_clip_transform_cpu.py",
    "gemm_ce_stats": "test_gpu_gemm_wide.py",
    "gemm_ce_grad": "test_gpu_gemm_wide.py",
    "linear_cross_entropy": "test_gpu_coca_train.py",
    "ce_stats_reduce": "test_gpu_parity.py",
    "contrastive_ce_stats": "test_gpu_parity.py",
    "contrastive_ce_grad": "test_gpu_parity.py",
    "adamw_step": "test_gpu_optim.py",
    "anyprecision_adamw_step": "test_gpu_optim.py",
    # pure host helpers
    "wgrad_splits": "test_abi_cpu.py",
    "gemm_ce_num_parts": "test_gpu_gemm_wide.py",
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


MUTANTS = {
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
