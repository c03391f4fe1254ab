"""TEST INFRASTRUCTURE ONLY: torch (CPU) emulation of the stochastic-depth variants of three kernel wrappers
(`branch_scale` / `rows_per_scale` of ops.add_layernorm_fwd, ops.layernorm_bwd and ops.cast_bf16, include/mmb200.h
`mmb_*_scaled`), layered over tests/emu_ops.py: without a branch_scale each call is emu_ops' own.  The emulation keeps
the kernels' roundings: the product s * y (s * g) is rounded to fp32 on its own, the gradient entering a branch is
rounded to bf16 after the product, and gsum sums those bf16 values."""
import torch

import emu_ops

BF, F32 = torch.bfloat16, torch.float32


def _rows(branch_scale, M, rows_per_scale):
    assert branch_scale.dtype == F32 and rows_per_scale > 0 and branch_scale.numel() * rows_per_scale == M
    return branch_scale.detach().repeat_interleave(rows_per_scale).view(M, 1)


def add_layernorm_fwd(x_in, y, x_out, ln_bf16, ln_f32, gamma, beta, mean, rstd, M, d, eps, row_idx=None,
                      rows_per_group=0, branch_scale=None, rows_per_scale=0):
    if branch_scale is not None:
        assert rows_per_group == 0 and y is not None
        y = _rows(branch_scale, M, rows_per_scale) * y.reshape(M, d).float()     # fp32 products, added by emu_ops
    emu_ops.add_layernorm_fwd(x_in, y, x_out, ln_bf16, ln_f32, gamma, beta, mean, rstd, M, d, eps, row_idx,
                              rows_per_group)


def layernorm_bwd(x, dy_bf16, dy_f32, mean, rstd, gamma, g_in, g_out, g_bf16, dgamma, dbeta, M, d, row_idx=None,
                  rows_per_group=0, gsum=None, branch_scale=None, rows_per_scale=0):
    if branch_scale is None:
        emu_ops.layernorm_bwd(x, dy_bf16, dy_f32, mean, rstd, gamma, g_in, g_out, g_bf16, dgamma, dbeta, M, d, row_idx,
                              rows_per_group, gsum)
        return
    assert rows_per_group == 0 and g_bf16 is not None
    go = g_out if g_out is not None else torch.empty(M, d)
    emu_ops.layernorm_bwd(x, dy_bf16, dy_f32, mean, rstd, gamma, g_in, go, None, dgamma, dbeta, M, d)
    gb = (_rows(branch_scale, M, rows_per_scale) * go.reshape(M, d)).to(BF)
    g_bf16.view(-1, d)[:M] = gb
    if gsum is not None:
        gsum.add_(gb.float().sum(0))


def cast_bf16(src, out=None, branch_scale=None, rows_per_scale=0):
    if branch_scale is not None:
        assert src.dim() == 2
        src = _rows(branch_scale, src.shape[0], rows_per_scale) * src.detach()
    return emu_ops.cast_bf16(src, out)


def install(monkeypatch):
    """emu_ops.install, then the three wrappers above in place of their emu_ops versions."""
    from multimodal_b200 import ops

    emu_ops.install(monkeypatch)
    for n in ("add_layernorm_fwd", "layernorm_bwd", "cast_bf16"):
        monkeypatch.setattr(ops, n, globals()[n])
