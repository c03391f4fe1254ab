"""TEST INFRASTRUCTURE ONLY: torch (CPU) emulation of the ReLU activation kind (ops.ACT_RELU, include/mmb200.h
`MMB_ACT_RELU`) in the kernel wrappers that take an activation: the GEMM's EPI_BF16_ACT / EPI_BF16_DACT epilogues and
ops.act_fwd / ops.act_bwd.  Layered over tests/emu_drop_path_ops.py (and so tests/emu_ops.py): any other kind is their
own call.  ReLU is exact: act(PRE) = max(PRE, 0) of the bf16 PRE, and the DACT / act_bwd output is the bf16-rounded
incoming gradient where PRE > 0 and +0 elsewhere (a select, not a product)."""
import torch

import emu_drop_path_ops
import emu_ops

BF, F32 = torch.bfloat16, torch.float32
ACT_RELU = 2


def relu_dgrad(g, pre):
    """g (fp32) where the bf16 pre-activation is > 0, +0 elsewhere."""
    return torch.where(pre.float() > 0, g, torch.zeros_like(g))


def gemm(A, B, *, a_mn=False, b_mn=False, epilogue=emu_ops.EPI_BF16, out=None, out2=None, bias=None, aux=None,
         alpha=1.0, act=0, splits=1, accumulate=False, colsum=None):
    if act != ACT_RELU or epilogue not in (emu_ops.EPI_BF16_ACT, emu_ops.EPI_BF16_DACT):
        return emu_ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=epilogue, out=out, out2=out2, bias=bias, aux=aux,
                            alpha=alpha, act=act, splits=splits, accumulate=accumulate, colsum=colsum)
    if epilogue == emu_ops.EPI_BF16_ACT:
        pre = emu_ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=emu_ops.EPI_BF16, out=out, bias=bias, alpha=alpha)
        if out2 is None:
            out2 = torch.empty_like(pre)
        out2.copy_(torch.clamp_min(pre, 0))
        return pre, out2
    assert aux is not None and aux.dtype == BF and bias is None
    acc = emu_ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, epilogue=emu_ops.EPI_F32, alpha=alpha)
    res = relu_dgrad(acc, aux).to(BF)
    if out is None:
        out = torch.empty_like(res)
    out.copy_(res)
    if colsum is not None:
        colsum.add_(res.float().sum(0))
    return out


def act_fwd(x, kind):
    return torch.clamp_min(x.detach(), 0) if kind == ACT_RELU else emu_ops.act_fwd(x, kind)


def act_bwd(dy, pre, dx, kind):
    if kind != ACT_RELU:
        return emu_ops.act_bwd(dy, pre, dx, kind)
    dx.copy_(relu_dgrad(dy.float(), pre).to(BF))


def install(monkeypatch):
    """emu_drop_path_ops.install, then the three wrappers above in place of their emu_ops versions."""
    from multimodal_b200 import ops

    emu_drop_path_ops.install(monkeypatch)
    for n in ("gemm", "act_fwd", "act_bwd"):
        monkeypatch.setattr(ops, n, globals()[n])
