"""torch.autograd glue beside the module runtimes (whose autograd node is engine.RuntimeFunction): the L2 normalisation
of CLIP's embeddings and the autocast dtype convention at the module boundary."""
from __future__ import annotations

import torch

from . import ops
from ._lib import MMBError


class L2NormalizeFunction(torch.autograd.Function):
    """F.normalize(x) along dim=1 for 2-D inputs (models/clip/model.py:72-73)."""

    @staticmethod
    def forward(ctx, x, eps):
        if x.dim() != 2:
            raise MMBError("L2 normalise kernel expects a 2-D [batch, embedding] tensor")
        xf = x.contiguous().float()
        B, E = xf.shape
        y = torch.empty_like(xf)
        inv = torch.empty(B, device=x.device, dtype=torch.float32)
        ops.l2norm_fwd(xf, y, None, inv, B, E, eps)
        ctx.save_for_backward(y, inv)
        return y.to(x.dtype)

    @staticmethod
    def backward(ctx, dy):
        y, inv = ctx.saved_tensors
        B, E = y.shape
        dx = torch.empty_like(y)
        ops.l2norm_bwd(dy.contiguous().float(), y, inv, dx, None, B, E)
        return dx.to(dy.dtype), None


def l2_normalize(x: torch.Tensor, eps: float = 1e-12) -> torch.Tensor:
    return L2NormalizeFunction.apply(x, eps)


def autocast_out(t: torch.Tensor) -> torch.Tensor:
    """Dtype convention of the reference under ``torch.autocast`` (examples/flava/native/train.py:296-298): the towers'
    last op is a matmul / Linear, whose autocast output is the autocast dtype (bf16).  The kernels always produce fp32
    embeddings; inside an autocast region they are cast at the module boundary (differentiably), outside they stay fp32
    as the reference's fp32 modules return."""
    if t.is_cuda and torch.is_autocast_enabled():
        return t.to(torch.get_autocast_gpu_dtype())
    return t
