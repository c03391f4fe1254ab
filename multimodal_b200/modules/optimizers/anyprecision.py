"""Drop-in for torchmultimodal.modules.optimizers.anyprecision.AnyPrecisionAdamW (anyprecision.py:16-199): same
constructor, same per-parameter state keys (`step`, `exp_avg`, `exp_avg_sq`, `compensation`) and dtypes, same update
rule.  The step of every parameter is ONE fused sm_90a kernel (mmb_anyprecision_adamw_step) instead of the
reference's ~12 elementwise passes; roundings to the state dtypes are reproduced one for one.

Parameters and gradients must be fp32 CUDA tensors (this runtime keeps fp32 master weights; bf16 operand copies are
internal), states may be fp32 or bf16.  No CPU path.
"""
from __future__ import annotations

from typing import Any, Dict, Iterable, Tuple, Union

import torch
from torch.optim.optimizer import Optimizer

from ... import ops
from ..._lib import MMBError

_OK = (torch.float32, torch.bfloat16)


class AnyPrecisionAdamW(Optimizer):
    def __init__(self, params: Union[Iterable[torch.Tensor], Iterable[Dict[str, Any]]], lr: float = 1e-3,
                 betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 use_kahan_summation: bool = False, momentum_dtype: torch.dtype = torch.float32,
                 variance_dtype: torch.dtype = torch.bfloat16,
                 compensation_buffer_dtype: torch.dtype = torch.bfloat16) -> None:
        for name, dt in (("momentum_dtype", momentum_dtype), ("variance_dtype", variance_dtype),
                         ("compensation_buffer_dtype", compensation_buffer_dtype)):
            if dt not in _OK:
                raise MMBError(f"AnyPrecisionAdamW: {name} must be torch.float32 or torch.bfloat16, got {dt}")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, use_kahan_summation=use_kahan_summation,
                        momentum_dtype=momentum_dtype, variance_dtype=variance_dtype,
                        compensation_buffer_dtype=compensation_buffer_dtype)
        super().__init__(params, defaults)

    @torch.no_grad()
    def step(self, closure: Any = None) -> None:
        if closure is not None:
            with torch.enable_grad():
                closure()   # as the reference: the returned loss is not kept (anyprecision.py:104-108)
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("AnyPrecisionAdamW does not support sparse gradients")
                if not p.is_cuda or p.dtype != torch.float32 or p.grad.dtype != torch.float32:
                    raise MMBError("AnyPrecisionAdamW: parameters and gradients must be fp32 CUDA tensors")
                if not p.is_contiguous() or not p.grad.is_contiguous():
                    raise MMBError("AnyPrecisionAdamW: parameters and gradients must be contiguous")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = torch.tensor(0.0)
                    state["exp_avg"] = torch.zeros_like(p, dtype=group["momentum_dtype"])
                    state["exp_avg_sq"] = torch.zeros_like(p, dtype=group["variance_dtype"])
                    if group["use_kahan_summation"]:
                        state["compensation"] = torch.zeros_like(p, dtype=group["compensation_buffer_dtype"])
                state["step"] += 1
                ops.anyprecision_adamw_step(p.data, p.grad, state["exp_avg"], state["exp_avg_sq"],
                                            state.get("compensation") if group["use_kahan_summation"] else None, None,
                                            group["lr"], beta1, beta2, group["eps"], group["weight_decay"],
                                            int(state["step"].item()), grad_scale=1.0, zero_grad=False)
