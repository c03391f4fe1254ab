"""Contrastive loss with temperature — drop-in for
torchmultimodal/modules/losses/contrastive_loss_with_temperature.py:17-201.

Same public surface (``ContrastiveLossOutput``, ``contrastive_loss_with_temperature``,
``ContrastiveLossWithTemperature``, ``DEFAULT_LOGIT_SCALE``), same ``ValueError`` / clamp quirks (:172-175, :193).
The computation is ``engine_loss.ContrastiveRuntime``: similarity GEMMs on Hopper tensor cores, temperature scaling +
cross-entropy + all gradients in one kernel pass; with torch.distributed initialised the peers' embeddings are pulled
over NVLink inside the runtime (no NCCL all_gather on this path).
"""
import math
from dataclasses import dataclass
from typing import Any, Dict, Optional, OrderedDict, Union

import torch
from torch import nn, Tensor

from ...engine_loss import contrastive_loss_apply
from ...utils.distributed import BackpropType


@dataclass
class ContrastiveLossOutput(OrderedDict):
    loss: Tensor
    logits_a: Tensor
    logits_b: Tensor
    loss_a: Tensor
    loss_b: Tensor


def contrastive_loss_with_temperature(
    embeddings_a: Tensor,
    embeddings_b: Tensor,
    logit_scale: nn.Parameter,
    mask: Optional[Tensor] = None,
    backprop_type: BackpropType = BackpropType.GLOBAL,
    cross_entropy_kwargs: Optional[Dict[str, Any]] = None,
) -> ContrastiveLossOutput:
    """Functional form; arguments as in the reference (:50-80).  ``cross_entropy_kwargs`` supports
    ``label_smoothing``; anything else raises (never silently ignored)."""
    smoothing = 0.0
    if cross_entropy_kwargs:
        extra = set(cross_entropy_kwargs) - {"label_smoothing"}
        if extra:
            raise NotImplementedError(f"cross_entropy_kwargs {sorted(extra)} are not supported by the fused loss kernel")
        smoothing = float(cross_entropy_kwargs.get("label_smoothing", 0.0))
    loss, logits_a, logits_b, loss_a, loss_b = contrastive_loss_apply(
        embeddings_a, embeddings_b, logit_scale, smoothing, backprop_type, mask, want_logits=True)
    return ContrastiveLossOutput(loss=loss, logits_a=logits_a, logits_b=logits_b, loss_a=loss_a, loss_b=loss_b)


DEFAULT_LOGIT_SCALE = math.log(1 / 0.07)


class ContrastiveLossWithTemperature(nn.Module):
    """Contrastive loss with a learnt, clamped temperature (CLIP / FLAVA).  Arguments and defaults as the reference
    (:121-183)."""

    def __init__(
        self,
        logit_scale: Union[float, nn.Parameter] = DEFAULT_LOGIT_SCALE,
        logit_scale_min: Optional[float] = math.log(1),
        logit_scale_max: Optional[float] = math.log(100),
    ):
        super().__init__()
        # Reference quirk kept on purpose (:172): the test is truthiness, so (min=0.0, max=None) also raises.
        if not logit_scale_min and not logit_scale_max:
            raise ValueError("Only one of `logit_scale_min` and `logit_scale_max` can be None.")
        self.logit_scale_min = logit_scale_min
        self.logit_scale_max = logit_scale_max
        if isinstance(logit_scale, nn.Parameter):
            self.logit_scale = logit_scale
        else:
            self.logit_scale = nn.Parameter(logit_scale * torch.ones([]))

    def forward(
        self,
        embeddings_a: Tensor,
        embeddings_b: Tensor,
        backprop_type: BackpropType = BackpropType.GLOBAL,
        cross_entropy_kwargs: Optional[Dict[str, Any]] = None,
        mask: Optional[Tensor] = None,
    ) -> Tensor:
        self.logit_scale.data.clamp_(self.logit_scale_min, self.logit_scale_max)  # :193, in place, every call
        smoothing = 0.0
        if cross_entropy_kwargs:
            extra = set(cross_entropy_kwargs) - {"label_smoothing"}
            if extra:
                raise NotImplementedError(
                    f"cross_entropy_kwargs {sorted(extra)} are not supported by the fused loss kernel")
            smoothing = float(cross_entropy_kwargs.get("label_smoothing", 0.0))
        return contrastive_loss_apply(embeddings_a, embeddings_b, self.logit_scale, smoothing, backprop_type, mask,
                                      want_logits=False)[0]
