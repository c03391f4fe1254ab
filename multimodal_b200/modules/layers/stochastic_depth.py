"""Stochastic depth (arXiv 1603.09382) — drop-in for torchvision's `StochasticDepth` / `stochastic_depth`
(torchvision/ops/stochastic_depth.py), which `TransformerEncoderLayer(drop_path_rate=...)` uses for both residual
branches (torchmultimodal/modules/layers/transformer.py:63-70).  The package does not import torchvision.

`drop_path_scales` is the one place the layer runtimes draw the noise.  It makes the reference's calls — per call
`torch.empty([B, 1, 1], float32, device).bernoulli_(1 - p)`, then `div_(1 - p)` when 1 - p > 0 — with the same shapes,
device, dtype and order (per layer the attention branch, then the feed-forward branch), and makes none where the
reference makes none (p == 0, or the module not training).  So with the same seed the same samples are dropped, and the
generator advances by the same amount.  The kernels take the drawn tensors as they are: a sample's factor is 0 or
1/(1-p) exactly as torch computed it, never recomputed from p.  Drawing a whole stack's noise before the stack runs is
equivalent to drawing it layer by layer, because nothing else draws in between."""
from typing import List, Optional, Sequence, Tuple

import torch
from torch import nn, Tensor


def _noise(p: float, mode: str, training: bool, size: Sequence[int], dtype, device) -> Optional[Tensor]:
    """The noise torchvision's stochastic_depth multiplies by, or None where it returns its input unchanged."""
    if p < 0.0 or p > 1.0:
        raise ValueError(f"drop probability has to be between 0 and 1, but got {p}")
    if mode not in ["batch", "row"]:
        raise ValueError(f"mode has to be either 'batch' or 'row', but got {mode}")
    if not training or p == 0.0:
        return None
    survival_rate = 1.0 - p
    if mode == "batch":
        size = [1] * len(size)
    noise = torch.empty(list(size), dtype=dtype, device=device)
    noise = noise.bernoulli_(survival_rate)
    if survival_rate > 0.0:
        noise.div_(survival_rate)
    return noise


class StochasticDepth(nn.Module):
    """torchvision.ops.StochasticDepth: randomly zeroes whole rows ("row") or the whole input ("batch") in training and
    rescales the kept ones by 1 / (1 - p).  Inside the layer runtimes the factor is applied by the residual-add and
    LayerNorm-backward kernels; called on its own the module multiplies its input."""

    def __init__(self, p: float, mode: str) -> None:
        super().__init__()
        self.p = p
        self.mode = mode

    def forward(self, input: Tensor) -> Tensor:
        noise = _noise(self.p, self.mode, self.training, [input.shape[0]] + [1] * (input.ndim - 1), input.dtype,
                       input.device)
        return input if noise is None else input * noise

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(p={self.p}, mode={self.mode})"


BranchScales = List[Tuple[Optional[Tensor], Optional[Tensor]]]


def drop_path_scales(layers: Sequence[nn.Module], batch_size: int, device) -> Optional[BranchScales]:
    """Stochastic depth of a stack of `TransformerEncoderLayer`s for one batch: per layer (attention, feed-forward)
    factors, each fp32 [batch_size] (0 or 1/(1-p) per sample) or None where nothing is drawn (no rate, p == 0, not
    training).  None when no layer draws, so that a stack without drop path runs its unscaled launches.  Raises
    ValueError for p outside [0, 1] in either mode, where the reference's forward raises."""
    out: BranchScales = []
    for layer in layers:
        pair = []
        for mod in (getattr(layer, "attention_dropout", None), getattr(layer, "feedforward_dropout", None)):
            noise = None
            if isinstance(mod, StochasticDepth):
                noise = _noise(mod.p, mod.mode, mod.training, [batch_size, 1, 1], torch.float32, device)
            pair.append(None if noise is None else noise.reshape(-1).expand(batch_size).contiguous())
        out.append((pair[0], pair[1]))
    return out if any(s is not None for pair in out for s in pair) else None
