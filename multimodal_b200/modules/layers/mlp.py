"""Parameter container mirroring torchmultimodal/modules/layers/mlp.py:13-66 (state-dict keys ``model.{i}.*``).
Inside the FLAVA encoders the MLP runs as two wgmma GEMMs with the GELU fused into the first epilogue."""
from typing import Callable, List, Optional, Union

import torch
from torch import nn

from ..._lib import MMBError


class MLP(nn.Module):
    def __init__(self, in_dim: int, out_dim: int, hidden_dims: Optional[Union[int, List[int]]] = None,
                 dropout: float = 0.5, activation: Callable[..., nn.Module] = nn.ReLU,
                 normalization: Optional[Callable[..., nn.Module]] = None) -> None:
        super().__init__()
        layers = nn.ModuleList()
        if hidden_dims is None:
            hidden_dims = []
        if isinstance(hidden_dims, int):
            hidden_dims = [hidden_dims]
        for hidden_dim in hidden_dims:
            layers.append(nn.Linear(in_dim, hidden_dim))
            if normalization:
                layers.append(normalization(hidden_dim))
            layers.append(activation())
            if dropout > 0:
                layers.append(nn.Dropout(dropout))
            in_dim = hidden_dim
        layers.append(nn.Linear(in_dim, out_dim))
        self.model = nn.Sequential(*layers)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """Standalone forward (values only) of the [Linear, activation, Linear] form: GEMM + fused activation, GEMM."""
        from ...engine_layers import mlp_forward

        return mlp_forward(self, x)
