"""Parameter containers mirroring torchmultimodal/modules/layers/attention.py:15-182 (`SelfAttention`,
`MultiHeadAttention` with separate query/key/value/output Linears).  The FLAVA runtimes pack q/k/v into one [3d, d]
operand and run the fused QKV GEMM + tensor-core attention; attention probabilities are never materialised."""
from typing import Any

from torch import nn, Tensor

from ..._lib import MMBError


class SelfAttention(nn.Module):
    def __init__(self, attn_dropout: float = 0.0) -> None:
        super().__init__()
        self.attn_dropout = attn_dropout

    def forward(self, *args: Any, **kwargs: Any) -> Tensor:
        raise MMBError("SelfAttention is fused into the encoder runtime; not a standalone op here")


class MultiHeadAttention(nn.Module):
    def __init__(self, dim_q: int, dim_kv: int, n_head: int, attn_module: nn.Module = None, add_bias: bool = True) -> None:
        super().__init__()
        if dim_q % n_head != 0 or dim_kv % n_head != 0:
            raise ValueError("The hidden size of q, k, v must be a multiple of the number of attention heads.")
        self.dim_q, self.dim_kv, self.n_head = dim_q, dim_kv, n_head
        self.query = nn.Linear(dim_q, dim_q, bias=add_bias)
        self.key = nn.Linear(dim_kv, dim_q, bias=add_bias)
        self.value = nn.Linear(dim_kv, dim_q, bias=add_bias)
        self.output = nn.Linear(dim_q, dim_q, bias=True)
        self.attn = attn_module if attn_module is not None else SelfAttention()
        self.cache = None

    def forward(self, *args: Any, **kwargs: Any) -> Tensor:
        raise MMBError("MultiHeadAttention is fused into the encoder runtime; not a standalone op here")
