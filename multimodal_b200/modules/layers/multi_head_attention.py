"""Parameter containers mirroring torchmultimodal/modules/layers/multi_head_attention.py:19-180
(`MultiHeadSelfAttention` with the fused ``input_proj [3d, d]``; `MultiHeadAttentionWithCache` with separate
``q_proj / k_proj / v_proj / output_proj``).  They execute inside the owning encoder / decoder / pooler runtime
(engine_coca.py): packed-QKV wgmma GEMM + attention kernel; F.scaled_dot_product_attention is never called."""
from typing import Any, Optional

from torch import nn, Tensor

from ..._lib import MMBError


class MultiHeadSelfAttention(nn.Module):
    def __init__(self, embed_dim: int, num_heads: int, dropout: float = 0.0):
        super().__init__()
        self.input_proj = nn.Linear(embed_dim, 3 * embed_dim)
        self.output_proj = nn.Linear(embed_dim, embed_dim)
        self.num_heads = num_heads
        self.dropout = dropout

    def forward(self, query: Tensor, attn_mask: Optional[Tensor] = None, is_causal: bool = False) -> Tensor:
        """Standalone forward (values only): packed in-projection GEMM -> attention kernel -> out-projection GEMM."""
        from ...engine_layers import mhsa_forward

        return mhsa_forward(self, query, attn_mask, is_causal)


class MultiHeadAttentionWithCache(nn.Module):
    def __init__(self, dim_q: int, dim_kv: int, num_heads: int, dropout: float = 0.0, add_bias: bool = True) -> None:
        super().__init__()
        self.num_heads = num_heads
        self.q_proj = nn.Linear(dim_q, dim_q, bias=add_bias)
        self.k_proj = nn.Linear(dim_kv, dim_q, bias=add_bias)
        self.v_proj = nn.Linear(dim_kv, dim_q, bias=add_bias)
        self.output_proj = nn.Linear(dim_q, dim_q)
        self.dropout = dropout

    def forward(self, *args: Any, **kwargs: Any) -> Tensor:
        raise MMBError("MultiHeadAttentionWithCache is fused into the decoder / pooler runtime; not a standalone op "
                       "here (KV-cache decoding is outside the accelerated forward path)")
