"""Parameter containers mirroring torchmultimodal/modules/layers/multi_head_attention.py:19-180
(`MultiHeadSelfAttention` with the fused ``input_proj [3d, d]``; `MultiHeadAttentionWithCache` with separate
``q_proj / k_proj / v_proj / output_proj``).  They execute inside the owning encoder / decoder / pooler runtime
(engine_coca_train.py): packed-QKV wgmma GEMM + attention kernel; F.scaled_dot_product_attention is never called.  Both are
also callable on their own (forward values, engine_layers.py); `MultiHeadAttentionWithCache` then keeps the reference's
key / value cache (`past_key_value` / `use_cache`) for autoregressive decoding, on the split-KV decode kernel."""
from typing import NamedTuple, Optional, Tuple, Union

from torch import nn, Tensor


class MHAWithCacheOutput(NamedTuple):
    attn_output: Tensor
    past_key_value: Tuple[Tensor, Tensor]


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

    def forward(self, query: Tensor, key: Tensor, value: Tensor, attn_mask: Optional[Tensor] = None,
                past_key_value: Optional[Tuple[Tensor, Tensor]] = None, is_causal: bool = False,
                use_cache: bool = False) -> Union[Tensor, MHAWithCacheOutput]:
        """Standalone forward (values only): projections -> key / value cache append -> attention (split-KV decode
        kernel for queries of at most 16 rows) -> out-projection.  The returned cache tensors [B, H, S, head_dim] are
        fresh on every call, as with torch.cat in the reference."""
        from ...engine_layers import mha_cache_forward

        return mha_cache_forward(self, query, key, value, attn_mask, past_key_value, is_causal, use_cache)
