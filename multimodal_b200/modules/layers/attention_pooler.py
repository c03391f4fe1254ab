"""`AttentionPooler` / `CascadedAttentionPooler` — drop-in for torchmultimodal/modules/layers/attention_pooler.py
:16-101.  Forward = `engine_coca_train.PoolerTrainRuntime`: LayerNorm-ed keys/values projected by one packed GEMM, the learned
queries projected once (they do not depend on the batch), cross-attention on the general attention kernel (head_dim 96
for CoCa ViT-L/14), output projection + ln_post.  With grad mode on and trainable parameters (or an input that requires grad) the call
runs under autograd (the learned queries' gradient is summed over the batch)."""
from typing import List

import torch
from torch import nn, Tensor

from ...engine import _RuntimeOwner
from .multi_head_attention import MultiHeadAttentionWithCache


class AttentionPooler(_RuntimeOwner):
    def __init__(self, input_embed_dim: int, output_embed_dim: int, n_head: int, n_queries: int = 256,
                 layer_norm_eps: float = 1e-5):
        super().__init__()
        self.query = nn.Parameter(torch.randn(n_queries, output_embed_dim))
        self.attn = MultiHeadAttentionWithCache(dim_q=output_embed_dim, dim_kv=input_embed_dim, num_heads=n_head)
        self.ln_q = nn.LayerNorm(output_embed_dim, layer_norm_eps)
        self.ln_k = nn.LayerNorm(input_embed_dim, layer_norm_eps)
        self.ln_post = nn.LayerNorm(output_embed_dim, layer_norm_eps)

    def forward(self, x: Tensor) -> Tensor:
        from ...engine import run, wants_grad
        if wants_grad(self) or (torch.is_grad_enabled() and x.requires_grad):
            (out,) = run(self._runtime(), None, (x,))
            return out.view(x.shape[0], self.query.shape[0], self.query.shape[1])
        with torch.no_grad():
            return self._runtime().infer(x)


def _pool_runtime(mod):
    from ...engine_coca_train import PoolerTrainRuntime
    return PoolerTrainRuntime(mod)


AttentionPooler._runtime_cls = staticmethod(_pool_runtime)


class CascadedAttentionPooler(nn.Module):
    def __init__(self, poolers: List[AttentionPooler]):
        super().__init__()
        self.poolers = nn.ModuleList(poolers)

    def forward(self, x: Tensor) -> List[Tensor]:
        pooler_outs = []
        for pooler in self.poolers:
            x = pooler(x)
            pooler_outs.append(x)
        return pooler_outs
