"""Mirror of torchmultimodal/modules/layers/transformer.py: `TransformerOutput` (:22-28, the NamedTuple every FLAVA /
CoCa encoder returns) and the parameter containers `TransformerEncoderLayer` / `TransformerEncoder` (:31-259) and
`TransformerDecoderLayer` / `TransformerDecoder` (:262-657) — same constructors, state-dict keys and creation order.
The layers execute inside `engine.TransformerStack` (fused kernels), owned by VisionTransformer / CoCaTextDecoder /
CoCaMultimodalDecoder; all four are also callable on their own (same kernels: `engine_layers.py`).  A
`TransformerEncoderLayer` / `TransformerEncoder` is then a runtime owner like the encoders: one runtime serves
torch.no_grad() and training (pre-norm: its own `TransformerStack`; post-norm: `PostNormLayersRuntime`).  The decoders
compute forward values, with the reference's key / value cache (`past_key_values` / `use_cache`) for autoregressive
decoding.

With `drop_path_rate` an encoder layer applies stochastic depth as the reference does: one shared
`StochasticDepth(p, "row")` (modules/layers/stochastic_depth.py) is both `attention_dropout` and `feedforward_dropout`,
and `TransformerEncoder` gives layer i the rate `torch.linspace(0, drop_path_rate, n_layer)[i]`.  In training the
runtimes draw the per-sample noise in the reference's order and scale each branch inside the residual-add and
LayerNorm-backward kernels; it adds no parameters."""
from typing import Callable, List, NamedTuple, Optional, Tuple

import torch
from torch import nn, Tensor

from ...engine import _RuntimeOwner


class TransformerOutput(NamedTuple):
    last_hidden_state: Optional[Tensor] = None
    pooler_output: Optional[Tensor] = None
    hidden_states: Optional[List[Tensor]] = None
    attentions: Optional[List[Tensor]] = None
    image_labels: Optional[Tensor] = None
    current_key_values: Optional[List[Tuple[Tensor, Tensor]]] = None


def _no_dropout(dropout: float, what: str) -> None:
    if dropout != 0.0:
        raise NotImplementedError(f"{what}: dropout > 0 is not on the accelerated path (reference default is 0.0)")


class TransformerEncoderLayer(_RuntimeOwner):
    def __init__(self, d_model: int, n_head: int, dim_feedforward: int, dropout: float = 0.0,
                 activation: Callable[..., nn.Module] = nn.ReLU, layer_norm_eps: float = 1e-12, norm_first: bool = False,
                 drop_path_rate: Optional[float] = None) -> None:
        super().__init__()
        from .mlp import MLP
        from .multi_head_attention import MultiHeadSelfAttention
        from .normalizations import Fp32LayerNorm
        from .stochastic_depth import StochasticDepth

        _no_dropout(dropout, "TransformerEncoderLayer")
        self.attention = MultiHeadSelfAttention(embed_dim=d_model, num_heads=n_head)
        if drop_path_rate is not None:
            self.attention_dropout = self.feedforward_dropout = StochasticDepth(drop_path_rate, mode="row")
        else:
            self.attention_dropout = nn.Dropout(dropout)
            self.feedforward_dropout = nn.Dropout(dropout)
        self.feedforward = MLP(d_model, d_model, dim_feedforward, dropout=dropout, activation=activation)
        self.attention_layernorm = Fp32LayerNorm(d_model, eps=layer_norm_eps)
        self.feedforward_layernorm = Fp32LayerNorm(d_model, eps=layer_norm_eps)
        self.norm_first = norm_first

    def forward(self, hidden_states: Tensor, attention_mask: Optional[Tensor] = None) -> Tensor:
        """Standalone forward (inside VisionTransformer the layer runs in the owner's fused TransformerStack)."""
        from ...engine_layers import encoder_layer_forward

        return encoder_layer_forward(self, hidden_states, attention_mask)


class TransformerEncoder(_RuntimeOwner):
    def __init__(self, n_layer: int, d_model: int, n_head: int, dim_feedforward: int, dropout: float = 0.0,
                 activation: Callable[..., nn.Module] = nn.ReLU, layer_norm_eps: float = 1e-12, norm_first: bool = False,
                 final_layer_norm_eps: Optional[float] = None, drop_path_rate: Optional[float] = None):
        super().__init__()
        from .normalizations import Fp32LayerNorm

        if drop_path_rate is not None:
            drop_rate = [x.item() for x in torch.linspace(0, drop_path_rate, n_layer)]
        else:
            drop_rate = [None for _ in range(n_layer)]
        self.layer = nn.ModuleList([
            TransformerEncoderLayer(d_model, n_head, dim_feedforward, dropout, activation, layer_norm_eps, norm_first,
                                    drop_rate[i]) for i in range(n_layer)])
        self.final_layer_norm = None
        if final_layer_norm_eps:
            self.final_layer_norm = Fp32LayerNorm(d_model, eps=final_layer_norm_eps)

    def forward(self, hidden_states: Tensor, attention_mask: Optional[Tensor] = None,
                return_hidden_states: bool = False) -> TransformerOutput:
        """Standalone forward (inside VisionTransformer the stack runs in the owner's fused TransformerStack)."""
        from ...engine_layers import encoder_forward

        return encoder_forward(self, hidden_states, attention_mask, return_hidden_states)


def _layers_runtime(owner, layers, final_ln):
    from ...engine_layers import EncoderLayersRuntime, PostNormLayersRuntime
    from ..._lib import MMBError

    kinds = {layer.norm_first for layer in layers}
    if len(kinds) != 1:
        raise MMBError("TransformerEncoder: layers that mix pre-norm and post-norm are not on the accelerated path")
    return (EncoderLayersRuntime if kinds.pop() else PostNormLayersRuntime)(owner, layers, final_ln)


def _layer_runtime(mod):
    return _layers_runtime(mod, [mod], None)


def _encoder_runtime(mod):
    return _layers_runtime(mod, mod.layer, mod.final_layer_norm)


TransformerEncoderLayer._runtime_cls = staticmethod(_layer_runtime)
TransformerEncoder._runtime_cls = staticmethod(_encoder_runtime)


class TransformerDecoderLayer(nn.Module):
    def __init__(self, d_model: int, n_head: int, dim_feedforward: int, dropout: float = 0.0,
                 activation: Callable[..., nn.Module] = nn.ReLU, layer_norm_eps: float = 1e-12, norm_first: bool = False,
                 use_cross_attention: bool = True, dim_kv: Optional[int] = None) -> None:
        super().__init__()
        from .mlp import MLP
        from .multi_head_attention import MultiHeadAttentionWithCache
        from .normalizations import Fp32LayerNorm

        _no_dropout(dropout, "TransformerDecoderLayer")
        dim_kv = dim_kv if dim_kv is not None else d_model
        self.attention = MultiHeadAttentionWithCache(dim_q=d_model, dim_kv=d_model, num_heads=n_head, dropout=dropout)
        self.attention_dropout = nn.Dropout(dropout)
        self.cross_attention: Optional[MultiHeadAttentionWithCache] = None
        self.use_cross_attention = use_cross_attention
        if self.use_cross_attention:
            self.cross_attention = MultiHeadAttentionWithCache(dim_q=d_model, dim_kv=dim_kv, num_heads=n_head,
                                                               dropout=dropout)
            self.cross_attention_layernorm = Fp32LayerNorm(d_model, eps=layer_norm_eps)
            self.cross_attention_dropout = nn.Dropout(dropout)
        self.feedforward = MLP(d_model, d_model, dim_feedforward, dropout=dropout, activation=activation)
        self.feedforward_dropout = nn.Dropout(dropout)
        self.attention_layernorm = Fp32LayerNorm(d_model, eps=layer_norm_eps)
        self.feedforward_layernorm = Fp32LayerNorm(d_model, eps=layer_norm_eps)
        self.norm_first = norm_first

    def forward(self, hidden_states: Tensor, encoder_hidden_states: Optional[Tensor] = None,
                attention_mask: Optional[Tensor] = None, cross_attention_mask: Optional[Tensor] = None,
                past_key_value: Optional[Tuple[Tensor, Tensor]] = None,
                use_cache: bool = False) -> Tuple[Tensor, Optional[Tuple[Tensor, Tensor]]]:
        """Standalone forward (values only; inside CoCa the layer runs in the fused TransformerStack)."""
        from ...engine_layers import decoder_layer_forward

        return decoder_layer_forward(self, hidden_states, encoder_hidden_states, attention_mask, cross_attention_mask,
                                     past_key_value, use_cache)


class TransformerDecoder(nn.Module):
    def __init__(self, n_layer: int, d_model: int, n_head: int, dim_feedforward: int, dropout: float = 0.0,
                 activation: Callable[..., nn.Module] = nn.ReLU, layer_norm_eps: float = 1e-12, norm_first: bool = False,
                 use_cross_attention: bool = True, dim_kv: Optional[int] = None,
                 final_layer_norm_eps: Optional[float] = None, cross_attention_interval: int = 1):
        super().__init__()
        from .normalizations import Fp32LayerNorm

        if use_cross_attention and cross_attention_interval != 1:
            raise NotImplementedError("cross_attention_interval != 1 is not on the accelerated path")
        self.layer = nn.ModuleList([
            TransformerDecoderLayer(d_model, n_head, dim_feedforward, dropout, activation, layer_norm_eps, norm_first,
                                    use_cross_attention and (i % cross_attention_interval == 0), dim_kv)
            for i in range(n_layer)])
        self.final_layer_norm = None
        if final_layer_norm_eps:
            self.final_layer_norm = Fp32LayerNorm(d_model, eps=final_layer_norm_eps)

    def forward(self, hidden_states: Tensor, encoder_hidden_states: Optional[Tensor] = None,
                attention_mask: Optional[Tensor] = None, cross_attention_mask: Optional[Tensor] = None,
                past_key_values: Optional[List[Tuple[Tensor, Tensor]]] = None, use_cache: bool = False,
                return_hidden_states: bool = False) -> TransformerOutput:
        """Standalone forward (values only; inside CoCa the stack runs in the fused TransformerStack)."""
        from ...engine_layers import decoder_forward

        return decoder_forward(self, hidden_states, encoder_hidden_states, attention_mask, cross_attention_mask,
                               past_key_values, use_cache, return_hidden_states)
