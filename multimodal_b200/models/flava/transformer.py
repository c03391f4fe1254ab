"""FLAVA transformer blocks — drop-in parameter containers for torchmultimodal/models/flava/transformer.py:18-310
(`FLAVATransformerWithoutEmbeddings`, `TransformerEncoderLayer`, `TransformerEncoder`, `init_transformer_weights`).

Same constructors, state-dict keys (``layer.{i}.attention.{query,key,value,output}``, ``feedforward.model.{0,2}``,
``attention_layernorm``, ``feedforward_layernorm``) and initialisation order.  The layers themselves never run as torch
modules: the owning encoder hands the whole stack to its ``engine_flava_train`` runtime (forward + backward under
autograd, or the forward alone under torch.no_grad(); DESIGN.md §10).
"""
from functools import partial
from typing import Any, Callable, Optional

import torch
from torch import nn, Tensor

from ..._lib import MMBError
from ...engine import _RuntimeOwner
from ...modules.layers.attention import MultiHeadAttention, SelfAttention
from ...modules.layers.mlp import MLP
from ...modules.layers.normalizations import Fp32LayerNorm
from ...modules.layers.transformer import TransformerOutput


class TransformerEncoderLayer(nn.Module):
    def __init__(self, d_model: int, n_head: int, dim_feedforward: int, dropout: float = 0.0,
                 activation: Callable[..., nn.Module] = nn.ReLU, layer_norm_eps: float = 1e-12,
                 norm_first: bool = False) -> None:
        super().__init__()
        if dropout != 0.0:
            raise NotImplementedError("dropout > 0 is not on the accelerated FLAVA path (reference default is 0.0)")
        self.attention = MultiHeadAttention(dim_q=d_model, dim_kv=d_model, n_head=n_head,
                                            attn_module=SelfAttention(dropout))
        self.attention_dropout = nn.Dropout(dropout)
        self.feedforward = MLP(d_model, d_model, dim_feedforward, dropout=dropout, activation=activation)
        self.feedforward_dropout = nn.Dropout(dropout)
        self.attention_layernorm = Fp32LayerNorm(d_model, eps=layer_norm_eps)
        self.feedforward_layernorm = Fp32LayerNorm(d_model, eps=layer_norm_eps)
        self.norm_first = norm_first

    def forward(self, *args: Any, **kwargs: Any) -> Tensor:
        raise MMBError("TransformerEncoderLayer runs inside its encoder's fused runtime; not a standalone op here")


class TransformerEncoder(nn.Module):
    def __init__(self, n_layer: int, d_model: int, n_head: int, dim_feedforward: int, dropout: float = 0.0,
                 activation: Callable[..., nn.Module] = nn.ReLU, layer_norm_eps: float = 1e-12, norm_first: bool = False,
                 final_layer_norm_eps: Optional[float] = None):
        super().__init__()
        self.layer = nn.ModuleList([
            TransformerEncoderLayer(d_model, n_head, dim_feedforward, dropout, activation, layer_norm_eps, norm_first)
            for _ in range(n_layer)])
        self.final_layer_norm = None
        if final_layer_norm_eps:
            raise NotImplementedError("final_layer_norm inside TransformerEncoder is not used by FLAVA")

    def forward(self, *args: Any, **kwargs: Any) -> TransformerOutput:
        raise MMBError("TransformerEncoder runs inside its encoder's fused runtime; not a standalone op here")


def init_transformer_weights(module: nn.Module, initializer_range: float) -> None:
    """Same rule as transformer.py:296-310: N(0, range) Linear/Conv/Embedding weights, zero biases and padding row,
    unit LayerNorms."""
    if isinstance(module, (nn.Linear, nn.Conv2d)):
        module.weight.data.normal_(mean=0.0, std=initializer_range)
        if module.bias is not None:
            module.bias.data.zero_()
    elif isinstance(module, nn.Embedding):
        module.weight.data.normal_(mean=0.0, std=initializer_range)
        if module.padding_idx is not None:
            module.weight.data[module.padding_idx].zero_()
    elif isinstance(module, nn.LayerNorm):
        module.bias.data.zero_()
        module.weight.data.fill_(1.0)


class FLAVATransformerWithoutEmbeddings(_RuntimeOwner):
    """The multimodal encoder (transformer.py:18-77): [cls | hidden_states] -> L layers -> layernorm -> pooler."""

    def __init__(self, encoder: nn.Module, layernorm: nn.Module, pooler: nn.Module, hidden_size: int = 768,
                 weight_init_fn: Optional[Callable] = None, initializer_range: float = 0.02, use_cls_token: bool = True,
                 **kwargs: Any):
        super().__init__()
        self.encoder = encoder
        self.layernorm = layernorm
        self.pooler = pooler
        if use_cls_token:
            self.cls_token = nn.Parameter(torch.zeros(1, 1, hidden_size))
        else:
            self.cls_token = None
        if weight_init_fn is None:
            weight_init_fn = partial(init_transformer_weights, initializer_range=initializer_range)
        self.apply(weight_init_fn)

    def forward(self, hidden_states: Optional[Tensor] = None, attention_mask: Optional[Tensor] = None) -> TransformerOutput:
        if hidden_states is None:
            raise ValueError("You have to specify hidden_states")
        if attention_mask is not None:
            raise NotImplementedError("attention_mask on the multimodal encoder is not on the accelerated path")
        from ... import engine_flava_train as T
        from ...engine import wants_grad
        if wants_grad(self) or (torch.is_grad_enabled() and hidden_states.requires_grad):
            return T.encoder_output(self._runtime(), (), (hidden_states,), self.pooler)
        with torch.no_grad():
            return self._runtime().infer(hidden_states, want_attn=bool(getattr(self, "output_attentions", False)))


def _mm_runtime(mod, image_proj=None, text_proj=None):
    from ...engine_flava_train import FlavaMMTrainRuntime
    return FlavaMMTrainRuntime(mod, image_proj, text_proj)


FLAVATransformerWithoutEmbeddings._runtime_cls = staticmethod(_mm_runtime)
