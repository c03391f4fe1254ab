"""`BERTTextEncoder` — drop-in for torchmultimodal/modules/encoders/bert_text_encoder.py:17-176.  Same constructor,
state-dict keys and argument meaning; the forward is `engine_flava_train.FlavaTextTrainRuntime` (fused embedding-sum + LayerNorm,
pad-derived key mask consumed by the tensor-core attention kernel, fused layer stack, layernorm, pooler).

On the accelerated path: `input_ids` (required), `attention_mask` of shape [batch, seq_len], `token_type_ids`.
`position_ids` / `inputs_embeds` raise NotImplementedError; `return_attn_weights=True` returns the
per-layer attention probabilities (recomputed from QKV + row LSE by mmb_attention_probs; the fused attention kernel
itself never materialises them)."""
from typing import Callable, Optional

import torch
from torch import nn, Tensor

from ...engine import _RuntimeOwner
from ...models.flava.transformer import TransformerEncoder
from ..layers.text_embedding import BERTTextEmbeddings
from ..layers.transformer import TransformerOutput


class BERTTextEncoder(_RuntimeOwner):
    def __init__(self, embeddings: nn.Module, encoder: nn.Module, layernorm: Optional[nn.Module] = None,
                 pooler: Optional[nn.Module] = None, weight_init_fn: Optional[Callable] = None) -> None:
        super().__init__()
        self.embeddings = embeddings
        self.encoder = encoder
        self.layernorm = layernorm
        self.pooler = pooler
        if weight_init_fn:
            self.apply(weight_init_fn)

    def forward(self, input_ids: Optional[Tensor] = None, attention_mask: Optional[Tensor] = None,
                token_type_ids: Optional[Tensor] = None, position_ids: Optional[Tensor] = None,
                inputs_embeds: Optional[Tensor] = None, return_attn_weights: bool = False,
                return_hidden_states: bool = False) -> TransformerOutput:
        if input_ids is None and inputs_embeds is None:
            raise ValueError("input_ids or inputs_embeds must not be None")
        if inputs_embeds is not None or position_ids is not None:
            raise NotImplementedError("inputs_embeds / position_ids are not on the accelerated path")
        if self.layernorm is None:
            raise NotImplementedError("BERTTextEncoder without a final layernorm is not on the accelerated path")
        from ... import engine_flava_train as T
        from ...engine import wants_grad
        if wants_grad(self):   # training: forward keeps activations, autograd nodes carry the explicit backward
            if return_attn_weights:
                raise NotImplementedError("attention probabilities are not produced by the training forward")
            out = T.encoder_output(self._runtime(), (input_ids, attention_mask, token_type_ids), (), self.pooler)
        else:
            with torch.no_grad():
                out = self._runtime().infer(input_ids, attention_mask, token_type_ids, want_attn=bool(return_attn_weights))
        if not return_hidden_states:
            out = out._replace(hidden_states=None)
        return out


def _txt_runtime(mod):
    from ...engine_flava_train import FlavaTextTrainRuntime
    return FlavaTextTrainRuntime(mod)


BERTTextEncoder._runtime_cls = staticmethod(_txt_runtime)


def bert_text_encoder(hidden_size: int = 768, num_hidden_layers: int = 6, num_attention_heads: int = 12,
                      intermediate_size: int = 3072, dropout: float = 0.1,
                      transform_act_fn: Callable[..., nn.Module] = nn.GELU, layer_norm_eps: float = 1e-12,
                      norm_first: bool = False, vocab_size: int = 30522, max_position_embeddings: int = 512,
                      type_vocab_size: int = 2, pad_token_id: int = 0, offset_pos_ids: bool = False,
                      layernorm: Optional[nn.Module] = None, pooler: Optional[nn.Module] = None,
                      weight_init_fn: Optional[Callable] = None) -> BERTTextEncoder:
    embeddings = BERTTextEmbeddings(hidden_size=hidden_size, vocab_size=vocab_size, pad_token_id=pad_token_id,
                                    max_position_embeddings=max_position_embeddings, type_vocab_size=type_vocab_size,
                                    layer_norm_eps=layer_norm_eps, dropout=dropout, offset_pos_ids=offset_pos_ids)
    encoder = TransformerEncoder(n_layer=num_hidden_layers, d_model=hidden_size, n_head=num_attention_heads,
                                 dim_feedforward=intermediate_size, dropout=dropout, activation=transform_act_fn,
                                 layer_norm_eps=layer_norm_eps, norm_first=norm_first)
    return BERTTextEncoder(embeddings=embeddings, encoder=encoder, layernorm=layernorm, pooler=pooler,
                           weight_init_fn=weight_init_fn)
