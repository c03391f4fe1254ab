"""CoCa multimodal decoder — drop-in for torchmultimodal/models/coca/multimodal_decoder.py:15-108.  Forward =
`engine_coca_train.MultimodalDecoderTrainRuntime`: causal self-attention on the tensor-core attention kernel, cross-attention to the captioning
image tokens on the general kernel, final LayerNorm + vocabulary projection GEMM (fp32 logits)."""
from typing import Callable, Optional

import torch
from torch import nn, Tensor

from ...engine import _RuntimeOwner
from ...modules.layers.transformer import TransformerDecoder
from ...utils.attention import get_causal_attention_mask


class CoCaMultimodalDecoder(_RuntimeOwner):
    def __init__(self, input_seq_len: int, text_embedding_dim: int, n_layer: int, n_head: int, dim_feedforward: int,
                 output_dim: Optional[int] = None, dropout: float = 0.0, activation: Callable[..., nn.Module] = nn.GELU,
                 layer_norm_eps: float = 1e-5, norm_first: bool = True, final_layer_norm_eps: Optional[float] = 1e-5,
                 visual_embedding_dim: Optional[int] = None):
        super().__init__()
        self.transformer_decoder = TransformerDecoder(
            n_layer=n_layer, d_model=text_embedding_dim, n_head=n_head, dim_feedforward=dim_feedforward, dropout=dropout,
            activation=activation, layer_norm_eps=layer_norm_eps, norm_first=norm_first, use_cross_attention=True,
            final_layer_norm_eps=final_layer_norm_eps, dim_kv=visual_embedding_dim)
        if output_dim is not None:
            self.output_projection = nn.Linear(text_embedding_dim, output_dim, bias=False)
        else:
            self.output_projection = None
        self.register_buffer("causal_mask", get_causal_attention_mask(input_seq_len).to(dtype=torch.bool),
                             persistent=False)

    def forward(self, texts: Tensor, images: Tensor) -> Tensor:
        seq_len = texts.shape[1]
        assert self.causal_mask.shape == (seq_len, seq_len)
        from ... import engine_coca_train as T
        if self.wants_graph(texts, images):
            hidden = self.hidden_states(texts, images)
            if self.output_projection is not None:
                hidden = T.linear_f32(hidden, self.output_projection)
            return hidden
        with torch.no_grad():
            return self._runtime().infer(texts, images)

    def wants_graph(self, texts: Tensor, images: Tensor) -> bool:
        from ...engine import wants_grad
        return wants_grad(self) or (torch.is_grad_enabled() and (texts.requires_grad or images.requires_grad))

    def hidden_states(self, texts: Tensor, images: Tensor) -> Tensor:
        """Training path: the decoder output after its final LayerNorm, [B, S, d] with autograd history (the vocabulary
        projection is applied by the caller: `forward`, or fused with the cross-entropy in CoCaForPretraining)."""
        from ...engine import run
        (out,) = run(self._runtime(), None, (texts, images))
        return out.view(texts.shape[0], texts.shape[1], -1)


def _mm_runtime(mod):
    from ...engine_coca_train import MultimodalDecoderTrainRuntime
    return MultimodalDecoderTrainRuntime(mod)


CoCaMultimodalDecoder._runtime_cls = staticmethod(_mm_runtime)
