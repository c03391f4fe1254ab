"""CoCa text decoder — drop-in for torchmultimodal/models/coca/text_decoder.py:16-252 (`CoCaTextEmbeddings`,
`CoCaTextDecoder`): same constructor, state-dict keys, initialisation and mask semantics.  Forward =
`engine_coca_train.TextDecoderTrainRuntime` (embedding gather + CLS append in one kernel, fused decoder stack, LayerNorm of the CLS
row only, projection GEMM)."""
from typing import Any, Callable, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn, Tensor

from ..._lib import MMBError
from ...engine import _RuntimeOwner
from ...modules.layers.transformer import TransformerDecoder
from ...utils.attention import get_causal_attention_mask


class CoCaTextEmbeddings(nn.Module):
    def __init__(self, vocab_size: int, num_positions: int, embedding_dim: int, pad_idx: Optional[int] = 0,
                 embed_cls: bool = True):
        super().__init__()
        self.num_positions = num_positions
        if embed_cls:
            self.cls_embedding = nn.Parameter(torch.empty(embedding_dim))
        else:
            self.cls_embedding = None
        self.token_embeddings = nn.Embedding(vocab_size, embedding_dim, pad_idx)
        self.position_embeddings = nn.Parameter(torch.empty(num_positions, embedding_dim))
        self.init_parameters()

    def init_parameters(self) -> None:
        nn.init.normal_(self.token_embeddings.weight, std=0.02)
        nn.init.normal_(self.position_embeddings, std=0.01)
        if self.cls_embedding is not None:
            nn.init.constant_(self.cls_embedding, 0.01)

    def forward(self, *args: Any, **kwargs: Any) -> Tensor:
        raise MMBError("CoCaTextEmbeddings runs inside CoCaTextDecoder's fused runtime; not a standalone op here")


class CoCaTextDecoder(_RuntimeOwner):
    def __init__(self, vocab_size: int, num_positions: int, embedding_dim: int, n_layer: int, n_head: int,
                 dim_feedforward: int, output_dim: int, pad_idx: Optional[int] = 0, embed_cls: bool = True,
                 dropout: float = 0.0, activation: Callable[..., nn.Module] = nn.GELU, layer_norm_eps: float = 1e-5,
                 norm_first: bool = True, final_layer_norm_eps: Optional[float] = 1e-5):
        super().__init__()
        self.pad_idx = pad_idx
        self.embed_cls = embed_cls
        self.num_positions = num_positions
        self.embeddings = CoCaTextEmbeddings(vocab_size=vocab_size, num_positions=num_positions,
                                             embedding_dim=embedding_dim, pad_idx=pad_idx, embed_cls=embed_cls)
        self.transformer_decoder = TransformerDecoder(
            n_layer=n_layer, d_model=embedding_dim, n_head=n_head, dim_feedforward=dim_feedforward, dropout=dropout,
            activation=activation, layer_norm_eps=layer_norm_eps, norm_first=norm_first, use_cross_attention=False)
        if final_layer_norm_eps is not None:
            self.ln_final = nn.LayerNorm(normalized_shape=embedding_dim, eps=final_layer_norm_eps)
        self.text_projection = nn.Linear(embedding_dim, output_dim, bias=False)
        self.register_buffer("causal_mask", get_causal_attention_mask(num_positions).to(dtype=torch.bool),
                             persistent=False)
        self.init_parameters(embedding_dim, n_layer)

    def init_parameters(self, embedding_dim: int, n_layer: int) -> None:
        attn_std = embedding_dim ** -0.5
        proj_std = (2 * embedding_dim * n_layer) ** -0.5
        fc_std = (2 * embedding_dim) ** -0.5
        for layer in self.transformer_decoder.layer:
            nn.init.normal_(layer.attention.q_proj.weight, std=attn_std)
            nn.init.normal_(layer.attention.k_proj.weight, std=attn_std)
            nn.init.normal_(layer.attention.v_proj.weight, std=attn_std)
            nn.init.normal_(layer.attention.output_proj.weight, std=proj_std)
            nn.init.normal_(layer.feedforward.model[0].weight, std=fc_std)
            nn.init.normal_(layer.feedforward.model[2].weight, std=proj_std)
        nn.init.normal_(self.text_projection.weight, std=embedding_dim ** 0.5)

    def build_mask(self, input_ids: Tensor, padding_mask: Optional[Tensor] = None) -> Tensor:
        """Same tensor as the reference (:141-162): causal for every text row; the appended CLS row additionally
        honours the padding mask (shifted by one column, column 0 always visible)."""
        if not self.embed_cls or self.pad_idx is None:
            return self.causal_mask
        if padding_mask is None:
            padding_mask = input_ids != self.pad_idx
        padding_mask = padding_mask.unsqueeze(1)
        padding_mask = F.pad(padding_mask, (1, 0, padding_mask.shape[2], 0), value=1.0)
        mask = (padding_mask * self.causal_mask).unsqueeze(1)
        return mask

    def forward(self, input_ids: Tensor, padding_mask: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
        if self.embed_cls:
            if input_ids.shape[1] == self.num_positions:
                input_ids = input_ids[:, :-1]
            if padding_mask is not None and padding_mask.shape[1] == self.num_positions:
                padding_mask = padding_mask[:, :-1]
        target_shape = self.num_positions - 1 if self.embed_cls else self.num_positions
        assert input_ids.shape[1] == target_shape, f"{input_ids.shape} doesn't match ({target_shape},*)"
        mask = self.build_mask(input_ids, padding_mask)
        S = self.num_positions
        mask_u8 = None
        if mask.dim() == 4:   # [B, 1, S, S] (batch-dependent); a bare causal_mask runs as the kernels' causal flag
            mask_u8 = (mask[:, 0] != 0).to(torch.uint8).contiguous()
        from ...engine import run, wants_grad
        if wants_grad(self):
            pooled, XF = run(self._runtime(), (input_ids, mask_u8, S), ())
            B = input_ids.shape[0]
            return pooled, XF.view(B, S, -1)[:, :-1]       # tokens: every row but the appended CLS one (:190-191)
        with torch.no_grad():
            return self._runtime().infer(input_ids, mask_u8, S)


def _txt_runtime(mod):
    from ...engine_coca_train import TextDecoderTrainRuntime
    return TextDecoderTrainRuntime(mod)


CoCaTextDecoder._runtime_cls = staticmethod(_txt_runtime)
