"""`VisionTransformer` — drop-in for torchmultimodal/modules/encoders/vision_transformer.py:19-203 (constructor,
`vision_transformer` builder and the vit_* presets).  Forward = `engine_coca_train.VisionTrainRuntime`.  ``attentions`` is None
(flash-style attention); a custom ``pooler`` module, if given, is applied to ``last_hidden_state`` as in the reference.
`GlobalAveragePooler` (MAE fine-tuning head) is outside SURVEY.md §8.  With `patch_drop_rate` the module drops patches in
training only (either grad mode, the same random draws as the reference): `hidden_states` and `last_hidden_state` are
then [B, off + L, d] for the L kept patches (off = 1 with a CLS token).  With `drop_path_rate` the encoder layers apply
stochastic depth in training only (either grad mode, the reference's per-layer rates and random draws, drawn after the
patch-dropping draws)."""
import warnings
from typing import Any, Callable, Optional, Tuple, Union

import torch
from torch import nn, Tensor

from ...engine import _RuntimeOwner
from ..layers.patch_embedding import PatchEmbeddings
from ..layers.transformer import TransformerEncoder, TransformerOutput


class VisionTransformer(_RuntimeOwner):
    def __init__(self, embeddings: nn.Module, encoder: nn.Module, pooler: Optional[nn.Module] = None,
                 weight_init_fn: Optional[Callable] = None) -> None:
        super().__init__()
        self.embeddings = embeddings
        self.encoder = encoder
        self.pooler = pooler
        if weight_init_fn:
            self.apply(weight_init_fn)

    def forward(self, images: Tensor, image_patches_mask: Optional[Tensor] = None,
                attention_mask: Optional[Tensor] = None) -> TransformerOutput:
        if attention_mask is not None:
            raise NotImplementedError("attention_mask on the vision encoder is not on the accelerated path")
        emb = self.embeddings
        _, _, height, width = images.shape
        if height != emb.image_size[0] or width != emb.image_size[1]:
            raise ValueError(f"Input image size ({height}*{width}) doesn't match image size \
                {emb.image_size[0]}*{emb.image_size[1]} expected by model")
        if image_patches_mask is not None and emb.mask_token is None:
            warnings.warn("image_patches_mask passed but use_image_masking in init was false. Ignoring.")
        from ...engine import run, wants_grad
        if wants_grad(self):   # training: forward keeps activations, the autograd node carries the explicit backward
            hidden = []
            (last,) = run(self._runtime(), (images, image_patches_mask, hidden), ())
            B, S, d = hidden[0].shape
            out = TransformerOutput(last_hidden_state=last.view(B, S, d), pooler_output=None, hidden_states=hidden,
                                    attentions=None)
        else:
            with torch.no_grad():
                out = self._runtime().infer(images, image_patches_mask)
        if self.pooler is not None:
            out = out._replace(pooler_output=self.pooler(out.last_hidden_state))
        return out


def _vit_runtime(mod):
    from ...engine_coca_train import VisionTrainRuntime
    return VisionTrainRuntime(mod)


VisionTransformer._runtime_cls = staticmethod(_vit_runtime)


def vision_transformer(*, patch_size: int, hidden_dim: int, dim_feedforward: int, n_layer: int, n_head: int,
                       image_size: Union[int, Tuple[int, int]] = 224, num_channels: int = 3,
                       activation: Callable[..., nn.Module] = nn.GELU, transformer_dropout: float = 0.0,
                       patch_embed_dropout_prob: float = 0.0, layer_norm_eps: float = 1e-6,
                       final_layer_norm_eps: Optional[float] = 1e-6, norm_first: bool = True,
                       include_cls_embed: bool = True, drop_path_rate: Optional[float] = None,
                       patch_drop_rate: Optional[Union[float, Tuple[float, float]]] = None,
                       pooler: Optional[nn.Module] = None, ckpt_path: str = None) -> VisionTransformer:
    if ckpt_path:
        raise NotImplementedError("checkpoint download needs network access; load a state_dict explicitly")
    image_embedding = PatchEmbeddings(image_size=image_size, patch_size=patch_size, hidden_size=hidden_dim,
                                      hidden_dropout_prob=patch_embed_dropout_prob, patch_drop_rate=patch_drop_rate,
                                      num_channels=num_channels, include_cls_embed=include_cls_embed)
    transformer_encoder = TransformerEncoder(n_layer=n_layer, d_model=hidden_dim, n_head=n_head,
                                             dim_feedforward=dim_feedforward, dropout=transformer_dropout,
                                             activation=activation, layer_norm_eps=layer_norm_eps, norm_first=norm_first,
                                             final_layer_norm_eps=final_layer_norm_eps, drop_path_rate=drop_path_rate)
    return VisionTransformer(embeddings=image_embedding, encoder=transformer_encoder, pooler=pooler)


def vit_b_16(pooler: Optional[nn.Module] = None, **kwargs: Any) -> VisionTransformer:
    return vision_transformer(patch_size=16, n_layer=12, n_head=12, hidden_dim=768, dim_feedforward=3072, pooler=pooler,
                              **kwargs)


def vit_b_32(pooler: Optional[nn.Module] = None, **kwargs: Any) -> VisionTransformer:
    return vision_transformer(patch_size=32, n_layer=12, n_head=12, hidden_dim=768, dim_feedforward=3072, pooler=pooler,
                              **kwargs)


def vit_l_16(pooler: Optional[nn.Module] = None, **kwargs: Any) -> VisionTransformer:
    return vision_transformer(patch_size=16, n_layer=24, n_head=16, hidden_dim=1024, dim_feedforward=4096, pooler=pooler,
                              **kwargs)


def vit_l_32(pooler: Optional[nn.Module] = None, **kwargs: Any) -> VisionTransformer:
    return vision_transformer(patch_size=32, n_layer=24, n_head=16, hidden_dim=1024, dim_feedforward=4096, pooler=pooler,
                              **kwargs)
