"""FLAVA image encoder — drop-in for torchmultimodal/models/flava/image_encoder.py:28-278 (`PatchEmbeddings`,
`ImageEmbeddings`, `ImageTransformer`, `flava_image_encoder`).  Same constructors / state-dict keys / init; the forward
is `engine_flava_train.FlavaImageTrainRuntime` (im2col + wgmma GEMM patch embedding, fused token assembly, fused layer stack).
Position-embedding interpolation (image_encoder.py:103-137) is out of scope (fixed 224x224 pre-training resolution)."""
import warnings
from functools import partial
from typing import Any, Callable, Optional, Tuple

import torch
from torch import nn, Tensor

from ..._lib import MMBError
from ...engine import _RuntimeOwner
from ...modules.layers.normalizations import Fp32LayerNorm
from ...modules.layers.transformer import TransformerOutput
from ...modules.losses.flava import Pooler
from .transformer import init_transformer_weights, TransformerEncoder


def to_2tuple(x: int) -> Tuple[int, int]:
    return (x, x)


class PatchEmbeddings(nn.Module):
    def __init__(self, image_size: int = 224, patch_size: int = 16, num_channels: int = 3, embed_dim: int = 768) -> None:
        super().__init__()
        if num_channels != 3:
            raise NotImplementedError("the im2col kernel is specialised for 3-channel images")
        image_size, patch_size = to_2tuple(image_size), to_2tuple(patch_size)
        self.image_size, self.patch_size = image_size, patch_size
        self.num_patches = (image_size[1] // patch_size[1]) * (image_size[0] // patch_size[0])
        self.projection = nn.Conv2d(num_channels, embed_dim, kernel_size=self.patch_size, stride=self.patch_size)

    def forward(self, *args: Any, **kwargs: Any) -> Tensor:
        raise MMBError("PatchEmbeddings runs inside ImageTransformer's fused runtime; not a standalone op here")


class ImageEmbeddings(nn.Module):
    def __init__(self, image_size: int = 224, patch_size: int = 16, num_channels: int = 3, hidden_size: int = 768,
                 hidden_dropout_prob: float = 0.0, use_image_masking: bool = True) -> None:
        super().__init__()
        self.cls_token = nn.Parameter(torch.zeros(1, 1, hidden_size))
        self.patch_embeddings = PatchEmbeddings(image_size=image_size, patch_size=patch_size, num_channels=num_channels,
                                                embed_dim=hidden_size)
        num_patches = self.patch_embeddings.num_patches
        self.position_embeddings = nn.Parameter(torch.zeros(1, num_patches + 1, hidden_size))
        self.dropout = nn.Dropout(hidden_dropout_prob)
        if use_image_masking:
            self.mask_token = nn.Parameter(torch.zeros(1, 1, hidden_size))
        else:
            self.mask_token = None

    def forward(self, *args: Any, **kwargs: Any) -> Tensor:
        raise MMBError("ImageEmbeddings runs inside ImageTransformer's fused runtime; not a standalone op here")


class ImageTransformer(_RuntimeOwner):
    def __init__(self, embeddings: nn.Module, encoder: nn.Module, layernorm: nn.Module, pooler: nn.Module,
                 weight_init_fn: Optional[Callable] = None, initializer_range: float = 0.02, **kwargs: Any) -> None:
        super().__init__()
        self.embeddings = embeddings
        self.encoder = encoder
        self.layernorm = layernorm
        self.pooler = pooler
        if weight_init_fn is None:
            weight_init_fn = partial(init_transformer_weights, initializer_range=initializer_range)
        self.apply(weight_init_fn)

    def forward(self, pixel_values: Optional[Tensor] = None, image_patches_mask: Optional[Tensor] = None,
                attention_mask: Optional[Tensor] = None) -> TransformerOutput:
        if pixel_values is None:
            raise ValueError("You have to specify pixel_values")
        if attention_mask is not None:
            raise NotImplementedError("attention_mask on the image encoder is not on the accelerated path")
        pe = self.embeddings.patch_embeddings
        _, _, height, width = pixel_values.shape
        if height != pe.image_size[0] or width != pe.image_size[1]:
            raise ValueError(
                f"Input image size ({height}*{width}) doesn't match model ({pe.image_size[0]}*{pe.image_size[1]}).")
        if image_patches_mask is not None and self.embeddings.mask_token is None:
            warnings.warn("image_patches_mask passed but use_image_masking in init was false. Ignoring.")
        from ... import engine_flava_train as T
        from ...engine import wants_grad
        if wants_grad(self):   # training: forward keeps activations, autograd nodes carry the explicit backward
            if getattr(self, "output_attentions", False):
                raise NotImplementedError("attention probabilities are not produced by the training forward")
            return T.encoder_output(self._runtime(), (pixel_values, image_patches_mask), (), self.pooler)
        with torch.no_grad():
            return self._runtime().infer(pixel_values, image_patches_mask,
                                         want_attn=bool(getattr(self, "output_attentions", False)))


def _img_runtime(mod):
    from ...engine_flava_train import FlavaImageTrainRuntime
    return FlavaImageTrainRuntime(mod)


ImageTransformer._runtime_cls = staticmethod(_img_runtime)


def flava_image_encoder(hidden_size: int = 768, num_attention_heads: int = 12, num_hidden_layers: int = 12,
                        use_image_masking: bool = False, dropout: float = 0.0, intermediate_size: int = 3072,
                        intermediate_activation: Callable[..., nn.Module] = nn.GELU, layer_norm_eps: float = 1e-12,
                        image_size: int = 224, patch_size: int = 16, num_channels: int = 3) -> ImageTransformer:
    embeddings = ImageEmbeddings(image_size=image_size, patch_size=patch_size, num_channels=num_channels,
                                 hidden_size=hidden_size, hidden_dropout_prob=dropout,
                                 use_image_masking=use_image_masking)
    encoder = TransformerEncoder(n_layer=num_hidden_layers, d_model=hidden_size, n_head=num_attention_heads,
                                 dim_feedforward=intermediate_size, activation=intermediate_activation,
                                 layer_norm_eps=layer_norm_eps, dropout=dropout, norm_first=True)
    layernorm = Fp32LayerNorm(hidden_size, eps=layer_norm_eps)
    pooler = Pooler(hidden_size=hidden_size)
    return ImageTransformer(embeddings=embeddings, encoder=encoder, layernorm=layernorm, pooler=pooler)
