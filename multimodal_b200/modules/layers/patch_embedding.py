"""`PatchEmbeddings` — parameter container mirroring torchmultimodal/modules/layers/patch_embedding.py:25-157
(conv projection with truncated-normal init, optional CLS token, position embeddings, optional mask token).  Executed
by `engine_coca_train.VisionTrainRuntime` as im2col + wgmma GEMM + one token-assembly kernel.  Random patch dropping
(`patch_drop_rate`: a float drops that share of the patches per sample, a (rate_h, rate_w) tuple drops whole patch rows
and columns; FLIP, arXiv 2212.00794) applies in training only: the keep indices come from
`modules/masking/random_masking.py` with the reference's random draws, and only the kept patches are embedded, by
gathered im2col and token-assembly kernels, so the encoder runs on the shortened sequence.  `hidden_dropout_prob` must
be 0."""
import math
from typing import Any, NamedTuple, Optional, Tuple, Union

import torch
from torch import nn, Tensor

from ..._lib import MMBError


class PatchEmbeddingsOutput(NamedTuple):
    embeddings: Tensor
    random_mask: Optional[Tensor] = None
    ids_restore: Optional[Tensor] = None


class PatchEmbeddings(nn.Module):
    def __init__(self, image_size: Union[int, Tuple[int, int]] = 224, patch_size: int = 16, num_channels: int = 3,
                 hidden_size: int = 768, hidden_dropout_prob: float = 0.0, use_image_masking: bool = False,
                 patch_drop_rate: Optional[Union[float, Tuple[float, float]]] = None,
                 include_cls_embed: bool = True) -> None:
        super().__init__()
        if isinstance(image_size, int):
            image_size = (image_size, image_size)
        if image_size[0] % patch_size != 0 or image_size[1] % patch_size != 0:
            raise ValueError("Image size needs to be divisible by patch size")
        if num_channels != 3:
            raise NotImplementedError("the im2col kernel is specialised for 3-channel images")
        if hidden_dropout_prob != 0.0:
            raise NotImplementedError("dropout is not on the accelerated path")
        self.num_patches_h = image_size[0] // patch_size
        self.num_patches_w = image_size[1] // patch_size
        num_patches = self.num_patches_h * self.num_patches_w
        self.include_cls_embed = include_cls_embed
        if self.include_cls_embed:
            self.cls_token = nn.Parameter(torch.zeros(1, 1, hidden_size))
            num_patches = num_patches + 1
        self.conv_projection = nn.Conv2d(num_channels, hidden_size, kernel_size=patch_size, stride=patch_size)
        self._init_conv_weights()
        self.image_size: Tuple[int, int] = image_size
        self.position_embeddings = nn.Parameter(torch.zeros(1, num_patches, hidden_size))
        self.dropout = nn.Dropout(hidden_dropout_prob)
        if use_image_masking:
            self.mask_token = nn.Parameter(torch.zeros(1, 1, hidden_size))
        else:
            self.mask_token = None
        self.patch_drop_rate = patch_drop_rate

    def _init_conv_weights(self) -> None:
        fan_in = (self.conv_projection.in_channels * self.conv_projection.kernel_size[0]
                  * self.conv_projection.kernel_size[1])
        nn.init.trunc_normal_(self.conv_projection.weight, std=math.sqrt(1 / fan_in))
        assert self.conv_projection.bias is not None
        nn.init.zeros_(self.conv_projection.bias)

    def forward(self, image: Tensor, image_patches_mask: Optional[Tensor] = None) -> PatchEmbeddingsOutput:
        """Standalone forward (values only): im2col + wgmma GEMM + token assembly, as inside VisionTransformer; with
        patch dropping in training, random_mask / ids_restore as the reference returns them."""
        from ...engine_layers import patch_embeddings_forward

        return patch_embeddings_forward(self, image, image_patches_mask)
