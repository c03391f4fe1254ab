"""CLIP ViT image encoder — drop-in for torchmultimodal/models/clip/image_encoder.py:22-113.

Same constructor signature, same state-dict keys/shapes, same initialisation (the parameter containers are created
in the reference's order, so ``torch.manual_seed(s); CLIPViTEncoder(...)`` yields bit-identical weights), same
``ValueError``s.  The forward is NOT torch's layer stack: it is ``engine.ViTTower`` — im2col+GEMM patch embedding,
fused LayerNorm / QKV / attention / MLP kernels on Hopper tensor cores (see DESIGN.md).
"""
import torch
from torch import nn, Tensor

from ...autograd import autocast_out as _autocast_out
from ...engine import _RuntimeOwner, run, ViTTower, wants_grad
from ...modules.layers.activation import SiLU
from ...modules.layers.normalizations import Fp32LayerNorm

EXPANSION = 4


class CLIPViTEncoder(_RuntimeOwner):
    """Vision transformer encoder for CLIP.

    Args:
        embedding_dim (int): output (projection) dimension.
        patch_size (int): patch edge.
        image_size (int): input image edge (square).
        width (int): transformer width (multiple of 128, width / heads == 64).
        heads (int): attention heads.
        layers (int): transformer layers.

    Inputs: x (Tensor): B x 3 x image_size x image_size, CUDA.
    """

    _runtime_cls = ViTTower

    def __init__(self, embedding_dim: int, patch_size: int, image_size: int, width: int, heads: int, layers: int):
        super().__init__()
        # --- parameter containers, created in the reference's order (image_encoder.py:50-80) ---
        self.conv = nn.Conv2d(in_channels=3, out_channels=width, kernel_size=patch_size, stride=patch_size, bias=False)
        self.image_size = image_size
        scale = width ** -0.5
        self.cls_token_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((image_size // patch_size) ** 2 + 1, width))
        self.ln_pre = Fp32LayerNorm(width)
        encoder_layer = nn.TransformerEncoderLayer(d_model=width, nhead=heads, dropout=0.0, activation=SiLU(),
                                                   norm_first=True, dim_feedforward=EXPANSION * width, batch_first=True)
        self.encoder = nn.TransformerEncoder(encoder_layer, num_layers=layers, enable_nested_tensor=False)
        self.ln_post = Fp32LayerNorm(width)
        self.projection = nn.Parameter(scale * torch.randn(width, embedding_dim))

    def forward(self, x: Tensor) -> Tensor:
        if x.size(2) != self.image_size or x.size(3) != self.image_size:
            raise ValueError(
                f"Expected input with width and height as {self.image_size}, found {x.size(2)} by {x.size(3)} ")
        if x.size(1) != 3:
            raise ValueError(f"Expected 3 channels found {x.size(1)}")
        if wants_grad(self):   # training: forward keeps activations, the autograd node carries the explicit backward
            (emb,) = run(self._runtime(), (x,))
        else:
            with torch.no_grad():
                emb = self._runtime().infer(x)
        return _autocast_out(emb)
