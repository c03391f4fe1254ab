"""CLIP text encoder — drop-in for torchmultimodal/models/clip/text_encoder.py:15-134.

Same constructor signature / defaults, state-dict keys, CLIP initialisation (``initialize_parameters``), causal
``mask`` attribute and ``ValueError`` on a wrong context length.  The forward is ``engine.TextTower``: bit-exact
int64 token gather and EOT ``argmax`` select, causal attention, and only the EOT row goes through ``ln_final`` +
projection (the reference normalises all 77 rows and keeps one; same result).
"""
import torch
from torch import nn, Tensor
from torch.nn import TransformerEncoder, TransformerEncoderLayer

from ..._lib import MMBError
from ...autograd import autocast_out as _autocast_out
from ...engine import _RuntimeOwner, run, TextTower, wants_grad
from ...modules.layers.activation import SiLU
from ...modules.layers.normalizations import Fp32LayerNorm


class CLIPTextEncoder(_RuntimeOwner):
    """CLIP text encoder (Transformer with causal attention).

    Args: embedding_dim, context_length, vocab_size, width, dim_feedforward, heads, layers, use_clip_init
          (same meaning and defaults as the reference).
    Inputs: text (Tensor[int64] B x context_length, CUDA); return_hidden_state (bool).
    """

    _runtime_cls = TextTower
    TOKEN_EMBEDDING_INIT_STD = 0.02
    POS_EMBEDDING_INIT_STD = 0.01

    def __init__(self, embedding_dim: int = 512, context_length: int = 77, vocab_size: int = 49408, width: int = 512,
                 dim_feedforward: int = 2048, heads: int = 8, layers: int = 12, use_clip_init: bool = True):
        super().__init__()
        self.token_embedding = torch.nn.Embedding(vocab_size, width)
        self.positional_embedding = torch.nn.Parameter(torch.empty(context_length, width))
        encoder_layer = TransformerEncoderLayer(d_model=width, dim_feedforward=dim_feedforward, nhead=heads, dropout=0.0,
                                                activation=SiLU(), norm_first=True)
        self.encoder = TransformerEncoder(encoder_layer, num_layers=layers, enable_nested_tensor=False)
        self.width = width
        self.context_length = context_length
        self.ln_final = Fp32LayerNorm(width)
        self.projection = nn.Linear(width, embedding_dim, bias=False)
        self.mask = torch.full((self.context_length, self.context_length), float("-inf")).triu(1)
        if use_clip_init:
            self.initialize_parameters()

    def initialize_parameters(self) -> None:
        # text_encoder.py:82-104
        nn.init.normal_(self.token_embedding.weight, std=self.TOKEN_EMBEDDING_INIT_STD)
        nn.init.normal_(self.positional_embedding, std=self.POS_EMBEDDING_INIT_STD)
        proj_std = (self.width ** -0.5) * ((2 * self.encoder.num_layers) ** -0.5)
        attn_std = self.width ** -0.5
        fc_std = (2 * self.width) ** -0.5
        for layer in self.encoder.layers:
            nn.init.normal_(layer.self_attn.in_proj_weight, std=attn_std)
            nn.init.normal_(layer.self_attn.out_proj.weight, std=proj_std)
            nn.init.normal_(layer.linear1.weight, std=fc_std)
            nn.init.normal_(layer.linear2.weight, std=proj_std)
        nn.init.normal_(self.projection.weight, std=self.width ** -0.5)

    def build_attention_mask(self) -> Tensor:
        return torch.full((self.context_length, self.context_length), float("-inf")).triu(1)

    def forward(self, text: Tensor, return_hidden_state: bool = False) -> Tensor:
        if text.size(1) != self.context_length:
            raise ValueError(f"length of input should be {self.context_length} but found {text.size(1)}")
        if wants_grad(self):
            if return_hidden_state:
                # the [B, 77, width] hidden-state output is not on the contrastive path and has no backward schedule:
                # returning a detached tensor would silently drop the gradient, so refuse instead
                raise MMBError("CLIPTextEncoder(return_hidden_state=True) returns forward values only (no backward "
                               "schedule for the per-token output); call it under torch.no_grad()")
            (emb,) = run(self._runtime(), (text,))
        else:
            with torch.no_grad():
                emb = self._runtime().infer(text, return_hidden_state=return_hidden_state)
        return _autocast_out(emb)
