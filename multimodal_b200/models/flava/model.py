"""FLAVA model — drop-in for the encoder path of torchmultimodal/models/flava/model.py:36-298, 428-520
(`FLAVAOutput`, `flava_multimodal_encoder`, `FLAVAModel`, `flava_model`).  BASELINE.json config 3 ("FLAVA encoders
forward") is `FLAVAModel.forward`.  Pre-training / classification heads, losses and the DALL-E codebook
(model.py:301-420, 524-744) are outside SURVEY.md §8 and not provided.
"""
from collections import namedtuple
from functools import partial
from typing import Any, Callable, List, Optional, Tuple, Union

import torch
from torch import nn, Tensor

from ...modules.layers.normalizations import Fp32LayerNorm
from ...modules.layers.transformer import TransformerOutput
from ...modules.losses.flava import FLAVAPretrainingLoss, FLAVAPretrainingLossOutput, Pooler
from .image_encoder import flava_image_encoder
from .text_encoder import flava_text_encoder
from .transformer import FLAVATransformerWithoutEmbeddings, TransformerEncoder

FLAVAOutput = namedtuple(
    "FLAVAOutput",
    ["image", "image_masked", "text", "text_masked", "multimodal", "multimodal_masked", "projected_image_embeddings",
     "projected_text_embeddings"],
    defaults=(None, None, None, None, None, None, None, None),
)
FLAVAOutput.__annotations__ = {
    "image": TransformerOutput, "image_masked": TransformerOutput, "text": TransformerOutput,
    "text_masked": TransformerOutput, "multimodal": TransformerOutput, "multimodal_masked": TransformerOutput,
}


def flava_multimodal_encoder(hidden_size: int = 768, num_attention_heads: int = 12, num_hidden_layers: int = 12,
                             dropout: float = 0.0, intermediate_size: int = 3072,
                             intermediate_activation: Callable[..., nn.Module] = nn.GELU,
                             layer_norm_eps: float = 1e-12) -> FLAVATransformerWithoutEmbeddings:
    encoder = TransformerEncoder(n_layer=num_hidden_layers, d_model=hidden_size, n_head=num_attention_heads,
                                 dim_feedforward=intermediate_size, activation=intermediate_activation,
                                 layer_norm_eps=layer_norm_eps, dropout=dropout, norm_first=True)
    layernorm = Fp32LayerNorm(hidden_size, eps=layer_norm_eps)
    pooler = Pooler(hidden_size=hidden_size)
    return FLAVATransformerWithoutEmbeddings(encoder=encoder, layernorm=layernorm, pooler=pooler, hidden_size=hidden_size)


class FLAVAModel(nn.Module):
    def __init__(self, image_encoder: nn.Module, text_encoder: nn.Module, mm_encoder: nn.Module,
                 image_to_mm_projection: nn.Module, text_to_mm_projection: nn.Module, text_projection: nn.Module,
                 image_projection: nn.Module, **kwargs: Any) -> None:
        super().__init__()
        self.image_encoder = image_encoder
        self.text_encoder = text_encoder
        self.mm_encoder = mm_encoder
        self.image_to_mm_projection = image_to_mm_projection
        self.text_to_mm_projection = text_to_mm_projection
        self.text_projection = text_projection
        self.image_projection = image_projection

    def forward(self, image: Optional[Tensor] = None, text: Optional[Tensor] = None,
                image_patches_mask: Optional[Tensor] = None, text_masked: Optional[Tensor] = None,
                required_embedding: Optional[str] = None, skip_unmasked_mm_encoder: bool = True) -> FLAVAOutput:
        if required_embedding is None:
            if image is not None and text is not None:
                required_embedding = "mm"
            elif image is not None:
                required_embedding = "image"
            else:
                required_embedding = "text"

        # The encoders' outputs alias per-encoder workspaces; the unmasked results must survive the masked pass of
        # the same encoder, so they are snapshotted (one D2D copy of the hidden states) when a second pass follows.
        two_image_passes = image is not None and required_embedding in ("image", "mm")
        two_text_passes = text is not None and text_masked is not None and required_embedding in ("text", "mm")

        image_encoding_out = self._encode_data_to_embeddings(
            image, required_embedding, ["image", "mm"], partial(self.encode_image, projection=True))
        if len(image_encoding_out) == 2:
            image_outputs, projected_image_embeddings = image_encoding_out[0], image_encoding_out[1]
        else:
            image_outputs, projected_image_embeddings = image_encoding_out, None

        text_encoding_out = self._encode_data_to_embeddings(
            text, required_embedding, ["text", "mm"], partial(self.encode_text, projection=True))
        if len(text_encoding_out) == 2:
            text_outputs, projected_text_embeddings = text_encoding_out[0], text_encoding_out[1]
        else:
            text_outputs, projected_text_embeddings = text_encoding_out, None

        multimodal_outputs = TransformerOutput()
        multimodal_masked_outputs = TransformerOutput()
        if required_embedding == "mm" and not skip_unmasked_mm_encoder:
            # every encoder call returns freshly allocated tensors: the masked passes below do not disturb these
            multimodal_outputs = self.encode_mm(
                image_outputs.hidden_states[-1] if image_outputs.hidden_states else None,
                text_outputs.hidden_states[-1] if text_outputs.hidden_states else None)

        image_masked_outputs = self._encode_data_to_embeddings(
            image, required_embedding, ["image", "mm"],
            partial(self.encode_image, image_patches_mask=image_patches_mask))
        assert type(image_masked_outputs) == TransformerOutput
        text_masked_outputs = self._encode_data_to_embeddings(
            text_masked, required_embedding, ["text", "mm"], self.encode_text)
        assert type(text_masked_outputs) == TransformerOutput

        if required_embedding == "mm":
            multimodal_masked_outputs = self.encode_mm(
                image_masked_outputs.hidden_states[-1] if image_masked_outputs.hidden_states else None,
                text_masked_outputs.hidden_states[-1] if text_masked_outputs.hidden_states else None)

        return FLAVAOutput(image=image_outputs, image_masked=image_masked_outputs, text=text_outputs,
                           text_masked=text_masked_outputs, multimodal=multimodal_outputs,
                           multimodal_masked=multimodal_masked_outputs,
                           projected_image_embeddings=projected_image_embeddings,
                           projected_text_embeddings=projected_text_embeddings)

    def encode_image(self, image: Tensor, image_patches_mask: Optional[Tensor] = None, projection: bool = False
                     ) -> Union[Tuple[TransformerOutput, Tensor], Optional[TransformerOutput]]:
        if image_patches_mask is not None:
            encoded_image = self.image_encoder(image, image_patches_mask)
        else:
            encoded_image = self.image_encoder(image)
        if projection:
            projected_embeddings = self._project_cls(self.image_encoder, encoded_image, self.image_projection, "iproj")
            return encoded_image, projected_embeddings
        return encoded_image

    def set_output_attentions(self, flag: bool = True) -> "FLAVAModel":
        """The reference always returns `TransformerOutput.attentions` ([B, H, S, S] fp32 per layer).  Here they cost an
        extra kernel and 4*S*S bytes per head and layer, so they are opt-in: call this (or set `.output_attentions`
        on an individual encoder) to get them; otherwise `attentions` is None."""
        self.output_attentions = bool(flag)
        for enc in (self.image_encoder, self.text_encoder, self.mm_encoder):
            if enc is not None:
                enc.output_attentions = bool(flag)
        return self

    def encode_text(self, text: Tensor, text_mask: Optional[Tensor] = None, projection: bool = False
                    ) -> Union[Tuple[TransformerOutput, Tensor], Optional[TransformerOutput]]:
        encoded_text = self.text_encoder(input_ids=text, attention_mask=text_mask,
                                         return_attn_weights=bool(getattr(self, "output_attentions", False)),
                                         return_hidden_states=True)
        if projection:
            projected_embeddings = self._project_cls(self.text_encoder, encoded_text, self.text_projection, "tproj")
            return encoded_text, projected_embeddings
        return encoded_text

    @staticmethod
    def _project_cls(encoder: nn.Module, out: TransformerOutput, linear: nn.Module, key: str) -> Tensor:
        from ... import engine_flava_train as T
        from ...engine import wants_grad
        if torch.is_grad_enabled() and (out.last_hidden_state.requires_grad or wants_grad(linear)):
            return T.first_token_linear(out.last_hidden_state, linear)
        with torch.no_grad():
            return encoder._runtime().project_first_token(out.last_hidden_state, linear, key)

    def _encode_data_to_embeddings(self, data: Optional[Tensor], selected_head_encoder: str, encoder_options: List[str],
                                   encode_callable: Callable[..., Any]) -> Any:
        output: Any = TransformerOutput()
        if data is not None and selected_head_encoder in encoder_options:
            output = encode_callable(data)
        return output

    def encode_mm(self, image_embedding: Tensor, text_embedding: Tensor) -> TransformerOutput:
        if image_embedding is None or text_embedding is None:
            return TransformerOutput()
        from ... import engine_flava_train as T
        from ...engine import wants_grad
        enc, ip, tp = self.mm_encoder, self.image_to_mm_projection, self.text_to_mm_projection
        if wants_grad(enc, ip, tp) or (torch.is_grad_enabled() and
                                          (image_embedding.requires_grad or text_embedding.requires_grad)):
            return T.encoder_output(enc._runtime(ip, tp), (), (image_embedding, text_embedding), enc.pooler)
        with torch.no_grad():
            return enc._runtime(ip, tp).infer(image_embedding, text_embedding,
                                              want_attn=bool(getattr(enc, "output_attentions", False)))


class FLAVAForPreTraining(nn.Module):
    """torchmultimodal/models/flava/model.py:300-377: FLAVAModel + image codebook + FLAVAPretrainingLoss.
    `image_codebook` is any module mapping `image_for_codebook` to integer token ids per patch (the reference's
    DalleVAEEncoder needs the DALL_E package and a download; it is not part of this library)."""

    def __init__(self, model: FLAVAModel, image_codebook: nn.Module, loss: FLAVAPretrainingLoss) -> None:
        super().__init__()
        self.model = model
        self.image_codebook = image_codebook
        self.loss = loss

    def encode_image(self, image: Tensor, cls_index: int = 0) -> Tensor:
        return self.model.encode_image(image, projection=True)[1]

    def encode_text(self, text: Tensor, text_mask: Optional[Tensor] = None, cls_index: int = 0) -> Tensor:
        return self.model.encode_text(text, text_mask, projection=True)[1]

    def _codebook_labels(self, image_for_codebook: Tensor, patches_mask: Tensor):
        """Token id per patch from the codebook; unmasked patches get the ignore label -1 (model.py:347-351)."""
        keep = patches_mask.flatten(1).to(torch.bool)
        ids = self.image_codebook(image_for_codebook).flatten(1)
        ids[~keep] = -1
        return ids, keep

    def forward(self, image: Optional[Tensor] = None, text: Optional[Tensor] = None,
                image_for_codebook: Optional[Tensor] = None, image_patches_mask: Optional[Tensor] = None,
                text_masked: Optional[Tensor] = None, required_embedding: Optional[str] = None,
                skip_unmasked_mm_encoder: bool = True, itm_labels: Optional[Tensor] = None,
                mlm_labels: Optional[Tensor] = None) -> FLAVAPretrainingLossOutput:
        mim_labels = None
        if image_for_codebook is not None:
            mim_labels, image_patches_mask = self._codebook_labels(image_for_codebook, image_patches_mask)
        enc: FLAVAOutput = self.model(image=image, text=text, image_patches_mask=image_patches_mask,
                                      text_masked=text_masked, required_embedding=required_embedding,
                                      skip_unmasked_mm_encoder=skip_unmasked_mm_encoder)
        # last hidden state of every encoder pass -> the loss's *_sequence arguments (model.py:362-377)
        seq = {f"{name}_sequence": getattr(enc, name).last_hidden_state
               for name in ("image", "text", "image_masked", "text_masked", "multimodal_masked")}
        seq["multimodal_sequence"] = None if skip_unmasked_mm_encoder else enc.multimodal.last_hidden_state
        return self.loss(itm_labels=itm_labels, mim_labels=mim_labels, mlm_labels=mlm_labels,
                         projected_image_embeddings=enc.projected_image_embeddings,
                         projected_text_embeddings=enc.projected_text_embeddings, **seq)


def flava_model_for_pretraining(image_codebook: Optional[nn.Module] = None, codebook_image_size: int = 112,
                                pretrained: bool = False, **flava_model_kwargs: Any) -> FLAVAForPreTraining:
    """models/flava/model.py:524-551.  The reference builds a DalleVAEEncoder codebook (DALL_E package + download);
    here the caller passes the codebook module (any module producing integer token ids per patch)."""
    if image_codebook is None:
        raise NotImplementedError("flava_model_for_pretraining: pass image_codebook=<module>; the reference's "
                                  "DalleVAEEncoder needs the DALL_E package and a network download")
    model = flava_model(**flava_model_kwargs)
    hidden_size = flava_model_kwargs.get("multimodal_hidden_size", 768)
    losses = FLAVAPretrainingLoss(hidden_size=hidden_size)
    return FLAVAForPreTraining(model=model, image_codebook=image_codebook, loss=losses)


def flava_model(
    # Image encoder specific parameters
    image_hidden_size: int = 768, image_num_attention_heads: int = 12, image_num_hidden_layers: int = 12,
    image_dropout: float = 0.0, image_intermediate_size: int = 3072,
    image_intermediate_activation: Callable[..., nn.Module] = nn.GELU, image_layer_norm_eps: float = 1e-12,
    use_image_masking: bool = True, image_size: int = 224, patch_size: int = 16, num_channels: int = 3,
    # Text encoder specific parameters
    text_hidden_size: int = 768, text_num_attention_heads: int = 12, text_num_hidden_layers: int = 12,
    text_dropout: float = 0.0, text_intermediate_size: int = 3072,
    text_intermediate_activation: Callable[..., nn.Module] = nn.GELU, text_layer_norm_eps: float = 1e-12,
    vocab_size: int = 30522, pad_token_id: int = 0, type_vocab_size: int = 2, max_position_embeddings: int = 512,
    # Multimodal encoder specific parameters
    multimodal_hidden_size: int = 768, multimodal_num_attention_heads: int = 12, multimodal_num_hidden_layers: int = 6,
    multimodal_dropout: float = 0.0, multimodal_intermediate_size: int = 3072,
    multimodal_intermediate_activation: Callable[..., nn.Module] = nn.GELU, multimodal_layer_norm_eps: float = 1e-12,
    # projection
    text_and_image_proj_size: int = 768, pretrained: bool = False, **kwargs: Any,
) -> FLAVAModel:
    if pretrained:
        raise NotImplementedError("pretrained checkpoints need network access; load a state_dict explicitly "
                                  "(keys are identical to the reference's)")
    image_encoder = flava_image_encoder(
        hidden_size=image_hidden_size, num_attention_heads=image_num_attention_heads,
        num_hidden_layers=image_num_hidden_layers, use_image_masking=use_image_masking, dropout=image_dropout,
        intermediate_size=image_intermediate_size, intermediate_activation=image_intermediate_activation,
        layer_norm_eps=image_layer_norm_eps, image_size=image_size, patch_size=patch_size, num_channels=num_channels)
    text_encoder = flava_text_encoder(
        hidden_size=text_hidden_size, num_attention_heads=text_num_attention_heads,
        num_hidden_layers=text_num_hidden_layers, dropout=text_dropout, intermediate_size=text_intermediate_size,
        intermediate_activation=text_intermediate_activation, layer_norm_eps=text_layer_norm_eps, vocab_size=vocab_size,
        pad_token_id=pad_token_id, type_vocab_size=type_vocab_size, max_position_embeddings=max_position_embeddings)
    mm_encoder = flava_multimodal_encoder(
        hidden_size=multimodal_hidden_size, num_attention_heads=multimodal_num_attention_heads,
        num_hidden_layers=multimodal_num_hidden_layers, dropout=multimodal_dropout,
        intermediate_size=multimodal_intermediate_size, intermediate_activation=multimodal_intermediate_activation,
        layer_norm_eps=multimodal_layer_norm_eps)
    image_to_mm_projection = nn.Linear(image_hidden_size, multimodal_hidden_size)
    text_to_mm_projection = nn.Linear(text_hidden_size, multimodal_hidden_size)
    image_projection = nn.Linear(image_hidden_size, text_and_image_proj_size)
    text_projection = nn.Linear(text_hidden_size, text_and_image_proj_size)
    return FLAVAModel(image_encoder=image_encoder, text_encoder=text_encoder, mm_encoder=mm_encoder,
                      image_to_mm_projection=image_to_mm_projection, text_to_mm_projection=text_to_mm_projection,
                      text_projection=text_projection, image_projection=image_projection)
