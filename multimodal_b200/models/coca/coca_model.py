"""CoCa — drop-in for torchmultimodal/models/coca/coca_model.py:27-460 (`MultimodalOutput`, `CoCaModel`, `coca_vit`,
`coca_vit_b_32`, `coca_vit_l_14`, `CoCaForPretraining`, `coca_for_pretraining`): same builders / kwargs / state-dict
schema / init order.  Forward only (BASELINE.json config 5 is a parity case in this round): every submodule runs on
the fused kernel stack (engine_coca_train.py); `CoCaForPretraining` returns the contrastive loss from the fused
`ContrastiveLossWithTemperature` and the captioning cross-entropy from `mmb_ce_labels`."""
import math
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Tuple, Union

import torch
from torch import nn, Tensor

from ... import ops
from ..._lib import MMBError
from ...modules.encoders.vision_transformer import vision_transformer
from ...modules.layers.attention_pooler import AttentionPooler, CascadedAttentionPooler
from ...modules.layers.transformer import TransformerOutput
from ...modules.losses.contrastive_loss_with_temperature import ContrastiveLossWithTemperature
from .multimodal_decoder import CoCaMultimodalDecoder
from .text_decoder import CoCaTextDecoder


class MultimodalOutput(NamedTuple):
    image_pooled_output: Tensor
    text_pooled_output: Tensor
    multimodal_embeddings: Tensor
    multimodal_pooled_embeddings: Optional[Tensor] = None


def _l2_normalize(x: Tensor) -> Tensor:
    """F.normalize(x, dim=-1) (eps 1e-12) on the fused kernel."""
    if torch.is_grad_enabled() and x.requires_grad:
        from ...autograd import l2_normalize
        return l2_normalize(x.float())
    x = x.contiguous().float()
    y = torch.empty_like(x)
    ops.l2norm_fwd(x, y, None, None, x.shape[0], x.shape[1])
    return y


class TrainHidden(NamedTuple):
    """Third field of `MultimodalOutput` on CoCaForPretraining's training path: the multimodal decoder's hidden states
    [B, S, d] (autograd history) and its vocabulary projection, consumed by the fused Linear -> CrossEntropy node."""
    hidden: Tensor
    projection: nn.Module


class CoCaModel(nn.Module):
    def __init__(self, vision_encoder: nn.Module, text_decoder: CoCaTextDecoder, multimodal_decoder: CoCaMultimodalDecoder,
                 vision_pooler: nn.Module, vision_proj: nn.Module):
        super().__init__()
        self.vision_encoder = vision_encoder
        self.text_decoder = text_decoder
        self.multimodal_decoder = multimodal_decoder
        self.vision_pooler = vision_pooler
        self.vision_proj = vision_proj
        self._proj_rt = None

    def forward(self, images: Tensor, texts: Tensor, text_padding_mask: Optional[Tensor] = None) -> MultimodalOutput:
        return self._forward_impl(images, texts, text_padding_mask, want_logits=True)

    def _forward_impl(self, images: Tensor, texts: Tensor, text_padding_mask: Optional[Tensor], want_logits: bool):
        """want_logits=False (CoCaForPretraining): the multimodal decoder stops before its vocabulary projection and the
        third field is (hidden bf16 [B*S, d], projection weight bf16 [V, d]) for the fused Linear -> CrossEntropy."""
        vision_encoder_outs = self.vision_encoder(images)
        if isinstance(vision_encoder_outs, TransformerOutput):
            image_embeddings = vision_encoder_outs.last_hidden_state
        elif isinstance(vision_encoder_outs, tuple):
            image_embeddings = vision_encoder_outs[0]
        else:
            image_embeddings = vision_encoder_outs
        assert isinstance(image_embeddings, Tensor), "Image embeddings must be Tensor"

        pooled_outputs = self.vision_pooler(image_embeddings)
        if isinstance(pooled_outputs, (list, tuple)):
            assert len(pooled_outputs) == 2
            captioning_image_embeddings, contrastive_image_embeddings = pooled_outputs
        else:   # parallel pooler: query 0 is the contrastive one
            contrastive_image_embeddings, captioning_image_embeddings = pooled_outputs[:, 0], pooled_outputs[:, 1:]
        contrastive_image_embeddings = self._vision_proj(contrastive_image_embeddings)
        shape = contrastive_image_embeddings.shape   # [B, 1, d] with the cascaded pooler: the reference keeps the 1
        contrastive_image_embeddings = _l2_normalize(contrastive_image_embeddings.reshape(-1, shape[-1])).view(shape)

        pooled_text_embeddings, text_tokens = self.text_decoder(texts, text_padding_mask)
        contrastive_text_embeddings = _l2_normalize(pooled_text_embeddings)

        if want_logits or getattr(self.multimodal_decoder, "output_projection", None) is None:
            multimodal_embeddings = self.multimodal_decoder(text_tokens, captioning_image_embeddings)
        elif self.multimodal_decoder.wants_graph(text_tokens, captioning_image_embeddings):
            # training: hidden states with autograd history; CoCaForPretraining fuses projection + cross-entropy
            multimodal_embeddings = TrainHidden(
                self.multimodal_decoder.hidden_states(text_tokens, captioning_image_embeddings),
                self.multimodal_decoder.output_projection)
        else:
            multimodal_embeddings = self.multimodal_decoder._runtime().infer(text_tokens, captioning_image_embeddings,
                                                                             return_hidden=True)
        return MultimodalOutput(contrastive_image_embeddings, contrastive_text_embeddings, multimodal_embeddings)

    def _vision_proj(self, x: Tensor) -> Tensor:
        """self.vision_proj(x) for x [B, 1, d] or [B, d] (coca_model.py:115) as a wgmma GEMM, fp32 out."""
        from ...engine import _Shadows

        if torch.is_grad_enabled() and (x.requires_grad or self.vision_proj.weight.requires_grad):
            from ...engine_coca_train import linear_f32
            return linear_f32(x.float(), self.vision_proj)
        squeeze = x.dim() == 3
        B = x.shape[0]
        x2 = x.reshape(-1, x.shape[-1]).contiguous().float()
        if self._proj_rt is None or self._proj_rt.device != x.device:
            self._proj_rt = _Shadows(x.device)
        xb = ops.cast_bf16(x2)
        w = self._proj_rt.get("vproj", [self.vision_proj.weight])
        out = torch.empty((x2.shape[0], w.shape[0]), device=x.device, dtype=torch.float32)
        ops.gemm(xb, w, bias=self.vision_proj.bias, epilogue=ops.EPI_F32, out=out)
        return out.view(B, -1, w.shape[0]) if squeeze else out


def coca_vit(
    *,
    vision_patch_size: int, vision_dim_feedforward: int, vision_n_layer: int, vision_n_head: int,
    vocab_size: int, num_text_positions: int, text_hidden_dim: int, text_n_layer: int, text_n_head: int,
    text_dim_feedforward: int, text_output_dim: int,
    fusion_n_layer: int, fusion_n_head: int, fusion_dim_feedforward: int,
    pooler_input_embed_dim: int, pooler_output_embed_dim: int, pooler_n_head: int,
    image_size: Union[int, Tuple[int, int]] = 224, num_channels: int = 3,
    vision_activation: Callable[..., nn.Module] = nn.GELU, vision_transformer_dropout: float = 0.0,
    patch_embed_dropout_prob: float = 0.0, vision_layer_norm_eps: float = 1e-5,
    vision_final_layer_norm_eps: Optional[float] = None, vision_norm_first: bool = True,
    vision_include_cls_embed: bool = False, vision_drop_path_rate: Optional[float] = None,
    vision_patch_drop_rate: Optional[Union[float, Tuple[float, float]]] = None,
    pad_idx: Optional[int] = 0, text_embed_cls: bool = True, text_dropout: float = 0.0,
    text_activation: Callable[..., nn.Module] = nn.GELU, text_layer_norm_eps: float = 1e-5, text_norm_first: bool = True,
    text_final_layer_norm_eps: Optional[float] = 1e-5,
    fusion_dropout: float = 0.0, fusion_activation: Callable[..., nn.Module] = nn.GELU,
    fusion_layer_norm_eps: float = 1e-5, fusion_norm_first: bool = True,
    fusion_final_layer_norm_eps: Optional[float] = 1e-5, multimodal_output_projection_dim: Optional[int] = None,
    cascaded_pooler: bool = True, pooler_n_queries: int = 256, pooler_layer_norm_eps: float = 1e-5,
) -> CoCaModel:
    """Arguments and construction order as the reference (coca_model.py:133-373)."""
    attention_pooler: nn.Module
    if cascaded_pooler:
        captioning_pooler = AttentionPooler(input_embed_dim=pooler_input_embed_dim,
                                            output_embed_dim=pooler_output_embed_dim, n_head=pooler_n_head,
                                            n_queries=pooler_n_queries, layer_norm_eps=pooler_layer_norm_eps)
        contrastive_pooler = AttentionPooler(input_embed_dim=pooler_output_embed_dim,
                                             output_embed_dim=pooler_output_embed_dim, n_head=pooler_n_head, n_queries=1,
                                             layer_norm_eps=pooler_layer_norm_eps)
        attention_pooler = CascadedAttentionPooler([captioning_pooler, contrastive_pooler])
    else:
        attention_pooler = AttentionPooler(input_embed_dim=pooler_input_embed_dim,
                                           output_embed_dim=pooler_output_embed_dim, n_head=pooler_n_head,
                                           n_queries=pooler_n_queries + 1, layer_norm_eps=pooler_layer_norm_eps)
    vision_proj = nn.Linear(pooler_output_embed_dim, pooler_output_embed_dim, bias=False)
    nn.init.normal_(vision_proj.weight, std=pooler_input_embed_dim ** -0.5)
    vision_encoder = vision_transformer(
        patch_size=vision_patch_size, hidden_dim=pooler_input_embed_dim, dim_feedforward=vision_dim_feedforward,
        n_layer=vision_n_layer, n_head=vision_n_head, image_size=image_size, num_channels=num_channels,
        activation=vision_activation, transformer_dropout=vision_transformer_dropout,
        patch_embed_dropout_prob=patch_embed_dropout_prob, layer_norm_eps=vision_layer_norm_eps,
        final_layer_norm_eps=vision_final_layer_norm_eps, norm_first=vision_norm_first,
        include_cls_embed=vision_include_cls_embed, drop_path_rate=vision_drop_path_rate,
        patch_drop_rate=vision_patch_drop_rate)
    text_decoder = CoCaTextDecoder(
        vocab_size=vocab_size, num_positions=num_text_positions, embedding_dim=text_hidden_dim, n_layer=text_n_layer,
        n_head=text_n_head, dim_feedforward=text_dim_feedforward, output_dim=text_output_dim, pad_idx=pad_idx,
        embed_cls=text_embed_cls, dropout=text_dropout, activation=text_activation, layer_norm_eps=text_layer_norm_eps,
        norm_first=text_norm_first, final_layer_norm_eps=text_final_layer_norm_eps)
    mm_input_seq_len = num_text_positions - 1 if text_embed_cls else num_text_positions
    multimodal_decoder = CoCaMultimodalDecoder(
        input_seq_len=mm_input_seq_len, text_embedding_dim=pooler_output_embed_dim, n_layer=fusion_n_layer,
        n_head=fusion_n_head, dim_feedforward=fusion_dim_feedforward, output_dim=multimodal_output_projection_dim,
        dropout=fusion_dropout, activation=fusion_activation, layer_norm_eps=fusion_layer_norm_eps,
        norm_first=fusion_norm_first, final_layer_norm_eps=fusion_final_layer_norm_eps)
    return CoCaModel(vision_encoder=vision_encoder, text_decoder=text_decoder, multimodal_decoder=multimodal_decoder,
                     vision_proj=vision_proj, vision_pooler=attention_pooler)


def coca_vit_b_32() -> CoCaModel:
    return coca_vit(vision_patch_size=32, vision_n_layer=12, vision_n_head=12, vision_dim_feedforward=3072,
                    vision_include_cls_embed=False, vocab_size=49408, num_text_positions=77, text_hidden_dim=512,
                    text_n_layer=12, text_n_head=8, text_dim_feedforward=2048, text_output_dim=512, fusion_n_layer=12,
                    fusion_n_head=8, fusion_dim_feedforward=2048, multimodal_output_projection_dim=49408,
                    pooler_input_embed_dim=768, pooler_output_embed_dim=512, pooler_n_head=8, cascaded_pooler=True)


def coca_vit_l_14() -> CoCaModel:
    return coca_vit(vision_patch_size=14, vision_n_layer=24, vision_n_head=16, vision_dim_feedforward=4096,
                    vision_include_cls_embed=False, vocab_size=49408, num_text_positions=77, text_hidden_dim=768,
                    text_n_layer=12, text_n_head=12, text_dim_feedforward=3072, text_output_dim=768, fusion_n_layer=12,
                    fusion_n_head=12, fusion_dim_feedforward=3072, multimodal_output_projection_dim=49408,
                    pooler_input_embed_dim=1024, pooler_output_embed_dim=768, pooler_n_head=8, cascaded_pooler=True)


class CoCaForPretraining(nn.Module):
    """coca_model.py:398-454: contrastive + captioning losses on top of CoCaModel.  Grad mode on + trainable parameters:
    both losses carry an autograd graph (engine_coca_train.py); under torch.no_grad(): forward values."""

    def __init__(self, model: CoCaModel, pad_idx: int = 0, contrastive_logit_scale_min: Optional[float] = math.log(1.0),
                 contrastive_logit_scale_max: Optional[float] = math.log(100.0)):
        super().__init__()
        self.model = model
        self.contrastive_loss = ContrastiveLossWithTemperature(logit_scale_min=contrastive_logit_scale_min,
                                                               logit_scale_max=contrastive_logit_scale_max)
        self.caption_loss = nn.CrossEntropyLoss(ignore_index=pad_idx)

    def forward(self, images: Tensor, texts: Tensor, text_padding_mask: Optional[Tensor] = None) -> Dict[str, Tensor]:
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            return self._forward_train(images, texts, text_padding_mask)
        with torch.no_grad():
            return self._forward_values(images, texts, text_padding_mask)

    def _forward_train(self, images: Tensor, texts: Tensor, text_padding_mask: Optional[Tensor] = None) -> Dict[str, Tensor]:
        """Both losses with autograd history (every stack, the poolers and the vocabulary head have backward schedules:
        engine_coca_train.py)."""
        from ...engine_coca_train import linear_cross_entropy

        fused = isinstance(self.model, CoCaModel)
        model_outs = (self.model._forward_impl(images, texts, text_padding_mask, want_logits=False) if fused
                      else self.model(images, texts, text_padding_mask))
        img = model_outs.image_pooled_output
        if img.dim() == 3:
            img = img.squeeze(1)
        contrastive_loss = self.contrastive_loss(img, model_outs.text_pooled_output)
        labels = texts[:, 1:].contiguous()              # captioning_labels (:443)
        mm = model_outs.multimodal_embeddings
        if isinstance(mm, TrainHidden):
            if mm.hidden.shape[:2] != labels.shape:
                raise ValueError(f"caption labels {tuple(labels.shape)} do not match the decoder output {tuple(mm.hidden.shape)}")
            captioning_loss = linear_cross_entropy(mm.hidden, mm.projection, labels, self.caption_loss.ignore_index)
        else:   # a model without a vocabulary projection of its own / a user-supplied model: logits arrive materialised
            from ...engine_flava_heads import cross_entropy
            captioning_loss = cross_entropy(mm.reshape(-1, mm.shape[-1]), labels.reshape(-1), self.caption_loss.ignore_index)
        return {"contrastive": contrastive_loss, "captioning": captioning_loss}

    def _forward_values(self, images: Tensor, texts: Tensor, text_padding_mask: Optional[Tensor] = None) -> Dict[str, Tensor]:
        fused = isinstance(self.model, CoCaModel)       # a user-supplied model only promises MultimodalOutput
        model_outs = (self.model._forward_impl(images, texts, text_padding_mask, want_logits=False) if fused
                      else self.model(images, texts, text_padding_mask))
        img = model_outs.image_pooled_output
        if img.dim() == 3:           # [B, 1, d] from the cascaded contrastive pooler
            img = img.squeeze(1)
        contrastive_loss = self.contrastive_loss(img, model_outs.text_pooled_output)
        labels = texts[:, 1:].contiguous()              # captioning_labels (:443)
        B, S = labels.shape
        acc = ops.zero_(torch.empty(2, device=labels.device, dtype=torch.float32))
        mm = model_outs.multimodal_embeddings
        if isinstance(mm, tuple):
            # fused vocabulary head (SURVEY §8 f3): hidden [B*S, d] x W[V, d]^T with the cross-entropy statistics taken
            # in the GEMM epilogue — the [B*S, 49 408] logits (7.7 GB fp32 at B = 512) are never written
            hidden, weight = mm
            if hidden.shape[0] != B * S:
                raise ValueError(f"caption labels {tuple(labels.shape)} do not match the decoder output rows {hidden.shape[0]}")
            ops.linear_cross_entropy(hidden, weight, labels.reshape(-1).to(torch.int32), self.caption_loss.ignore_index, acc)
        else:
            logits = mm
            if logits.shape[1] != S:
                raise ValueError(f"caption labels {tuple(labels.shape)} do not match logits {tuple(logits.shape)}")
            V = logits.shape[-1]
            ops.ce_labels(logits.reshape(B * S, V).contiguous().float(), labels.long().view(-1), 1,
                          self.caption_loss.ignore_index, B * S, V, None, acc)
        captioning_loss = acc[0] / acc[1]
        return {"contrastive": contrastive_loss, "captioning": captioning_loss}


def coca_for_pretraining(pad_idx: int = 0, **kwargs: Any) -> CoCaForPretraining:
    model = coca_vit(**kwargs)
    return CoCaForPretraining(model, pad_idx=pad_idx)
