"""Drop-in for ``OnePeacePretrainModel`` (models/one_peace/one_peace_pretrain.py:29-196), registered under the
reference's name ``one_peace_pretrain``: modality-shared encoder + lightweight decoder (d=768, 2 layers in the 4B
recipe, pretrain_vl_3B.yaml:151-168) with the mask-token canvas, the three contrastive projection heads and the
``*_mask_head`` / ``decoder_*_embed`` linears.  Same constructor, parameter names and ``forward`` contract:

    model(return_logit_scale=True)                                   -> exp(clamp(logit_scale))            (:123-127)
    model(src_tokens=..., encoder_type='text' | 'image' | 'audio')   -> (L2-normalised CLS logits, features)  (:162-173)
    model(..., encoder_type='vl' | 'al')                             -> (text features, image / audio features) (:174-177)
    model(..., *_preserve_ids=..., encoder_type=...)                 -> decoder features at every position    (:136-161)

Every arithmetic step is an sm_90a kernel behind the C-ABI, forward and backward (one_peace_b200/autograd.py for the
encoder and decoder layer stacks, autograd_general.py for the bias canvases, preserve_ids gathers, linears and the DCL loss).
"""
import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from .. import kernels as K
from ..components import Linear, PackCache, bf16, f32, trunc_normal_
from ..fairseq_compat import register_model
from ..unify_model_config import UnifyModelConfig
from .one_peace_base import ModelWrapper, OnePeaceBaseModel, init_one_peace_params


@dataclass
class OnePeacePretrainConfig(UnifyModelConfig):
    reset_logit_scale: bool = False
    logit_scale_init: float = 1 / 0.07
    stage2_pretrain: bool = False


@register_model("one_peace_pretrain", dataclass=OnePeacePretrainConfig)
class OnePeacePretrainModel(OnePeaceBaseModel):
    def __init__(self, cfg: OnePeacePretrainConfig, src_dict):
        super().__init__(cfg, src_dict)
        enc, dec = cfg.encoder, cfg.decoder
        enc_dim, dec_dim = enc.embed_dim, dec.embed_dim
        self.encoder_wrapper = ModelWrapper(enc, src_dict)
        self.decoder_wrapper = ModelWrapper(dec)
        self.logit_scale = nn.Parameter(torch.ones([]) * math.log(cfg.logit_scale_init))
        for m in ("text", "image", "audio"):                       # registration order = the reference's (:48-53)
            if getattr(enc, f"use_{m}_moe"):
                setattr(self, f"{m}_proj", Linear(enc_dim, enc_dim))
        for m in ("text", "image", "audio"):                       # :55-74
            setattr(self, f"{m}_mask_token", None)
            if getattr(enc, f"use_{m}_moe") and getattr(dec, f"use_{m}_moe"):
                setattr(self, f"decoder_{m}_embed", Linear(enc_dim, dec_dim))
                setattr(self, f"{m}_mask_token", nn.Parameter(torch.zeros(1, dec_dim)))
                setattr(self, f"{m}_mask_head", Linear(dec_dim, enc_dim))
                trunc_normal_(getattr(self, f"{m}_mask_token"))
        self.apply(init_one_peace_params)
        # activation checkpointing (:78-98) is the activation policy of the hand-written backward itself (one layer's
        # activations are recomputed while its adjoint runs), so there is nothing to wrap
        if cfg.stage2_pretrain:                                    # :100-106
            self.text_proj.requires_grad_(False)
            self.encoder_wrapper.requires_grad_(False)
            self.encoder_wrapper.audio_adapter.requires_grad_(True)
            self.encoder_wrapper.fusion_model.audio_layer_norm.requires_grad_(True)
            for layer in self.encoder_wrapper.fusion_model.layers:
                layer.audio_ffn.requires_grad_(True)
        self._proj_cache = {}

    def set_num_updates(self, num_updates):
        super().set_num_updates(num_updates)
        self.num_updates = num_updates

    # ------------------------------------------------------------------------------------------------
    def _linear(self, x, lin):
        """nn.Linear over the last dim through the wgmma GEMM, differentiable."""
        from ..autograd_general import LinearFn
        shp = x.shape
        y = LinearFn.apply(x.reshape(-1, shp[-1]), lin.weight, lin.bias)
        return y.view(*shp[:-1], lin.weight.shape[0])

    def _contrastive(self, encoder_type, **inputs):
        """(L2-normalised projection of the CLS feature, per-token features) of one single-modality encoder pass (:162-173)."""
        from ..autograd import HeadFn
        from ..autograd_general import FinalNormFn
        ew = self.encoder_wrapper
        fm = ew.fusion_model
        info = ew.adapt(encoder_type, **inputs)
        x, _ = fm.run_layers(info, encoder_type)                  # (B,S,d) fp32 before the modality's final LayerNorm
        B, S, d = x.shape
        ln = getattr(fm, f"{encoder_type}_layer_norm")
        proj = getattr(self, f"{encoder_type}_proj")
        if torch.is_grad_enabled() and (x.requires_grad or any(q.requires_grad for q in self.parameters())):
            logits = HeadFn.apply(x, ln.weight, ln.bias, proj.weight, proj.bias, ln.eps)
            feats = FinalNormFn.apply(x.reshape(B * S, d), ln.weight, ln.bias, ln.eps).view(B, S, d)
        else:
            feats = torch.empty_like(x)
            K.layernorm(x.view(B * S, d), f32(ln.weight), f32(ln.bias), feats.view(B * S, d), eps=ln.eps)
            cls = torch.empty(B, d, dtype=torch.bfloat16, device=x.device)
            K.row_gather(feats.view(B * S, d), torch.arange(B, device=x.device) * S, out=cls)
            cache = self._proj_cache.setdefault(encoder_type, PackCache())
            w, b = cache.get([proj.weight, proj.bias], lambda: (bf16(proj.weight), f32(proj.bias)))
            raw = torch.empty(B, w.shape[0], dtype=torch.float32, device=x.device)
            K.gemm(cls, w, K.EPI_STORE_F32, raw, bias=b)
            logits = K.l2_normalize_rows(raw)
        dt = proj.weight.dtype
        return logits.to(dt), feats.to(dt)

    def forward(self, src_tokens: Optional[torch.Tensor] = None, text_preserve_ids: Optional[torch.Tensor] = None,
                src_images: Optional[torch.Tensor] = None, image_preserve_ids: Optional[torch.Tensor] = None,
                src_audios: Optional[torch.Tensor] = None, audio_padding_masks: Optional[torch.Tensor] = None,
                audio_preserve_ids: Optional[torch.Tensor] = None, encoder_type: str = None,
                return_logit_scale: bool = False):
        if return_logit_scale:
            with torch.no_grad():
                self.logit_scale.clamp_(0, math.log(100))
            return self.logit_scale.exp()
        has_ids = text_preserve_ids is not None or image_preserve_ids is not None or audio_preserve_ids is not None
        if not has_ids and encoder_type in ("text", "image", "audio"):
            return self._contrastive(encoder_type, src_tokens=src_tokens, src_images=src_images, src_audios=src_audios,
                                     audio_padding_masks=audio_padding_masks)
        enc_t, enc_i, enc_a = self.encoder_wrapper(
            src_tokens=src_tokens, text_preserve_ids=text_preserve_ids, src_images=src_images,
            image_preserve_ids=image_preserve_ids, src_audios=src_audios, audio_padding_masks=audio_padding_masks,
            audio_preserve_ids=audio_preserve_ids, encoder_type=encoder_type)
        if not has_ids:
            if encoder_type == "vl":
                return enc_t, enc_i
            if encoder_type == "al":
                return enc_t, enc_a
            raise NotImplementedError
        emb_t = self._linear(enc_t, self.decoder_text_embed) if enc_t is not None else None
        emb_i = self._linear(enc_i, self.decoder_image_embed) if enc_i is not None else None
        emb_a = self._linear(enc_a, self.decoder_audio_embed) if enc_a is not None else None
        dec_t, dec_i, dec_a = self.decoder_wrapper(
            src_tokens=src_tokens, text_preserve_ids=text_preserve_ids, text_preserve_embed=emb_t,
            text_mask_token=self.text_mask_token, src_images=src_images, image_preserve_ids=image_preserve_ids,
            image_preserve_embed=emb_i, image_mask_token=self.image_mask_token, src_audios=src_audios,
            audio_padding_masks=audio_padding_masks, audio_preserve_ids=audio_preserve_ids, audio_preserve_embed=emb_a,
            audio_mask_token=self.audio_mask_token, encoder_type=encoder_type)
        dec_t = self._linear(dec_t, self.text_mask_head) if dec_t is not None else None
        dec_i = self._linear(dec_i, self.image_mask_head) if dec_i is not None else None
        dec_a = self._linear(dec_a, self.audio_mask_head) if dec_a is not None else None
        return dec_t, dec_i, dec_a

    @classmethod
    def build_model(cls, cfg, task):
        return cls(cfg, task.source_dictionary)

    def upgrade_state_dict_named(self, state_dict, name):
        """:179-196."""
        super().upgrade_state_dict_named(state_dict, name)
        if self.cfg.reset_logit_scale:
            state_dict.pop("logit_scale", None)
        if self.cfg.stage2_pretrain:
            for key in [k for k in state_dict if "image_" in k]:
                del state_dict[key]
        prefix = f"{name}." if name else ""
        for key, value in self.state_dict().items():
            state_dict.setdefault(prefix + key, value)
