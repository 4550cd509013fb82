"""Drop-in for ``OnePeaceClassifyModel`` (models/one_peace/one_peace_classify.py) with the attention-pooling head of
``OnePeaceClassifyHead`` (models/one_peace/one_peace_base.py:132-235) — the model of the VGGSound, FSD50K, VQA, NLVR2, AQA and
RefCOCO fine-tuning recipes.  Registered under the reference's name ``one_peace_classify``.

Parameter names and registration order are the reference's (classify_head first, then encoder_wrapper), so checkpoints and
utils/layer_decay.get_parameter_groups see the same model.  The head runs as one autograd node (autograd_classify.py).
Refused before any kernel runs, as no recipe uses them: attn_pooling=False (CLS-row head), pooler_dropout > 0 and
head_type='val'."""
import contextlib
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from ..autograd_classify import ClassifyHeadFn, head_pack, head_params
from ..autograd_general import FinalNormFn
from ..components import LayerNorm, Linear, PackCache, trunc_normal_
from ..fairseq_compat import register_model
from ..unify_model_config import UnifyModelConfig
from .one_peace_base import ModelWrapper, OnePeaceBaseModel, init_one_peace_params


@dataclass
class OnePeaceClassifyConfig(UnifyModelConfig):
    head_scale_ratio: int = 1
    use_pooler: bool = False
    pooler_dropout: float = 0.0
    attn_pooling: bool = False
    use_image_features: bool = False
    freeze_finetune_updates: int = 0


# modalities behind every head type (one_peace_classify.py:70-85)
_HEAD_MODALITIES = {"text": ("text",), "image": ("image",), "audio": ("audio",), "vl": ("text", "image"),
                    "al": ("text", "audio")}
_ALL_MODALITIES = ("text", "image", "audio")


class MultiheadAttentionPooling(nn.Module):
    """Parameter holder of one_peace_base.py:132-144 (k_proj without bias, v_proj and out_proj with bias, query q)."""

    def __init__(self, embed_dim, num_heads):
        super().__init__()
        self.embed_dim, self.num_heads, self.head_dim = embed_dim, num_heads, embed_dim // num_heads
        self.k_proj = Linear(embed_dim, embed_dim, bias=False)
        self.v_proj = Linear(embed_dim, embed_dim, bias=True)
        self.out_proj = Linear(embed_dim, embed_dim, bias=True)
        self.q = nn.Parameter(torch.zeros(1, 1, num_heads, self.head_dim))
        trunc_normal_(self.q)


class OnePeaceClassifyHead(nn.Module):
    """Parameter holder of one_peace_base.py:175-214 (attention pooling only)."""

    def __init__(self, use_pooler, pooler_dropout, input_dim, num_heads, head_scale_ratio, num_classes, use_two_images=False):
        super().__init__()
        self.attn_pooling = True
        self.norm = LayerNorm(input_dim)
        self.attn_pooling_func = MultiheadAttentionPooling(input_dim, num_heads)
        self.pooler = nn.Sequential(nn.Dropout(p=pooler_dropout), Linear(input_dim, input_dim), nn.Tanh(),
                                    nn.Dropout(p=pooler_dropout)) if use_pooler else None
        inner_dim = int(input_dim * head_scale_ratio)
        self.classifier = nn.Sequential(Linear(input_dim * 2 if use_two_images else input_dim, inner_dim), LayerNorm(inner_dim),
                                        nn.GELU(), Linear(inner_dim, num_classes))


@register_model("one_peace_classify", dataclass=OnePeaceClassifyConfig)
class OnePeaceClassifyModel(OnePeaceBaseModel):
    def __init__(self, cfg: OnePeaceClassifyConfig, src_dict, head_type, num_classes=None, use_two_images=False):
        if not cfg.attn_pooling:
            raise NotImplementedError("one_peace_classify: only the attention-pooling head (attn_pooling=True) is built")
        if cfg.pooler_dropout > 0:
            raise NotImplementedError("one_peace_classify: pooler_dropout > 0 is not supported")
        if head_type not in _HEAD_MODALITIES:
            raise NotImplementedError(f"one_peace_classify: head_type={head_type!r} is not supported "
                                      f"(one of {sorted(_HEAD_MODALITIES)})")
        super().__init__(cfg, src_dict)
        enc = cfg.encoder
        self.head_type = head_type
        self.num_classes = num_classes
        self.classify_head = OnePeaceClassifyHead(cfg.use_pooler, cfg.pooler_dropout, enc.embed_dim, enc.attention_heads,
                                                  cfg.head_scale_ratio, num_classes, use_two_images)
        self.modalities = _HEAD_MODALITIES[head_type]
        for m in _ALL_MODALITIES:
            setattr(enc, f"use_{m}_moe", m in self.modalities)
        self.encoder_wrapper = ModelWrapper(enc, src_dict, num_layers=enc.layers,
                                            **{f"use_{m}_norm": m in self.modalities for m in _ALL_MODALITIES})
        self.apply(init_one_peace_params)
        self._head_cache = PackCache()

    def set_num_updates(self, num_updates):
        super().set_num_updates(num_updates)
        self.num_updates = num_updates

    def _encode(self, encoder_type, src_tokens, src_images, src_audios, audio_padding_masks):
        """-> (features fp32 [B, S, d] after the final LayerNorm of the modality the head reads, its padding mask or None)
        (one_peace_classify.py:112-160: text unless use_image_features, else image, else audio)."""
        ew = self.encoder_wrapper
        fm = ew.fusion_model
        if encoder_type in ("text", "image", "audio"):
            info = ew.adapt(encoder_type, src_tokens=src_tokens, src_images=src_images, src_audios=src_audios,
                            audio_padding_masks=audio_padding_masks)
            x, pad = fm.run_layers(info, encoder_type)
            ln = getattr(fm, f"{encoder_type}_layer_norm")
            B, S, d = x.shape
            feats = FinalNormFn.apply(x.reshape(B * S, d), ln.weight, ln.bias, ln.eps).view(B, S, d)
            return feats, pad
        t, i, a, tp, ip, ap = ew(src_tokens=src_tokens, src_images=src_images, src_audios=src_audios,
                                 audio_padding_masks=audio_padding_masks, encoder_type=encoder_type, return_padding_mask=True)
        if t is not None and not self.cfg.use_image_features:
            return t, tp
        if i is not None:
            return i, ip
        return a, ap

    def forward(self, src_tokens: Optional[torch.Tensor] = None, src_images: Optional[torch.Tensor] = None,
                src_images_2: Optional[torch.Tensor] = None, src_audios: Optional[torch.Tensor] = None,
                audio_padding_masks: Optional[torch.Tensor] = None):
        """-> logits [B, num_classes] in the head's dtype (one_peace_classify.py:112-160)."""
        ft = self.cfg.freeze_finetune_updates <= self.num_updates if hasattr(self, "num_updates") else True
        with torch.no_grad() if not ft else contextlib.ExitStack():
            f1, pad = self._encode(self.head_type, src_tokens, src_images, src_audios, audio_padding_masks)
            f2 = None
            if src_images_2 is not None:
                f2, _ = self._encode(self.head_type, src_tokens, src_images_2, src_audios, audio_padding_masks)
        head = self.classify_head
        meta = (head_pack(head, self._head_cache), pad, head.norm.eps, head.classifier[1].eps)
        logits = ClassifyHeadFn.apply(meta, f1, f2, *head_params(head))
        return logits.to(head.classifier[3].weight.dtype)

    @classmethod
    def build_model(cls, cfg, task):
        cfg.encoder.image_adapter.rel_bucket_size = task.cfg.patch_image_size // 16
        return cls(cfg, task.source_dictionary, head_type=task.cfg.head_type, num_classes=task.cfg.num_classes,
                   use_two_images=task.cfg.use_two_images)

    def upgrade_state_dict_named(self, state_dict, name):
        """one_peace_classify.py:167-176 with the adapters' per-layer relative-position tables (adapter/text.py:166-185): a
        single table is copied to every layer; parameters absent from the checkpoint (a fresh head) keep their initial values."""
        super().upgrade_state_dict_named(state_dict, name)
        self.remove_pretraining_modules(state_dict)
        prefix = f"{name}." if name else ""
        for m in self.modalities:
            p = f"{prefix}encoder_wrapper.{m}_adapter."
            if p + "rel_pos_table.weight" in state_dict:
                state_dict[p + "rel_pos_table_list.0.weight"] = state_dict.pop(p + "rel_pos_table.weight")
            if p + "rel_pos_table_list.0.weight" in state_dict and p + "rel_pos_table_list.1.weight" not in state_dict:
                w = state_dict[p + "rel_pos_table_list.0.weight"]
                for i in range(len(getattr(self.encoder_wrapper, f"{m}_adapter").rel_pos_table_list)):
                    state_dict[f"{p}rel_pos_table_list.{i}.weight"] = w.clone()
        for key, value in self.state_dict().items():
            state_dict.setdefault(prefix + key, value)

    def remove_pretraining_modules(self, state_dict):
        """one_peace_classify.py:178-211: the *_proj heads, the unused modality norms, and every text_ / image_ / audio_ key of
        a modality this head type does not use."""
        for m in _ALL_MODALITIES:
            state_dict.pop(f"{m}_proj.weight", None)
            state_dict.pop(f"{m}_proj.bias", None)
        for m in _ALL_MODALITIES:
            if m not in self.modalities:
                for key in [k for k in state_dict if f"{m}_" in k]:
                    del state_dict[key]
