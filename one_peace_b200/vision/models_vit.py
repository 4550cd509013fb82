"""Drop-in for the ImageNet classifier of the vision branch, ``one_peace_vision/classification/models_vit.py`` (``OnePeaceViT``
and ``one_piece_g_256`` / ``_384`` / ``_448`` / ``_512``), run by that branch's ``main_ft.py``.

The module tree, parameter names, buffers and registration order are the reference's, so ``misc.load_model`` loads a
fine-tuned checkpoint strictly, ``main_ft.py`` loads a converted pretraining checkpoint after its own interpolation, and
``utils/lr_decay.param_groups_lrd`` assigns the same layer ids.  The arithmetic is the project's:

    hMLP stem, CLS + positions          autograd.ImageEmbedFn (three patch GEMMs)
    one relative-position table         shared by every layer: LUT form for S <= kernels.ATTN_TC_MAX_S, dense (H, S, S_pad) above
    40 encoder layers                   eval: TransformerEncoder.run_fused; training: autograd.run_encoder_stack (drop-path as
                                        transformer_layer.py's residual_connection, the table's gradient summed over the layers)
    head                                autograd_classify.VitHeadFn: mean over the patch rows + fc_norm (csrc/vit_head.cu), or
                                        encoder.layer_norm on the CLS row, then the head GEMM

``use_checkpoint`` is accepted; whether the training stack keeps its activations or recomputes each layer in the backward (the
reference's checkpointing) is decided by the project's activation policy (autograd.keep_activations: recompute when the
activations do not fit in half of the free memory; ``OPB_ACTIVATIONS=recompute`` forces it).

Refused in the constructor, as no recipe uses them: dropout, attention_dropout or activation_dropout > 0 (``main_ft.py``
defaults ``--dropout 0.0``), ``rp_bias=True`` and ``shared_rp_bias=False``.  An input whose side is not 16 * bucket_size raises
ValueError (the reference would fail on the positional table's shape).
"""
import torch
import torch.nn as nn

from .. import kernels as K
from .. import relpos
from ..adapter.image import hmlp_stem, hmlp_stem_tensors, image_lut_bias, make_image_bucket_position
from ..autograd import ImageEmbedFn, RelPosBiasFn, TrainBias, _pad8, run_encoder_stack
from ..autograd_classify import VitHeadFn
from ..components import Embedding, PackCache, bf16, f32
from ..transformer.transformer_encoder import TransformerEncoder
from ..transformer.transformer_layer import TransformerEncoderLayer
from ..unify_model_config import AdjustEncDecConfig

__all__ = ["OnePeaceViT", "one_piece_g_256", "one_piece_g_384", "one_piece_g_448", "one_piece_g_512"]


class ImageAdaptor(nn.Module):
    """Parameter holder of models_vit.py:102-169 (shared_rp_bias=True): hMLP stem, cls_embedding, pos_embed, rel_pos_table and
    the rp_bucket buffer."""

    def __init__(self, attention_heads, bucket_size, embed_dim):
        super().__init__()
        self.embed_images = hmlp_stem(embed_dim)
        scale = embed_dim ** -0.5
        self.cls_embedding = nn.Parameter(scale * torch.randn(1, 1, embed_dim))
        self.bucket_size = bucket_size
        self.pos_embed = nn.Parameter(scale * torch.randn(bucket_size ** 2 + 1, embed_dim))
        self.attention_heads = attention_heads
        num_rel_dis = (2 * bucket_size - 1) ** 2 + 3
        self.rel_pos_table = Embedding(num_rel_dis, attention_heads, zero_init=True)
        self.register_buffer("rp_bucket", make_image_bucket_position(bucket_size, num_rel_dis))
        self._lut_cache = relpos.LutCache()

    def forward(self, src_images, train):
        """-> (x fp32 [B, S, d], [bias]): a kernels.RelPosBias for the fused inference loop, or a TrainBias (dense table tracked
        by autograd, plus its LUT form when S <= kernels.ATTN_TC_MAX_S) for the training stack."""
        R = src_images.shape[-1]
        if src_images.dim() != 4 or src_images.shape[-2] != R or R != 16 * self.bucket_size:
            raise ValueError(f"OnePeaceViT with bucket_size {self.bucket_size} takes [B, 3, {16 * self.bucket_size}, "
                             f"{16 * self.bucket_size}] images, got {tuple(src_images.shape)}")
        x = ImageEmbedFn.apply(src_images, self.pos_embed, *hmlp_stem_tensors(self.embed_images), self.cls_embedding)
        S = self.bucket_size ** 2 + 1
        H = self.attention_heads
        table = self.rel_pos_table.weight
        fast = image_lut_bias(self._lut_cache, table, self.rp_bucket, self.bucket_size) if S <= K.ATTN_TC_MAX_S else None
        if train:
            return x, [TrainBias(RelPosBiasFn.apply(table, self.rp_bucket, S, H), fast)]
        if fast is None:
            fast = K.RelPosBias(dense=K.relpos_bias_build(f32(table), self.rp_bucket, S, H))
        return x, [fast]


class VitEncoder(nn.Module):
    """Parameter holder of models_vit.py:300-361: `layers` (the project's TransformerEncoderLayer with the image FFN only) and
    `layer_norm` (a LayerNorm without global_pool, else an Identity).  The fused inference loop is TransformerEncoder's."""

    run_fused = TransformerEncoder.run_fused

    def __init__(self, cfg, global_pool, use_checkpoint):
        super().__init__()
        self.cfg = cfg
        self.global_pool = global_pool
        self.num_attention_heads = cfg.attention_heads
        self.use_checkpoint = use_checkpoint
        dpr = [v.item() for v in torch.linspace(0, cfg.drop_path_rate, cfg.layers, device="cpu")]     # also under a meta device
        self.layers = nn.ModuleList([TransformerEncoderLayer(cfg, drop_path_rate=dpr[i]) for i in range(cfg.layers)])
        self.num_layers = len(self.layers)
        self.layer_norm = nn.LayerNorm(cfg.embed_dim) if not global_pool else nn.Identity()


class OnePeaceViT(nn.Module):
    def __init__(self, activation_dropout=0.0, attention_dropout=0.0, attention_heads=24, bucket_size=16, dropout=0.0,
                 drop_path_rate=0.0, embed_dim=1536, ffn_embed_dim=6144, global_pool=True, init_scale=0.001, layers=40,
                 layer_scale_init_value=1e-2, num_classes=1000, rp_bias=False, shared_rp_bias=True, use_checkpoint=False):
        super().__init__()
        if dropout > 0 or attention_dropout > 0 or activation_dropout > 0:
            raise NotImplementedError("OnePeaceViT: dropout, attention_dropout and activation_dropout must be 0 "
                                      "(main_ft.py's default --dropout 0.0)")
        if rp_bias or not shared_rp_bias:
            raise NotImplementedError("OnePeaceViT: only the shared relative-position table (rp_bias=False, "
                                      "shared_rp_bias=True) of the one_piece_g_* variants is built")
        cfg = AdjustEncDecConfig(embed_dim=embed_dim, ffn_embed_dim=ffn_embed_dim, layers=layers, attention_heads=attention_heads,
                                 drop_path_rate=drop_path_rate, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                                 magneto_scale_attn=True, scale_attn=False, scale_fc=True, scale_heads=False,
                                 use_text_moe=False, use_image_moe=True, use_audio_moe=False, use_layer_scale=True,
                                 layer_scale_init_value=layer_scale_init_value)
        self.image_adapter = ImageAdaptor(attention_heads, bucket_size, embed_dim)
        self.encoder = VitEncoder(cfg, global_pool, use_checkpoint)
        self.global_pool = global_pool
        self.fc_norm = nn.LayerNorm(embed_dim) if global_pool else nn.Identity()
        self.head = nn.Linear(embed_dim, num_classes)
        nn.init.trunc_normal_(self.head.weight, std=.02)
        with torch.no_grad():
            self.head.weight.mul_(init_scale)
            self.head.bias.mul_(init_scale)
        self._head_cache = PackCache()

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"image_adapter.pos_embed", "image_adapter.cls_embedding"}

    def _head(self):
        norm = self.fc_norm if self.global_pool else self.encoder.layer_norm
        return norm, [norm.weight, norm.bias, self.head.weight, self.head.bias]

    def _head_pack(self):
        _, ps = self._head()

        def build():
            nw, nb, w, b = ps
            n_cls = w.shape[0]
            n_pad = _pad8(n_cls)
            wp = torch.zeros(n_pad, w.shape[1], dtype=torch.bfloat16, device=w.device)
            wp[:n_cls].copy_(bf16(w))
            bp = torch.zeros(n_pad, dtype=torch.float32, device=w.device)
            bp[:n_cls].copy_(f32(b))
            return dict(norm_w=f32(nw), norm_b=f32(nb), w=wp, b=bp, n_cls=n_cls)
        return self._head_cache.get(ps, build)

    def forward_features(self, src_images):
        """-> the last layer's residual stream fp32 [B, S, d] (before encoder.layer_norm, which the CLS head applies)."""
        train = self.training or (torch.is_grad_enabled() and (src_images.requires_grad or
                                                               any(p.requires_grad for p in self.parameters())))
        for layer in self.encoder.layers:
            layer.check_structure()
        x, bias = self.image_adapter(src_images, train)
        if train:
            return run_encoder_stack(self.encoder, x, bias, None, "image")
        B, S, d = x.shape
        self.encoder.run_fused(x.view(B * S, d), bias, None, B, S, "image")
        return x

    def forward(self, src_images):
        """-> logits fp32 [B, num_classes] (models_vit.py:436-439); autocast does not change them."""
        with torch.autocast("cuda", enabled=False):
            x = self.forward_features(src_images)
            norm, ps = self._head()
            return VitHeadFn.apply((self._head_pack(), self.global_pool, norm.eps), x, *ps)


def one_piece_g_256(**kwargs):
    return OnePeaceViT(bucket_size=16, rp_bias=False, shared_rp_bias=True, **kwargs)


def one_piece_g_384(**kwargs):
    return OnePeaceViT(bucket_size=24, rp_bias=False, shared_rp_bias=True, **kwargs)


def one_piece_g_448(**kwargs):
    return OnePeaceViT(bucket_size=28, rp_bias=False, shared_rp_bias=True, **kwargs)


def one_piece_g_512(**kwargs):
    return OnePeaceViT(bucket_size=32, rp_bias=False, shared_rp_bias=True, **kwargs)
