"""Drop-in for the semantic segmentation backbone of the vision branch,
``one_peace_vision/seg/mmseg_custom/models/backbones/onepeace_adapter.py`` (``OnePeaceAdapter``, the ViT-Adapter around
``onepeace.py``'s ``OnePeace``), as ``configs/ade20k/mask2former_onepeace_adapter_g_896_40k_ade20k_ss.py`` builds it.

The module tree, parameter and buffer names, shapes, dtypes and registration order are the reference's, so a checkpoint
saved from it loads strictly and ``init_weights()`` reads ``pretrained=`` as onepeace.py:547-578 does.  Every layer's
``rp_bucket`` is one tensor registered under all the layers' names.  Inference only (eval BatchNorm), on B images:

    SPM convs, BN, ReLU, max-pool   torch (cuDNN) in bf16 channels-last, each BN folded into its conv (cached per version)
    fc1..fc4                        GEMMs on the channels-last maps; fc2..fc4 add level_embed in their bias and write each
                                    level straight into its rows of c (fp32 [B * T, d], T = sum of the three level sizes)
    ViT stem                        autograd.image_stem: hMLP stem + CLS + pos_embed -> fp32 rows [B * (bucket^2 + 1), d]
    per interaction block           injector: x[patches] += gamma * MSDA(LN(x[patches]), LN(c)), the residual in
                                    output_proj's epilogue (rows remapped past the CLS rows); its layers through
                                    TransformerEncoder.run_fused, one LUT-form relative-position bias per layer;
                                    extractor(s): c += MSDA(LN(c), LN(x[patches])), c += fc2(dwconv_gelu(fc1(LN(c))))
    output maps                     the transposed conv as one GEMM with N = 4 d, then one csrc/seg.cu kernel per level
                                    sums c_l, the bilinear ViT term and (level 1) the transposed conv, applies the folded
                                    eval BatchNorm and writes fp32 NCHW

Refused in the constructor, as no segmentation config uses them: dropout, attention_dropout or activation_dropout > 0,
``rp_bias=False``, ``shared_rp_bias=True``, ``with_cffn=False``, ``add_vit_feature=False``, interaction_indexes that do
not split the layers into contiguous runs covering all of them, ``embed_dim * deform_ratio / deform_num_heads != 32``
and an odd bucket_size.  ``forward`` raises ValueError for an input that is not [B, 3, 16 bucket, 16 bucket], and NotImplementedError when a
gradient is required (no backward is built) or in train mode (the BatchNorms run only with their running statistics).
``rp_bucket`` stays one tensor when the module is moved or converted (``SegEncoder._apply``).
"""
import math
import pickle
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import kernels as K
from .. import relpos
from . import _get_rank, resize_abs_pos_embed
from .ms_deform_attn import MSDeformAttn, msda_forward, msda_pack
from ..adapter.image import (geometric_sequence_interpolation, hmlp_stem, hmlp_stem_tensors, image_lut_bias,
                             make_image_bucket_position)
from ..autograd import image_stem, pack_image_stem
from ..components import Embedding, PackCache, bf16, f32
from ..transformer.transformer_encoder import TransformerEncoder
from ..transformer.transformer_layer import TransformerEncoderLayer
from ..unify_model_config import AdjustEncDecConfig

try:  # pragma: no cover - mmseg is not installed in the build image
    from mmseg.models.builder import BACKBONES
    _register = BACKBONES.register_module()
except Exception:
    def _register(cls):
        return cls

__all__ = ["OnePeaceAdapter", "level_shapes", "reference_points", "fold_bn", "convt_weight"]

LN_EPS = 1e-6     # the adapter's LayerNorms (onepeace_adapter.py:49)


def level_shapes(side):
    """(H, W) of c2, c3, c4 for a bucket_size `side` (adapter_modules.py:25-44: h // 8, h // 16, h // 32 of a 16 side input)."""
    return [(2 * side, 2 * side), (side, side), (side // 2, side // 2)]


def reference_points(shapes):
    """adapter_modules.py:10-22: the cell centres (x, y) / (W, H) of every level, levels in order -> fp32 [sum H W, 2]."""
    out = []
    for h, w in shapes:
        y, x = torch.meshgrid(torch.linspace(0.5, h - 0.5, h, dtype=torch.float32),
                              torch.linspace(0.5, w - 0.5, w, dtype=torch.float32), indexing="ij")
        out.append(torch.stack((x.reshape(-1) / w, y.reshape(-1) / h), -1))
    return torch.cat(out, 0)


def fold_bn(bn):
    """Eval BatchNorm as (scale, shift) with y = x * scale + shift, computed in fp64."""
    scale = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    shift = bn.bias.detach().double() - bn.running_mean.detach().double() * scale
    return scale, shift


def convt_weight(w):
    """ConvTranspose2d(d, d, 2, 2) weight [c_in, c_out, dy, dx] as a GEMM weight [(dy, dx, c_out), c_in]."""
    return w.permute(2, 3, 1, 0).reshape(4 * w.shape[1], w.shape[0])


class ImageAdaptor(nn.Module):
    """onepeace.py:112-185 with shared_rp_bias=False: hMLP stem, cls_embedding, pos_embed."""

    def __init__(self, attention_heads=24, bucket_size=16, embed_dim=1536, dropout=0.0, shared_rp_bias=False):
        super().__init__()
        self.bucket_size = bucket_size
        self.dropout = nn.Dropout(dropout)
        self.embed_images = hmlp_stem(embed_dim)
        scale = embed_dim ** -0.5
        self.cls_embedding = nn.Parameter(scale * torch.randn(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(scale * torch.randn(bucket_size ** 2 + 1, embed_dim))
        self.shared_rp_bias = shared_rp_bias
        self._stem_cache = PackCache()

    def stem(self, img):
        """hMLP stem + CLS + pos_embed (onepeace.py:166-181) -> fp32 [B * (bucket^2 + 1), d]."""
        stem = hmlp_stem_tensors(self.embed_images)
        pk = self._stem_cache.get(stem + [self.cls_embedding, self.pos_embed],
                                  lambda: dict(pack_image_stem(*stem), pos=f32(self.pos_embed),
                                               cls=f32(self.cls_embedding).view(-1)))
        x = image_stem(pk, img, pk["pos"], pk["cls"])[0]
        return x.view(-1, x.shape[-1])


class SegLayer(TransformerEncoderLayer):
    """onepeace.py:235-308 with rp_bias=True: the project's layer with its own rel_pos_table, modules registered in the
    reference's order (final_layer_norm before image_ffn)."""

    def __init__(self, cfg, drop_path_rate, bucket_size, rp_bucket):
        super().__init__(cfg, drop_path_rate=drop_path_rate)
        self._modules["image_ffn"] = self._modules.pop("image_ffn")
        self.rp_bias = True
        self.rel_pos_table = Embedding((2 * bucket_size - 1) ** 2 + 3, cfg.attention_heads, zero_init=True)
        self.register_buffer("rp_bucket", rp_bucket)
        self._lut_pack = PackCache()


class SegEncoder(nn.Module):
    """onepeace.py:311-366: the layers (one shared rp_bucket tensor); the fused inference loop is TransformerEncoder's."""

    def __init__(self, cfg, bucket_size):
        super().__init__()
        self.cfg = cfg
        self.bucket_size = bucket_size
        self.dropout_module = nn.Dropout(cfg.dropout)
        self.attention_heads = cfg.attention_heads
        self.num_attention_heads = cfg.attention_heads
        side = bucket_size
        rp_bucket = make_image_bucket_position(side, (2 * side - 1) ** 2 + 3)
        dpr = [v.item() for v in torch.linspace(0, cfg.drop_path_rate, cfg.layers, device="cpu")]
        self.layers = nn.ModuleList([SegLayer(cfg, dpr[i], side, rp_bucket) for i in range(cfg.layers)])
        self.num_layers = len(self.layers)
        self._lut_cache = relpos.LutCache()

    def _apply(self, fn, recurse=True):
        """Moves / converts the shared rp_bucket once and points every layer at the result: nn.Module._apply would give
        each layer its own copy (40 x 79 MB of int64 at 896^2)."""
        shared = [layer for layer in self.layers[1:] if layer._buffers.get("rp_bucket") is self.layers[0].rp_bucket]
        for layer in shared:
            layer._buffers["rp_bucket"] = None            # _apply skips None buffers
        try:
            super()._apply(fn, recurse)
        finally:
            for layer in shared:
                layer._buffers["rp_bucket"] = self.layers[0].rp_bucket
        return self

    def biases(self):
        """One LUT-form RelPosBias per layer, each rebuilt when its table changes."""
        side = self.bucket_size
        out = []
        for layer in self.layers:
            table, bucket = layer.rel_pos_table.weight, layer.rp_bucket
            out.append(layer._lut_pack.get([table], lambda: image_lut_bias(self._lut_cache, table, bucket, side)))
        return out

    def run_block(self, rows, lo, hi, biases, B, S):
        """TransformerEncoder.run_fused over layers lo..hi (inclusive)."""
        view = types.SimpleNamespace(layers=self.layers[lo:hi + 1], cfg=self.cfg, num_attention_heads=self.num_attention_heads)
        return TransformerEncoder.run_fused(view, rows, biases[lo:hi + 1], None, B, S, "image")


class DWConv(nn.Module):
    """adapter_modules.py:69-84: parameter holder of the depthwise 3x3 conv."""

    def __init__(self, dim):
        super().__init__()
        self.dwconv = nn.Conv2d(dim, dim, 3, 1, 1, bias=True, groups=dim)


class ConvFFN(nn.Module):
    """adapter_modules.py:47-84: fc1, the depthwise 3x3 conv (dwconv.dwconv), GELU, fc2."""

    def __init__(self, in_features, hidden_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.dwconv = DWConv(hidden_features)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_features, in_features)
        self.drop = nn.Dropout(0.0)


class Extractor(nn.Module):
    """adapter_modules.py:87-121 (with_cffn=True): c += MSDA(LN(c), LN(x)); c += ConvFFN(LN(c))."""

    def __init__(self, dim, num_heads, n_points, n_levels, deform_ratio, cffn_ratio):
        super().__init__()
        self.query_norm = nn.LayerNorm(dim, eps=LN_EPS)
        self.feat_norm = nn.LayerNorm(dim, eps=LN_EPS)
        self.attn = MSDeformAttn(d_model=dim, n_levels=n_levels, n_heads=num_heads, n_points=n_points, ratio=deform_ratio)
        self.with_cffn = True
        self.with_cp = False
        self.ffn = ConvFFN(dim, int(dim * cffn_ratio))
        self.ffn_norm = nn.LayerNorm(dim, eps=LN_EPS)
        self.drop_path = nn.Identity()
        self._ffn_pack = PackCache()

    def ffn_pack(self):
        f = self.ffn
        ps = [f.fc1.weight, f.fc1.bias, f.dwconv.dwconv.weight, f.dwconv.dwconv.bias, f.fc2.weight, f.fc2.bias]

        def build():
            w1, b1, dw, db, w2, b2 = ps
            return dict(w1=bf16(w1), b1=f32(b1), dw=f32(dw.reshape(dw.shape[0], 9).t()), db=f32(db), w2=bf16(w2), b2=f32(b2))
        return self._ffn_pack.get(ps, build)


class Injector(nn.Module):
    """adapter_modules.py:124-149: x += gamma * MSDA(LN(x), LN(c))."""

    def __init__(self, dim, num_heads, n_points, n_levels, deform_ratio, init_values):
        super().__init__()
        self.with_cp = False
        self.query_norm = nn.LayerNorm(dim, eps=LN_EPS)
        self.feat_norm = nn.LayerNorm(dim, eps=LN_EPS)
        self.attn = MSDeformAttn(d_model=dim, n_levels=n_levels, n_heads=num_heads, n_points=n_points, ratio=deform_ratio)
        self.gamma = nn.Parameter(init_values * torch.ones(dim), requires_grad=True)


class InteractionBlockWithCls(nn.Module):
    """adapter_modules.py:191-231."""

    def __init__(self, dim, num_heads, n_points, init_values, cffn_ratio, deform_ratio, extra_extractor):
        super().__init__()
        self.injector = Injector(dim, num_heads, n_points, 3, deform_ratio, init_values)
        self.extractor = Extractor(dim, num_heads, n_points, 1, deform_ratio, cffn_ratio)
        self.extra_extractors = nn.Sequential(*[Extractor(dim, num_heads, n_points, 1, deform_ratio, cffn_ratio)
                                                for _ in range(2)]) if extra_extractor else None


def _conv_bn_relu(cin, cout, stride):
    return [nn.Conv2d(cin, cout, kernel_size=3, stride=stride, padding=1, bias=False), nn.SyncBatchNorm(cout),
            nn.ReLU(inplace=True)]


class SpatialPriorModule(nn.Module):
    """adapter_modules.py:234-294."""

    def __init__(self, inplanes=64, embed_dim=384):
        super().__init__()
        self.with_cp = False
        self.stem = nn.Sequential(*(_conv_bn_relu(3, inplanes, 2) + _conv_bn_relu(inplanes, inplanes, 1) +
                                    _conv_bn_relu(inplanes, inplanes, 1) + [nn.MaxPool2d(kernel_size=3, stride=2, padding=1)]))
        self.conv2 = nn.Sequential(*_conv_bn_relu(inplanes, 2 * inplanes, 2))
        self.conv3 = nn.Sequential(*_conv_bn_relu(2 * inplanes, 4 * inplanes, 2))
        self.conv4 = nn.Sequential(*_conv_bn_relu(4 * inplanes, 4 * inplanes, 2))
        self.fc1 = nn.Conv2d(inplanes, embed_dim, kernel_size=1, stride=1, padding=0, bias=True)
        self.fc2 = nn.Conv2d(2 * inplanes, embed_dim, kernel_size=1, stride=1, padding=0, bias=True)
        self.fc3 = nn.Conv2d(4 * inplanes, embed_dim, kernel_size=1, stride=1, padding=0, bias=True)
        self.fc4 = nn.Conv2d(4 * inplanes, embed_dim, kernel_size=1, stride=1, padding=0, bias=True)
        self._pack = PackCache()

    def conv_pack(self):
        """Each (conv, BN) pair as a bf16 channels-last conv weight with the eval BN folded in, plus its fp32 bias."""
        pairs = [(s[i], s[i + 1]) for s, idx in ((self.stem, (0, 3, 6)), (self.conv2, (0,)), (self.conv3, (0,)),
                                                (self.conv4, (0,))) for i in idx]
        ps = [t for c, bn in pairs for t in (c.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var)]

        def build():
            out = []
            for c, bn in pairs:
                scale, shift = fold_bn(bn)
                w = (c.weight.detach().double() * scale.view(-1, 1, 1, 1)).to(torch.bfloat16)
                out.append((w.contiguous(memory_format=torch.channels_last), shift.to(torch.bfloat16), c.stride))
            return out
        return self._pack.get(ps, build)

    def features(self, img):
        """-> channels-last bf16 c1 (after the max-pool), c2, c3, c4."""
        convs = self.conv_pack()
        x = img.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        for w, b, s in convs[:3]:
            x = F.relu(F.conv2d(x, w, b, stride=s, padding=1))
        c1 = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
        outs = [c1]
        for w, b, s in convs[3:]:
            outs.append(F.relu(F.conv2d(outs[-1], w, b, stride=s, padding=1)))
        return outs


@_register
class OnePeaceAdapter(nn.Module):
    def __init__(self, pretrain_size=256, conv_inplane=64, n_points=4, deform_num_heads=6, init_values=0.0, cffn_ratio=0.25,
                 deform_ratio=1.0, with_cffn=True, interaction_indexes=None, add_vit_feature=True, with_cp=False,
                 activation_dropout=0.0, attention_dropout=0.0, attention_heads=24, bucket_size=16, dropout=0.0,
                 embed_dim=1536, drop_path_rate=0.0, ffn_embed_dim=6144, layers=40, layer_scale_init_value=1e-2,
                 norm_cfg=dict(type="LN"), pretrained=None, use_checkpoint=False, rp_bias=True, shared_rp_bias=False):
        super().__init__()
        if dropout > 0 or attention_dropout > 0 or activation_dropout > 0:
            raise NotImplementedError("OnePeaceAdapter: dropout, attention_dropout and activation_dropout must be 0 (the "
                                      "segmentation configs use 0; only inference is built)")
        if not rp_bias or shared_rp_bias:
            raise NotImplementedError("OnePeaceAdapter: only per-layer relative-position tables (rp_bias=True, "
                                      "shared_rp_bias=False) of the segmentation configs are built")
        if not with_cffn or not add_vit_feature:
            raise NotImplementedError("OnePeaceAdapter: with_cffn=False and add_vit_feature=False are not built")
        runs = [list(r) for r in (interaction_indexes or [])]
        if not runs or any(len(r) != 2 or r[0] > r[1] for r in runs) or runs[0][0] != 0 or runs[-1][1] != layers - 1 \
                or any(a[1] + 1 != b[0] for a, b in zip(runs, runs[1:])):
            raise NotImplementedError(f"OnePeaceAdapter: interaction_indexes {interaction_indexes} must split the {layers} "
                                      "layers into contiguous runs covering all of them")
        if embed_dim * deform_ratio / deform_num_heads != 32:
            raise NotImplementedError(f"OnePeaceAdapter: embed_dim * deform_ratio / deform_num_heads = "
                                      f"{embed_dim * deform_ratio / deform_num_heads:g}; only 32 channels per deformable "
                                      "head are built")
        if bucket_size % 2:
            raise NotImplementedError(f"OnePeaceAdapter: bucket_size {bucket_size} is odd (the c4 level needs an even grid)")
        self.init_cfg = dict(type="Pretrained", checkpoint=pretrained)
        cfg = AdjustEncDecConfig(embed_dim=embed_dim, ffn_embed_dim=ffn_embed_dim, layers=layers, attention_heads=attention_heads,
                                 drop_path_rate=drop_path_rate, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                                 magneto_scale_attn=True, scale_attn=False, scale_fc=True, scale_heads=False,
                                 use_text_moe=False, use_image_moe=True, use_audio_moe=False, use_layer_scale=True,
                                 layer_scale_init_value=layer_scale_init_value)
        self.image_adapter = ImageAdaptor(attention_heads, bucket_size, embed_dim, dropout, shared_rp_bias)
        self.encoder = SegEncoder(cfg, bucket_size)
        self.rp_bias = rp_bias
        self.shared_rp_bias = shared_rp_bias
        self.num_block = self.encoder.num_layers
        self.pretrain_size = (pretrain_size, pretrain_size)
        self.flags = [i for i in range(-1, self.num_block, self.num_block // 4)][1:]
        self.interaction_indexes = interaction_indexes
        self.add_vit_feature = add_vit_feature
        self.level_embed = nn.Parameter(torch.zeros(3, embed_dim))
        self.spm = SpatialPriorModule(inplanes=conv_inplane, embed_dim=embed_dim)
        self.interactions = nn.Sequential(*[
            InteractionBlockWithCls(embed_dim, deform_num_heads, n_points, init_values, cffn_ratio, deform_ratio,
                                    extra_extractor=(i == len(runs) - 1)) for i in range(len(runs))])
        self.up = nn.ConvTranspose2d(embed_dim, embed_dim, 2, 2)
        self.norm1 = nn.SyncBatchNorm(embed_dim)
        self.norm2 = nn.SyncBatchNorm(embed_dim)
        self.norm3 = nn.SyncBatchNorm(embed_dim)
        self.norm4 = nn.SyncBatchNorm(embed_dim)
        self.up.apply(self._init_weights)
        self.spm.apply(self._init_weights)
        self.interactions.apply(self._init_weights)
        for m in self.modules():
            if isinstance(m, MSDeformAttn):
                m._reset_parameters()
        nn.init.normal_(self.level_embed)
        self._head_pack = PackCache()
        self._layout = {}
        self.part_events = None     # a list: forward appends (part name, recorded CUDA event) at each part's end

    @staticmethod
    def _init_weights(m):
        """onepeace_adapter.py:68-81."""
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, (nn.LayerNorm, nn.BatchNorm2d)):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)
        elif isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
            fan_out = m.kernel_size[0] * m.kernel_size[1] * m.out_channels // m.groups
            m.weight.data.normal_(0, math.sqrt(2.0 / fan_out))
            if m.bias is not None:
                m.bias.data.zero_()

    resize_abs_pos_embed = resize_abs_pos_embed

    def resize_rel_pos_embed(self, checkpoint):
        """onepeace.py:493-545: the shared image_adapter.rel_pos_table_list.0.weight expanded to every layer's
        rel_pos_table, rp_bucket keys dropped, and tables of another grid resampled by geometric_sequence_interpolation."""
        state_dict = checkpoint["state_dict"] if "state_dict" in checkpoint else checkpoint
        if "image_adapter.rel_pos_table_list.0.weight" in state_dict:
            if _get_rank() == 0:
                print("Expand the shared relative position embedding to each transformer block. ")
            table = state_dict.pop("image_adapter.rel_pos_table_list.0.weight")
            for i in range(self.encoder.num_layers):
                state_dict[f"encoder.layers.{i}.rel_pos_table.weight"] = table.clone()
        own = self.state_dict()
        for key in list(state_dict.keys()):
            if "image_adapter.rp_bucket" in key:
                state_dict.pop(key)
            if "rel_pos_table.weight" in key and key in own:
                table = state_dict[key]
                src = int((table.shape[0] - 3) ** 0.5)
                dst = int((own[key].shape[0] - 3) ** 0.5)
                if src != dst:
                    new = geometric_sequence_interpolation(src, dst, table[:-3], table.shape[1])
                    state_dict[key] = torch.cat((new, table[-3:]), dim=0)
        return state_dict

    def init_weights(self, pretrained=None):
        """onepeace.py:547-578: trunc-normal Linear weights, zero biases and unit LayerNorms, then the checkpoint of
        `pretrained` (or the constructor's), .pkl or .pth, resized and loaded non-strictly."""
        def _init(m):
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.LayerNorm):
                nn.init.constant_(m.bias, 0)
                nn.init.constant_(m.weight, 1.0)
        self.apply(_init)
        path = pretrained or self.init_cfg.get("checkpoint")
        if not path:
            return
        if path.endswith(".pkl"):
            with open(path, "rb") as f:
                model = pickle.load(f, encoding="latin1")["model"]
        else:
            ckpt = torch.load(path, map_location="cpu", weights_only=False)
            model = ckpt["state_dict"] if "state_dict" in ckpt else ckpt
        self.resize_abs_pos_embed(model)
        state_dict = self.resize_rel_pos_embed(model)
        msg = self.load_state_dict(state_dict, False)
        if _get_rank() == 0:
            print(msg)

    def _pack(self):
        """fc1..fc4 as bf16 GEMM weights (level_embed folded into fc2..fc4's biases), the transposed conv as a [(dy, dx,
        c_out), c_in] GEMM weight with its bias repeated over (dy, dx), and norm1..norm4 folded to (scale, shift)."""
        s = self.spm
        norms = [self.norm1, self.norm2, self.norm3, self.norm4]
        ps = [s.fc1.weight, s.fc1.bias, s.fc2.weight, s.fc2.bias, s.fc3.weight, s.fc3.bias, s.fc4.weight, s.fc4.bias,
              self.level_embed, self.up.weight, self.up.bias] + \
            [t for n in norms for t in (n.weight, n.bias, n.running_mean, n.running_var)]

        def build():
            fc = [(bf16(c.weight.reshape(c.weight.shape[0], -1)),
                   f32(c.bias.detach().double() + (self.level_embed[i - 1].detach().double() if i else 0)))
                  for i, c in enumerate((s.fc1, s.fc2, s.fc3, s.fc4))]
            bn = [tuple(f32(t) for t in fold_bn(n)) for n in norms]
            return dict(fc=fc, up_w=bf16(convt_weight(self.up.weight)), up_b=f32(self.up.bias.repeat(4)), bn=bn)
        return self._head_pack.get(ps, build)

    def layout(self, B, device):
        """Per batch size: reference points of the injector (the ViT grid) and of the extractors (the three c levels),
        fp32 [rows, 1, 2], and the row indices of level c2 in c."""
        key = (B, str(device))
        if key not in self._layout:
            side = self.image_adapter.bucket_size
            shapes = level_shapes(side)
            T = sum(h * w for h, w in shapes)
            ref_x = reference_points([(side, side)]).repeat(B, 1).view(-1, 1, 2)
            ref_c = reference_points(shapes).repeat(B, 1).view(-1, 1, 2)
            n2 = shapes[0][0] * shapes[0][1]
            c2_rows = (torch.arange(B).view(-1, 1) * T + torch.arange(n2).view(1, -1)).reshape(-1)
            self._layout[key] = (ref_x.to(device).contiguous(), ref_c.to(device).contiguous(), c2_rows.to(device))
        return self._layout[key]

    def forward(self, x):
        """-> [f1, f2, f3, f4], fp32 NCHW [B, d, 4 bucket, 4 bucket] ... [B, d, bucket / 2, bucket / 2]
        (onepeace_adapter.py:93-135); autocast does not change them."""
        side = self.image_adapter.bucket_size
        if x.dim() != 4 or tuple(x.shape[1:]) != (3, 16 * side, 16 * side):
            raise ValueError(f"OnePeaceAdapter with bucket_size {side} takes [B, 3, {16 * side}, {16 * side}] images, "
                             f"got {tuple(x.shape)}")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("OnePeaceAdapter: only inference is built; run under torch.no_grad() (mmseg's "
                                      "single_gpu_test does)")
        if self.training:
            raise NotImplementedError("OnePeaceAdapter: only eval mode is built (BatchNorm with its running statistics); "
                                      "call .eval() first, as mmseg's single_gpu_test does")
        for layer in self.encoder.layers:
            layer.check_structure()
        with torch.autocast("cuda", enabled=False):
            return self._forward(x)

    def _mark(self, part):
        if self.part_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.part_events.append((part, ev))

    def _forward(self, img):
        B, dev = img.shape[0], img.device
        side = self.image_adapter.bucket_size
        d = self.level_embed.shape[1]
        shapes = level_shapes(side)
        sizes = [h * w for h, w in shapes]
        T, starts = sum(sizes), [0, sizes[0], sizes[0] + sizes[1]]
        S, n_patch = side * side + 1, side * side
        pk = self._pack()
        ref_x, ref_c, c2_rows = self.layout(B, dev)

        def e(rows, n, dt=torch.bfloat16):
            return torch.empty(rows, n, dtype=dt, device=dev)

        self._mark("start")
        # SPM, then fc1 into c1 and fc2..fc4 (+ level_embed) into their rows of c
        feats = self.spm.features(img)
        c1 = K.gemm(feats[0].permute(0, 2, 3, 1).reshape(-1, feats[0].shape[1]), pk["fc"][0][0], K.EPI_STORE_F32,
                    e(B * 16 * side * side, d, torch.float32), bias=pk["fc"][0][1])
        c = e(B * T, d, torch.float32)
        for l, f in enumerate(feats[1:]):
            K.gemm(f.permute(0, 2, 3, 1).reshape(-1, f.shape[1]), pk["fc"][l + 1][0], K.EPI_STORE_F32, c,
                   bias=pk["fc"][l + 1][1], out_group=sizes[l], out_group_stride=T, out_row_offset=starts[l])
        self._mark("spm")
        # ViT stem
        rows = self.image_adapter.stem(img)
        biases = self.encoder.biases()
        self._mark("stem")

        def ln_patches(norm, out):     # LayerNorm of the patch rows (every row but each sample's CLS row)
            return K.layernorm(rows[1:], f32(norm.weight), f32(norm.bias), out, rows=B * S - 1, eps=norm.eps,
                               row_period=S, row_valid=n_patch, out_period=n_patch)

        def ln_c(norm, out):
            return K.layernorm(c, f32(norm.weight), f32(norm.bias), out, eps=norm.eps)

        outs = []
        qx, qc = e(B * n_patch, d), e(B * T, d)
        for blk, (lo, hi) in zip(self.interactions, self.interaction_indexes):
            inj = blk.injector
            ln_patches(inj.query_norm, qx)
            ln_c(inj.feat_norm, qc)
            a = inj.attn
            msda_forward(msda_pack(a, a._pack), qx, qc, ref_x, shapes, starts, B, n_patch, a.n_heads, a.n_points, rows,
                         K.EPI_RESID_F32, gamma=f32(inj.gamma), resid=rows, out_group=n_patch, out_group_stride=S,
                         out_row_offset=1)
            self._mark("injectors")
            self.encoder.run_block(rows, lo, hi, biases, B, S)
            self._mark("layers")
            exts = [blk.extractor] + (list(blk.extra_extractors) if blk.extra_extractors is not None else [])
            for ext in exts:
                ln_c(ext.query_norm, qc)
                ln_patches(ext.feat_norm, qx)
                a = ext.attn
                msda_forward(msda_pack(a, a._pack), qc, qx, ref_c, [(side, side)], [0], B, T, a.n_heads, a.n_points, c,
                             K.EPI_RESID_F32, resid=c)
                fp = ext.ffn_pack()
                ln_c(ext.ffn_norm, qc)
                h = K.gemm(qc, fp["w1"], K.EPI_STORE_BF16, e(B * T, fp["w1"].shape[0]), bias=fp["b1"])
                h = K.seg_dwconv_gelu(h, fp["dw"], fp["db"], shapes, B)
                K.gemm(h, fp["w2"], K.EPI_RESID_F32, c, bias=fp["b2"], resid=c)
            outs.append(rows.clone())
            self._mark("extractors")
        # output maps
        c2b = K.row_gather(c, c2_rows, out_dtype=torch.bfloat16)
        up = K.gemm(c2b, pk["up_w"], K.EPI_STORE_F32, e(B * sizes[0], 4 * d, torch.float32), bias=pk["up_b"])
        sc, sh = zip(*pk["bn"])
        res = [K.seg_out_map(c1, 16 * side * side, 0, outs[0], S, 1, side, sc[0], sh[0], B, 4 * side, 4 * side, extra=up)]
        for l, (h, w) in enumerate(shapes):
            res.append(K.seg_out_map(c, T, starts[l], outs[l + 1], S, 1, side, sc[l + 1], sh[l + 1], B, h, w))
        self._mark("output_maps")
        return res
