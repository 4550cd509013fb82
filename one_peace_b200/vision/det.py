"""Drop-in for the COCO detection backbone of the vision branch, ``one_peace_vision/det/models/onepeace.py`` (``OnePeace``
and ``get_onepeace_lr_decay_rate``), as ``configs/onepeace/cascade_mask_rcnn_vitdet_50ep.py`` builds it.

The module tree, parameter and buffer names, shapes, dtypes and registration order are the reference's, so the released
``onepeace_det_coco.pth`` loads strictly and detectron2's optimizer builder assigns the same lr-decay rates.  Inference only:

    hMLP stem + pos_embed[1:]        the classifier's patchify + three patch GEMMs, no CLS row
    window-major rows                one row_gather after the stem keeps every window_size^2 window contiguous through all
                                     layers; one more at the end restores the row-major grid of ``last_feat``
    relative position                the shared table, bicubically resized to the global (2 bucket - 1)^2 and window
                                     (2 window - 1)^2 grids when they differ from the pretraining grid (cached against the
                                     table's version), in LUT form; plus the decomposed rel_pos_h / rel_pos_w terms
                                     (csrc/relpos_decomp.cu: opb_relpos_decomp_proj, then opb_attention_decomp_fwd)
    layers                           TransformerEncoder.run_fused: window layers attend over B * (bucket / window)^2
                                     sequences of window^2 rows, global layers over B sequences of bucket^2 rows

Refused in the constructor: dropout, attention_dropout or activation_dropout > 0, ``rp_bias=True``, ``shared_rp_bias=False``,
``use_decomposed_rel_pos=False`` and a bucket_size that is not a multiple of window_size (windows that need padding).
``forward`` raises ValueError for an input that is not [B, 3, 16 bucket, 16 bucket] and NotImplementedError when a
gradient is required (no backward is built).
"""
import pickle

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import kernels as K
from .. import relpos
from ..adapter.image import LayerNorm2D, make_image_bucket_position
from ..components import Embedding, PackCache, bf16, f32
from ..transformer.multihead_attention import MultiheadAttention
from ..transformer.transformer_encoder import TransformerEncoder
from ..transformer.transformer_layer import TransformerEncoderLayer
from ..unify_model_config import AdjustEncDecConfig

try:  # pragma: no cover - detectron2 is not installed in the build image
    from detectron2.modeling import Backbone
except Exception:
    class Backbone(nn.Module):
        """The surface of detectron2's ``Backbone`` that its FPN and ROI heads read."""

        def __init__(self):
            super().__init__()

        @property
        def size_divisibility(self):
            return 0

        @property
        def padding_constraints(self):
            return {}

        def output_shape(self):
            return {name: dict(channels=self._out_feature_channels[name], stride=self._out_feature_strides[name])
                    for name in self._out_features}

__all__ = ["OnePeace", "get_onepeace_lr_decay_rate"]

Q_UNSCALE = 8.0      # the QKV epilogue stores q * head_dim^-0.5; the decomposed terms use the unscaled q


def _get_rank():
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_rank()
    return 0


def resize_table(table, src_side, dst_side):
    """onepeace.py:123-144: the (src_side x src_side) rows of a relative-position table [src_side^2 + 3, H] bicubically
    resized to (dst_side x dst_side), the three extra rows kept; the table itself when the sides agree."""
    if src_side == dst_side:
        return table
    body = table[:-3].view(1, src_side, src_side, -1).permute(0, 3, 1, 2)
    body = F.interpolate(body, size=(dst_side, dst_side), mode="bicubic")
    return torch.cat((body.permute(0, 2, 3, 1).reshape(dst_side ** 2, -1), table[-3:]), dim=0)


class DetBias:
    """Attention layout of one layer: LUT-form bias `rp`, the sequence view (B sequences of S rows) of the window-major rows,
    the kh x kw grid and each row's coordinates on it (int32 device tensors)."""

    def __init__(self, rp, B, S, side, pos_y, pos_x):
        self.rp, self.B, self.S, self.side, self.pos_y, self.pos_x = rp, B, S, side, pos_y, pos_x


class DetAttention(MultiheadAttention):
    """onepeace.py:160-216 with use_decomposed_rel_pos=True: the project's attention module plus rel_pos_h / rel_pos_w."""

    def __init__(self, embed_dim, num_heads, dropout=0.0, use_decomposed_rel_pos=True, input_size=None):
        super().__init__(embed_dim, num_heads, dropout=dropout, magneto_scale_attn=True)
        self.dropout_module = nn.Dropout(dropout)
        self.use_decomposed_rel_pos = use_decomposed_rel_pos
        self.rel_pos_h = nn.Parameter(torch.zeros(2 * input_size[0] - 1, self.head_dim))
        self.rel_pos_w = nn.Parameter(torch.zeros(2 * input_size[1] - 1, self.head_dim))
        self._cache = PackCache()

    def run_attention(self, qkv, bias, key_pad, B, S, out=None, ln_stats=None, lse=None):
        """`bias` is the layer's DetBias; the rows B * S are viewed as bias.B sequences of bias.S rows."""
        assert key_pad is None and bias.B * bias.S == B * S
        side = bias.side
        if self.rel_pos_h.shape[0] != 2 * side - 1:
            raise ValueError(f"rel_pos_h has {self.rel_pos_h.shape[0]} rows for a {side} x {side} attention grid")
        rph, rpw = self._cache.get([self.rel_pos_h, self.rel_pos_w],
                                   lambda: (f32(self.rel_pos_h).contiguous(), f32(self.rel_pos_w).contiguous()))
        H = self.num_heads
        rel_h, rel_w = K.relpos_decomp_proj(qkv, rph, rpw, bias.pos_y, bias.pos_x, bias.B, bias.S, H, side, side,
                                            q_unscale=Q_UNSCALE)
        return K.attention_decomp(qkv, bias.rp, rel_h, rel_w, bias.pos_y, bias.pos_x, bias.B, bias.S, H, side, side,
                                  out=out, ln_stats=ln_stats, lse=lse)


class DetLayer(TransformerEncoderLayer):
    """onepeace.py:219-331 (rp_bias=False): the project's layer (fused-LayerNorm forward) with a DetAttention."""

    def __init__(self, cfg, drop_path_rate, bucket_size, pretrain_bucket_size, use_decomposed_rel_pos, window_size):
        super().__init__(cfg, drop_path_rate=drop_path_rate)
        side = window_size if window_size > 0 else bucket_size
        self.self_attn = DetAttention(cfg.embed_dim, cfg.attention_heads, dropout=cfg.attention_dropout,
                                      use_decomposed_rel_pos=use_decomposed_rel_pos, input_size=(side, side))
        self.dropout = nn.Dropout(cfg.dropout)
        self.activation_dropout = nn.Dropout(cfg.activation_dropout)
        self.drop_path = nn.Identity()
        self.rp_bias = False
        self.window_size = window_size
        self.bucket_size = side
        self.pretrain_bucket_size = window_size if window_size > 0 else pretrain_bucket_size


class DetImageAdaptor(nn.Module):
    """onepeace.py:78-157 (shared_rp_bias=True).  The reference builds it with its default pretrain_bucket_size 16 whatever
    OnePeace is given, so the shared table always has 31^2 + 3 rows."""

    def __init__(self, attention_heads=24, bucket_size=64, embed_dim=1536, dropout=0.0, pretrain_bucket_size=16,
                 shared_rp_bias=True, window_size=0):
        super().__init__()
        self.dropout = nn.Dropout(dropout)
        c4 = embed_dim // 4
        self.embed_images = nn.Sequential(
            nn.Conv2d(3, c4, kernel_size=4, stride=4), LayerNorm2D(c4), nn.GELU(),
            nn.Conv2d(c4, c4, kernel_size=2, stride=2), LayerNorm2D(c4), nn.GELU(),
            nn.Conv2d(c4, embed_dim, kernel_size=2, stride=2))
        scale = embed_dim ** -0.5
        self.pretrain_bucket_size = pretrain_bucket_size
        self.bucket_size = bucket_size
        self.pos_embed = nn.Parameter(scale * torch.randn(bucket_size ** 2 + 1, embed_dim))
        self.window_size = window_size
        self.shared_rp_bias = shared_rp_bias
        num_rel_dis_pretrain = (2 * pretrain_bucket_size - 1) ** 2 + 3
        num_rel_dis = (2 * bucket_size - 1) ** 2 + 3
        num_rel_dis_window = (2 * window_size - 1) ** 2 + 3
        self.rel_pos_table = Embedding(num_rel_dis_pretrain, attention_heads, zero_init=True)
        self.register_buffer("rp_bucket", make_image_bucket_position(bucket_size, num_rel_dis)[1:, 1:].contiguous())
        self.register_buffer("rp_bucket_window",
                             make_image_bucket_position(window_size, num_rel_dis_window)[1:, 1:].contiguous())
        self._stem_cache = PackCache()
        self._lut_cache = PackCache()
        self._layout = {}

    def _stem_pack(self):
        e = self.embed_images
        ps = [e[0].weight, e[0].bias, e[1].layer_norm.weight, e[1].layer_norm.bias, e[3].weight, e[3].bias,
              e[4].layer_norm.weight, e[4].layer_norm.bias, e[6].weight, e[6].bias, self.pos_embed]

        def build():
            w1, b1, l1w, l1b, w2, b2, l2w, l2b, w3, b3, pos = ps
            c4, d = w1.shape[0], w3.shape[0]
            return dict(w1=bf16(w1.reshape(c4, 48)), b1=f32(b1), l1w=f32(l1w), l1b=f32(l1b),
                        w2=bf16(w2.permute(0, 2, 3, 1).reshape(c4, 4 * c4)), b2=f32(b2), l2w=f32(l2w), l2b=f32(l2b),
                        w3=bf16(w3.permute(0, 2, 3, 1).reshape(d, 4 * c4)), b3=f32(b3),
                        pos=f32(pos[1:]).contiguous())
        return self._stem_cache.get(ps, build)

    def stem(self, img):
        """hMLP stem + pos_embed[1:] (onepeace.py:146-152) -> fp32 [B * side^2, d], row-major grid per sample."""
        pk = self._stem_pack()
        B, _, R, _ = img.shape
        c4, d = pk["w1"].shape[0], pk["w3"].shape[0]
        g1, g2, w = R // 4, R // 8, R // 16
        dev = img.device
        im = img if img.dtype in (torch.float32, torch.bfloat16) else img.float()
        a1 = K.image_patchify4(im.contiguous())
        y1 = K.gemm(a1, pk["w1"], K.EPI_STORE_BF16, torch.empty(B * g1 * g1, c4, dtype=torch.bfloat16, device=dev),
                    bias=pk["b1"])
        a2 = K.layernorm(y1, pk["l1w"], pk["l1b"], torch.empty(B * g2 * g2, 4 * c4, dtype=torch.bfloat16, device=dev),
                         gelu=True, merge_grid_w=g1)
        y2 = K.gemm(a2, pk["w2"], K.EPI_STORE_BF16, torch.empty(B * g2 * g2, c4, dtype=torch.bfloat16, device=dev),
                    bias=pk["b2"])
        a3 = K.layernorm(y2, pk["l2w"], pk["l2b"], torch.empty(B * w * w, 4 * c4, dtype=torch.bfloat16, device=dev),
                         gelu=True, merge_grid_w=g2)
        x = torch.empty(B * w * w, d, dtype=torch.float32, device=dev)
        return K.gemm(a3, pk["w3"], K.EPI_RESID_F32, x, bias=pk["b3"], resid=pk["pos"], resid_period=w * w)

    def luts(self):
        """(global, window) LUT-form biases of the shared table, resized as get_rel_pos_bias (onepeace.py:123-144) does;
        rebuilt when the table changes."""
        table = self.rel_pos_table.weight
        src = 2 * self.pretrain_bucket_size - 1

        def build():
            out = []
            for side in (self.bucket_size, self.window_size):
                t = resize_table(f32(table.detach()), src, 2 * side - 1).contiguous()
                idx = torch.arange((2 * side - 1) ** 2, dtype=torch.int32, device=table.device)
                out.append(K.relpos_lut_build(t, idx))
            return out
        return self._lut_cache.get([table], build)

    def layout(self, B, device):
        """-> (perm int64 [B * S]: window-major row -> row-major row, inverse, global DetBias, window DetBias)."""
        key = (B, str(device))
        if key not in self._layout:
            side, win = self.bucket_size, self.window_size
            S, n_win = side * side, (side // win) ** 2
            order, y, x, ly, lx = relpos.window_major_order(side, win)
            base = torch.arange(B, dtype=torch.int64).repeat_interleave(S) * S
            perm = base + torch.from_numpy(order).repeat(B)
            inv = torch.empty_like(perm)
            inv[perm] = torch.arange(B * S, dtype=torch.int64)
            i32 = lambda a: torch.from_numpy(a).to(device=device, dtype=torch.int32).contiguous()
            _, gr, gc = relpos.grid_lut_index(side, order)
            _, wr, wc = relpos.grid_lut_index(win)
            g = dict(B=B, S=S, side=side, pos_y=i32(y), pos_x=i32(x), codes=(i32(gr), i32(gc)))
            w = dict(B=B * n_win, S=win * win, side=win, pos_y=i32(ly[:win * win]), pos_x=i32(lx[:win * win]),
                     codes=(i32(wr), i32(wc)))       # every window has the same local grid
            self._layout[key] = (perm.to(device), inv.to(device), g, w)
        return self._layout[key]


class DetEncoder(nn.Module):
    """onepeace.py:334-409; the fused inference loop is TransformerEncoder's."""

    run_fused = TransformerEncoder.run_fused

    def __init__(self, cfg, bucket_size, pretrain_bucket_size, use_decomposed_rel_pos, window_size, window_block_indexes):
        super().__init__()
        self.cfg = cfg
        self.dropout_module = nn.Dropout(cfg.dropout)
        self.attention_heads = cfg.attention_heads
        self.num_attention_heads = cfg.attention_heads
        self.window_size = window_size
        self.layers = nn.ModuleList([])
        dpr = [v.item() for v in torch.linspace(0, cfg.drop_path_rate, cfg.layers, device="cpu")]
        for i in range(cfg.layers):
            self.layers.append(DetLayer(cfg, dpr[i], bucket_size, pretrain_bucket_size, use_decomposed_rel_pos,
                                        window_size if i in window_block_indexes else 0))
        self.num_layers = len(self.layers)


class OnePeace(Backbone):
    def __init__(self, activation_dropout=0.0, attention_dropout=0.0, attention_heads=24, bucket_size=64,
                 pretrain_bucket_size=16, dropout=0.0, embed_dim=1536, drop_path_rate=0.0, ffn_embed_dim=6144, layers=40,
                 layer_scale_init_value=1e-2, out_feature="last_feat", rp_bias=False, use_decomposed_rel_pos=False,
                 shared_rp_bias=True, use_checkpoint=False, window_size=0, window_block_indexes=(), pretrained=None):
        super().__init__()
        if dropout > 0 or attention_dropout > 0 or activation_dropout > 0:
            raise NotImplementedError("OnePeace: dropout, attention_dropout and activation_dropout must be 0 (the detection "
                                      "configs use 0; only inference is built)")
        if rp_bias or not shared_rp_bias:
            raise NotImplementedError("OnePeace: only the shared relative-position table (rp_bias=False, shared_rp_bias=True) "
                                      "of the detection config is built")
        if not use_decomposed_rel_pos:
            raise NotImplementedError("OnePeace: only use_decomposed_rel_pos=True (the detection config) is built")
        if window_size <= 0 or bucket_size % window_size != 0:
            raise NotImplementedError(f"OnePeace: bucket_size {bucket_size} must be a multiple of window_size {window_size} "
                                      "(windows that need padding are not built)")
        cfg = AdjustEncDecConfig(embed_dim=embed_dim, ffn_embed_dim=ffn_embed_dim, layers=layers, attention_heads=attention_heads,
                                 drop_path_rate=drop_path_rate, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                                 magneto_scale_attn=True, scale_attn=False, scale_fc=True, scale_heads=False,
                                 use_text_moe=False, use_image_moe=True, use_audio_moe=False, use_layer_scale=True,
                                 layer_scale_init_value=layer_scale_init_value)
        self.image_adapter = DetImageAdaptor(attention_heads=attention_heads, bucket_size=bucket_size, embed_dim=embed_dim,
                                             dropout=dropout, shared_rp_bias=shared_rp_bias, window_size=window_size)
        self.encoder = DetEncoder(cfg, bucket_size, pretrain_bucket_size, use_decomposed_rel_pos, window_size,
                                  tuple(window_block_indexes))
        self.rp_bias = rp_bias
        self.shared_rp_bias = shared_rp_bias
        self.use_checkpoint = use_checkpoint
        self._out_feature_channels = {out_feature: embed_dim}
        self._out_feature_strides = {out_feature: 16}
        self._out_features = [out_feature]
        self.apply(self._init_weights)
        if pretrained:
            if pretrained.endswith(".pkl"):
                with open(pretrained, "rb") as f:
                    checkpoint_model = pickle.load(f, encoding="latin1")["model"]
            else:
                checkpoint_model = torch.load(pretrained, map_location="cpu", weights_only=False)["model"]
            self.resize_abs_pos_embed(checkpoint_model)
            checkpoint_model.pop("image_adapter.rp_bucket")
            self.resize_rel_pos_embed(checkpoint_model)
            if _get_rank() == 0:
                print(self.load_state_dict(checkpoint_model, strict=False))
                print(f"Loading OFA Encoder pretrained weights from {pretrained}.")

    def resize_abs_pos_embed(self, checkpoint):
        """onepeace.py:535-558: bicubic resize of the checkpoint's positional rows, the first row kept."""
        pos = checkpoint["image_adapter.pos_embed"]
        dim = pos.shape[-1]
        num_patches = self.image_adapter.bucket_size ** 2
        extra = self.image_adapter.pos_embed.shape[-2] - num_patches
        orig, new = int((pos.shape[-2] - extra) ** 0.5), int(num_patches ** 0.5)
        if orig != new:
            if _get_rank() == 0:
                print(f"Position interpolate from {orig}x{orig} to {new}x{new}")
            tok = pos[extra:].reshape(-1, orig, orig, dim).permute(0, 3, 1, 2)
            tok = F.interpolate(tok, size=(new, new), mode="bicubic", align_corners=False)
            checkpoint["image_adapter.pos_embed"] = torch.cat((pos[:extra], tok.permute(0, 2, 3, 1).flatten(0, 2)), dim=0)

    def resize_rel_pos_embed(self, checkpoint):
        """onepeace.py:560-613 with shared_rp_bias=True: rel_pos_table_list.0.weight -> rel_pos_table.weight, rp_bucket keys
        dropped.  The reference's per-layer geometric resampling only touches encoder rel_pos_table keys, which the
        shared-table model does not have."""
        state_dict = checkpoint["state_dict"] if "state_dict" in checkpoint else checkpoint
        if "image_adapter.rel_pos_table_list.0.weight" in state_dict:
            state_dict["image_adapter.rel_pos_table.weight"] = state_dict["image_adapter.rel_pos_table_list.0.weight"]
        for key in list(state_dict.keys()):
            if "image_adapter.rp_bucket" in key:
                state_dict.pop(key)
            if "rel_pos_table.weight" in key and "encoder" in key:
                raise NotImplementedError(f"{key}: per-layer relative-position tables (rp_bias=True) are not built")
        return state_dict

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def forward(self, x):
        """-> {out_feature: fp32 [B, embed_dim, bucket, bucket]} (onepeace.py:624-629); autocast does not change it."""
        ad = self.image_adapter
        side = ad.bucket_size
        if x.dim() != 4 or tuple(x.shape[1:]) != (3, 16 * side, 16 * side):
            raise ValueError(f"OnePeace with bucket_size {side} takes [B, 3, {16 * side}, {16 * side}] images, "
                             f"got {tuple(x.shape)}")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("OnePeace: only inference is built; run under torch.no_grad() (detectron2's "
                                      "inference_on_dataset does)")
        for layer in self.encoder.layers:
            layer.check_structure()
        B = x.shape[0]
        with torch.autocast("cuda", enabled=False):
            rows = ad.stem(x)
            perm, inv, g, w = ad.layout(B, x.device)
            rows = K.row_gather(rows, perm)
            lut_g, lut_w = ad.luts()
            biases = []
            for layer in self.encoder.layers:
                lay, lut = (w, lut_w) if layer.window_size > 0 else (g, lut_g)
                rp = K.RelPosBias(lut=lut, code_row=lay["codes"][0], code_col=lay["codes"][1])
                biases.append(DetBias(rp, lay["B"], lay["S"], lay["side"], lay["pos_y"], lay["pos_x"]))
            S = side * side
            self.encoder.run_fused(rows, biases, None, B, S, "image")
            out = K.row_gather(rows, inv).view(B, side, side, -1).permute(0, 3, 1, 2).contiguous()
        return {self._out_features[0]: out}


def get_onepeace_lr_decay_rate(name, lr_decay_rate=0.9, num_layers=40):
    """onepeace.py:632-653: lr_decay_rate ** (num_layers + 1 - layer_id), layer_id 0 for the image adapter, i + 1 for
    encoder layer i, num_layers + 1 for everything else."""
    layer_id = num_layers + 1
    if name.startswith("backbone"):
        if ".image_adapter" in name:
            layer_id = 0
        elif ".layers." in name and ".residual." not in name:
            layer_id = int(name[name.find(".layers."):].split(".")[2]) + 1
        if _get_rank() == 0:
            print(f"{name} layer_id: {layer_id}")
    return lr_decay_rate ** (num_layers + 1 - layer_id)
