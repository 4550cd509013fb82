"""Drop-in for the Kinetics-400 action-recognition backbone of the vision branch,
``one_peace_vision/video/mmaction_custom/models/backbones/onepeace.py`` (``OnePeaceViT``), as
``configs/recognition/onepeace_k400*.py`` builds it.

The module tree, parameter and buffer names, shapes, dtypes and registration order are the reference's, so
``onepeace_video_k400.pth`` loads through mmcv's ``load_checkpoint`` and the configs' ``paramwise_cfg`` keys match.
Evaluation only:

    input                           NCTHW clips, reordered to (b t) c h w frames (a copy)
    hMLP stem, CLS + positions      autograd.ImageEmbedFn (three patch GEMMs), then one row_gather adds temporal_embedding[t]
                                    to every row of frame t, CLS row included: ((patch + pos) + temporal) in fp32
    rows                            frame-major, row (b T + t) N + n with N = bucket^2 + 1, fp32 residual stream
    layers                          VideoLayer.forward_video: the temporal pass attends along t at a row stride of N
                                    (csrc/attention_temporal.cu), the spatial pass over the N rows of each frame with the
                                    shared relative-position table in LUT form; every LayerNorm is folded into the GEMM
                                    that reads it, as in TransformerEncoderLayer.forward_rows_fused
    output                          image_layer_norm of the CLS rows only -> fp32 [B, d, T, 1, 1] for mmaction's I3DHead

Refused in the constructor, as no config uses them: dropout, attention_dropout or activation_dropout > 0,
``rp_bias=True``, ``shared_rp_bias=False`` and ``num_tadapter=2``.  ``forward`` raises ValueError for an input that is
not [B, 3, num_frames, 16 bucket, 16 bucket] and NotImplementedError when a gradient is required (no backward is built).
"""
import pickle

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import kernels as K
from .. import relpos
from ..adapter.image import LayerNorm2D, geometric_sequence_interpolation, make_image_bucket_position
from ..autograd import ImageEmbedFn
from ..components import Embedding, PackCache, bf16, f32
from ..transformer.transformer_layer import TransformerEncoderLayer
from ..unify_model_config import AdjustEncDecConfig

try:  # pragma: no cover - mmaction is not installed in the build image
    from mmaction.models.builder import BACKBONES
    _register = BACKBONES.register_module()
except Exception:
    def _register(cls):
        return cls

__all__ = ["OnePeaceViT"]


def _get_rank():
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_rank()
    return 0


class Adapter(nn.Module):
    """onepeace.py:21-39: fc2(gelu(fc1(x))), plus x when skip_connect."""

    def __init__(self, D_features, mlp_ratio=0.25, act_layer=nn.GELU, skip_connect=True):
        super().__init__()
        self.skip_connect = skip_connect
        D_hidden_features = int(D_features * mlp_ratio)
        self.act = act_layer()
        self.D_fc1 = nn.Linear(D_features, D_hidden_features)
        self.D_fc2 = nn.Linear(D_hidden_features, D_features)


class ImageAdaptor(nn.Module):
    """Parameter holder of onepeace.py:130-205 (shared_rp_bias=True): hMLP stem, cls_embedding, pos_embed,
    temporal_embedding, the shared rel_pos_table and the rp_bucket buffer."""

    def __init__(self, attention_heads=24, bucket_size=16, num_frames=32, dropout=0.0, embed_dim=1536,
                 shared_rp_bias=True):
        super().__init__()
        self.dropout_module = nn.Dropout(dropout)
        c4 = embed_dim // 4
        self.embed_images = nn.Sequential(
            nn.Conv2d(3, c4, kernel_size=4, stride=4), LayerNorm2D(c4), nn.GELU(),
            nn.Conv2d(c4, c4, kernel_size=2, stride=2), LayerNorm2D(c4), nn.GELU(),
            nn.Conv2d(c4, embed_dim, kernel_size=2, stride=2))
        scale = embed_dim ** -0.5
        self.cls_embedding = nn.Parameter(scale * torch.randn(1, 1, embed_dim))
        self.bucket_size = bucket_size
        self.num_frames = num_frames
        self.pos_embed = nn.Parameter(scale * torch.randn(bucket_size ** 2 + 1, embed_dim))
        self.temporal_embedding = nn.Parameter(torch.zeros(1, num_frames, embed_dim))
        self.shared_rp_bias = shared_rp_bias
        num_rel_dis = (2 * bucket_size - 1) ** 2 + 3
        self.rel_pos_table = Embedding(num_rel_dis, attention_heads, zero_init=True)
        self.register_buffer("rp_bucket", make_image_bucket_position(bucket_size, num_rel_dis))
        self._lut_cache = relpos.LutCache()
        self._temporal_cache = PackCache()

    def stem(self, frames):
        """hMLP stem + CLS + pos_embed + temporal_embedding (onepeace.py:187-201) of frames [B T, 3, R, R], clip-major
        -> fp32 [B T N, d] frame-major rows."""
        e = self.embed_images
        x = ImageEmbedFn.apply(frames, self.pos_embed, e[0].weight, e[0].bias, e[1].layer_norm.weight,
                               e[1].layer_norm.bias, e[3].weight, e[3].bias, e[4].layer_norm.weight, e[4].layer_norm.bias,
                               e[6].weight, e[6].bias, self.cls_embedding)
        BT, N, d = x.shape
        T = self.num_frames
        add = self._temporal_cache.get([self.temporal_embedding],
                                       lambda: f32(self.temporal_embedding[0]).repeat_interleave(N, dim=0).contiguous())
        idx = torch.arange(BT * N, dtype=torch.int64, device=x.device)
        assert add.shape[0] == T * N
        return K.row_gather(x.view(BT * N, d), idx, add=add)         # row (b T + t) N + n gains temporal[t]

    def lut_bias(self):
        """The shared table in LUT form for the spatial pass over S = bucket^2 + 1 rows (rebuilt when the table changes)."""
        S = self.bucket_size ** 2 + 1
        if S > K.ATTN_TC_MAX_S:
            raise NotImplementedError(f"OnePeaceViT: bucket_size {self.bucket_size} gives {S} tokens per frame; the LUT-form "
                                      f"attention is built for at most {K.ATTN_TC_MAX_S}")
        lut = self._lut_cache.get(S, self.rp_bucket.device, self.rp_bucket,
                                  lambda n: relpos.image_codes(n, self.bucket_size))
        return K.RelPosBias(lut=K.relpos_lut_build(f32(self.rel_pos_table.weight), lut[0]), code_row=lut[1],
                            code_col=lut[2])


class VideoLayer(TransformerEncoderLayer):
    """onepeace.py:254-352 (num_tadapter=1, rp_bias=False): the project's layer plus MLP_Adapter, S_Adapter and T_Adapter.
    One self_attn and one self_attn_layer_norm serve the temporal and the spatial pass."""

    def __init__(self, cfg, drop_path_rate, scale, num_frames):
        super().__init__(cfg, drop_path_rate=drop_path_rate)
        d = cfg.embed_dim
        self.MLP_Adapter = Adapter(d, skip_connect=False)
        self.S_Adapter = Adapter(d)
        self.scale = scale
        self.T_Adapter = Adapter(d, skip_connect=False)
        self.num_tadapter = 1
        self.num_frames = num_frames

    def _adapter_pack(self):
        cache = self._cache.setdefault("_adapters", PackCache())
        t, s, m = self.T_Adapter, self.S_Adapter, self.MLP_Adapter
        ps = [t.D_fc1.weight, t.D_fc1.bias, t.D_fc2.weight, t.D_fc2.bias, s.D_fc1.weight, s.D_fc1.bias, s.D_fc2.weight,
              s.D_fc2.bias, m.D_fc1.weight, m.D_fc1.bias, m.D_fc2.weight, m.D_fc2.bias, self.final_layer_norm.weight,
              self.final_layer_norm.bias]

        def build():
            m1w, m1c, m1b = self._fold([m.D_fc1.weight], self.final_layer_norm, [m.D_fc1.bias])
            return dict(t1w=bf16(t.D_fc1.weight), t1b=f32(t.D_fc1.bias), t2w=bf16(t.D_fc2.weight), t2b=f32(t.D_fc2.bias),
                        s1w=bf16(s.D_fc1.weight), s1b=f32(s.D_fc1.bias), s2w=bf16(s.D_fc2.weight), s2b=f32(s.D_fc2.bias),
                        m1w=m1w, m1c=m1c, m1b=m1b, m2w=bf16(m.D_fc2.weight), m2b=f32(m.D_fc2.bias),
                        scale=torch.full((self.embed_dim,), float(self.scale), dtype=torch.float32,
                                         device=m.D_fc2.weight.device))
        return cache.get(ps, build)

    def forward_video(self, x, ln1, ws, bias, Bv, T, N):
        """x fp32 [Bv T N, d] frame-major residual stream (in place), ws["xb"] its bf16 copy, ln1 its LayerNorm-1
        statistics (dict(ln_mu=, ln_rstd=) or dict(ln_partial=...)).  Returns the statistics of the layer output."""
        d, F_, H = self.embed_dim, self.ffn_embed_dim, self.self_attn.num_heads
        a = self._fused_attn_pack()
        f = self._fused_ffn_pack("image")
        ad = self._adapter_pack()
        n_t = (d + 255) // 256
        eps1, eps_in, eps2 = self.self_attn_layer_norm.eps, self.self_attn.ln.eps, self.final_layer_norm.eps
        tail = ws["tail"]
        # temporal pass: xt = T_Adapter(attn(LN1(x)) along t); y = x + xt feeds only the spatial pass
        K.gemm_ln(ws["xb"], a["wqkv"], K.EPI_STORE_BF16, ws["qkv"], ln_colsum=a["cqkv"], bias=a["dqkv"], colscale=a["qscale"],
                  workspace=tail, **ln1)
        K.attention_temporal(ws["qkv"], Bv, T, N, H, out=ws["o"], ln_stats=ws["part_a"])
        K.gemm_ln(ws["o"], a["wo"], K.EPI_STORE_BF16, ws["a"], ln_partial=(ws["part_a"], H, d, eps_in), ln_colsum=a["co"],
                  bias=a["do"], workspace=tail)
        K.gemm(ws["a"], ad["t1w"], K.EPI_GELU_BF16, ws["h"], bias=ad["t1b"])
        K.gemm_ln(ws["h"], ad["t2w"], K.EPI_RESID_F32, ws["y"], bias=ad["t2b"], resid=x, stats_out=ws["part_b"],
                  out_bf16=ws["yb"], workspace=tail)
        # spatial pass: a = attn(LN1(y)) per frame; x = x + gamma_1 * (a + S_fc2(gelu(S_fc1(a)))), x the layer input
        K.gemm_ln(ws["yb"], a["wqkv"], K.EPI_STORE_BF16, ws["qkv"], ln_partial=(ws["part_b"], n_t, d, eps1),
                  ln_colsum=a["cqkv"], bias=a["dqkv"], colscale=a["qscale"], workspace=tail)
        self.self_attn.run_attention(ws["qkv"], bias, None, Bv * T, N, out=ws["o"], ln_stats=ws["part_a"])
        K.gemm_ln(ws["o"], a["wo"], K.EPI_STORE_BF16, ws["a"], ln_partial=(ws["part_a"], H, d, eps_in), ln_colsum=a["co"],
                  bias=a["do"], workspace=tail)
        K.gemm(ws["a"], ad["s1w"], K.EPI_GELU_BF16, ws["h"], bias=ad["s1b"])
        K.scale_resid_fwd(x, ws["a"], a["g1"], None, ws["y"])                       # y = x + gamma_1 * a
        K.gemm_ln(ws["h"], ad["s2w"], K.EPI_RESID_F32, x, bias=ad["s2b"], gamma=a["g1"], resid=ws["y"],
                  stats_out=ws["part_b"], out_bf16=ws["xb"], workspace=tail)
        # joint pass: both FFN and MLP_Adapter read LN2 of this x; x + gamma_2 * ffn(xn), then + scale * MLP_Adapter(xn)
        K.gemm_ln(ws["xb"], f["w01"], K.EPI_GEGLU_BF16, ws["u"], ln_partial=(ws["part_b"], n_t, d, eps2),
                  ln_colsum=f["c01"], bias=f["d01"], stats_out=ws["part_c"])
        K.gemm_ln(ws["xb"], ad["m1w"], K.EPI_GELU_BF16, ws["h"], ln_partial=(ws["part_b"], n_t, d, eps2),
                  ln_colsum=ad["m1c"], bias=ad["m1b"])
        n_rec = 2 * ((2 * F_) // 256)
        K.gemm_ln(ws["u"], f["w2"], K.EPI_RESID_F32, x, ln_partial=(ws["part_c"], n_rec, F_, f["lnf_eps"]), ln_colsum=f["c2"],
                  bias=f["d2"], gamma=f["g2"], resid=x, workspace=tail)
        K.gemm_ln(ws["h"], ad["m2w"], K.EPI_RESID_F32, x, bias=ad["m2b"], gamma=ad["scale"], resid=x,
                  stats_out=ws["part_d"], out_bf16=ws["xb"], workspace=tail)
        return dict(ln_partial=(ws["part_d"], n_t, d, eps1))

    @staticmethod
    def video_workspace(M, d, F_, H, device):
        ws = TransformerEncoderLayer.fused_workspace(M, d, F_, H, device)
        ws.update(a=torch.empty(M, d, dtype=torch.bfloat16, device=device),
                  yb=torch.empty(M, d, dtype=torch.bfloat16, device=device),
                  y=torch.empty(M, d, dtype=torch.float32, device=device),
                  h=torch.empty(M, int(d * 0.25), dtype=torch.bfloat16, device=device))
        return ws


class TransformerEncoder(nn.Module):
    """Parameter holder of onepeace.py:355-420: `layers` and `image_layer_norm`."""

    def __init__(self, cfg, num_frames, scale):
        super().__init__()
        self.cfg = cfg
        self.num_attention_heads = cfg.attention_heads
        dpr = [v.item() for v in torch.linspace(0, cfg.drop_path_rate, cfg.layers, device="cpu")]   # also under meta
        self.layers = nn.ModuleList([VideoLayer(cfg, dpr[i], scale, num_frames) for i in range(cfg.layers)])
        self.num_layers = len(self.layers)
        self.image_layer_norm = nn.LayerNorm(cfg.embed_dim)

    def run(self, rows, bias, Bv, T, N):
        """The layer loop on the frame-major fp32 rows [Bv T N, d], in place."""
        d = rows.shape[1]
        ws = VideoLayer.video_workspace(rows.shape[0], d, self.cfg.ffn_embed_dim, self.num_attention_heads, rows.device)
        K.row_stats_cast(rows, ws["xb"], ws["mu"], ws["rstd"], eps=self.layers[0].self_attn_layer_norm.eps)
        ln1 = dict(ln_mu=ws["mu"], ln_rstd=ws["rstd"])
        for layer in self.layers:
            ln1 = layer.forward_video(rows, ln1, ws, bias, Bv, T, N)
        return rows


@_register
class OnePeaceViT(nn.Module):
    def __init__(self, activation_dropout=0.0, attention_dropout=0.0, attention_heads=12, adapter_scale=0.5, bucket_size=16,
                 num_tadapter=1, num_frames=32, dropout=0.1, drop_path_rate=0.0, embed_dim=1536, ffn_embed_dim=6144,
                 layers=40, layer_scale_init_value=1e-2, rp_bias=False, shared_rp_bias=True, use_checkpoint=False,
                 pretrained=None):
        super().__init__()
        if dropout > 0 or attention_dropout > 0 or activation_dropout > 0:
            raise NotImplementedError("OnePeaceViT: dropout, attention_dropout and activation_dropout must be 0 (the "
                                      "recognition configs use 0; only evaluation is built)")
        if rp_bias or not shared_rp_bias:
            raise NotImplementedError("OnePeaceViT: only the shared relative-position table (rp_bias=False, "
                                      "shared_rp_bias=True) of the recognition configs is built")
        if num_tadapter != 1:
            raise NotImplementedError("OnePeaceViT: only num_tadapter=1 (the recognition configs) is built")
        self.pretrained = pretrained
        cfg = AdjustEncDecConfig(embed_dim=embed_dim, ffn_embed_dim=ffn_embed_dim, layers=layers, attention_heads=attention_heads,
                                 drop_path_rate=drop_path_rate, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                                 magneto_scale_attn=True, scale_attn=False, scale_fc=True, scale_heads=False,
                                 use_text_moe=False, use_image_moe=True, use_audio_moe=False, use_layer_scale=True,
                                 layer_scale_init_value=layer_scale_init_value)
        self.image_adapter = ImageAdaptor(attention_heads=attention_heads, bucket_size=bucket_size, num_frames=num_frames,
                                          dropout=dropout, embed_dim=embed_dim, shared_rp_bias=shared_rp_bias)
        self.encoder = TransformerEncoder(cfg, num_frames, adapter_scale)
        self.rp_bias = rp_bias
        self.shared_rp_bias = shared_rp_bias
        self.use_checkpoint = use_checkpoint

    def resize_abs_pos_embed(self, checkpoint):
        """onepeace.py:526-551: bicubic resize of the checkpoint's positional rows, the first row kept."""
        pos = checkpoint["image_adapter.pos_embed"]
        dim = pos.shape[-1]
        num_patches = self.image_adapter.bucket_size ** 2
        extra = self.image_adapter.pos_embed.shape[-2] - num_patches
        orig, new = int((pos.shape[-2] - extra) ** 0.5), int(num_patches ** 0.5)
        if orig != new:
            if _get_rank() == 0:
                print("Position interpolate from %dx%d to %dx%d" % (orig, orig, new, new))
            tok = pos[extra:].reshape(-1, orig, orig, dim).permute(0, 3, 1, 2)
            tok = F.interpolate(tok, size=(new, new), mode="bicubic", align_corners=False)
            checkpoint["image_adapter.pos_embed"] = torch.cat((pos[:extra], tok.permute(0, 2, 3, 1).flatten(0, 2)), dim=0)

    def resize_rel_pos_embed(self, checkpoint):
        """onepeace.py:553-609 with shared_rp_bias=True: rel_pos_table_list.0.weight -> rel_pos_table.weight, the
        image_adapter.rp_bucket keys dropped, and every rel_pos_table.weight of another grid size resampled by geometric
        sequence interpolation (adapter.image.geometric_sequence_interpolation, the interp2d-free form)."""
        state_dict = checkpoint["state_dict"] if "state_dict" in checkpoint else checkpoint
        if "image_adapter.rel_pos_table_list.0.weight" in state_dict:
            state_dict["image_adapter.rel_pos_table.weight"] = state_dict.pop("image_adapter.rel_pos_table_list.0.weight").clone()
        own = self.state_dict()
        for key in list(state_dict.keys()):
            if "image_adapter.rp_bucket" in key:
                state_dict.pop(key)
            if "rel_pos_table.weight" in key and key in own:
                table = state_dict[key]
                src_num_pos, heads = table.size()
                src = int((src_num_pos - 3) ** 0.5)
                dst = int((own[key].shape[0] - 3) ** 0.5)
                if src != dst:
                    new = geometric_sequence_interpolation(src, dst, table[:-3], heads)
                    state_dict[key] = torch.cat((new, table[-3:]), dim=0)
        return state_dict

    def init_weights(self, pretrained=None):
        """onepeace.py:611-665: trunc-normal Linear weights, unit LayerNorms, then the pickled checkpoint (if any), then
        every adapter's D_fc2 zeroed."""
        def _init_weights(m):
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.LayerNorm):
                nn.init.constant_(m.bias, 0)
                nn.init.constant_(m.weight, 1.0)

        if pretrained:
            self.pretrained = pretrained
        if isinstance(self.pretrained, str):
            self.apply(_init_weights)
            with open(self.pretrained, "rb") as fh:
                model = pickle.load(fh, encoding="latin1")["model"]
            self.resize_abs_pos_embed(model)
            state_dict = self.resize_rel_pos_embed(model)
            msg = self.load_state_dict(state_dict, strict=False)
            if _get_rank() == 0:
                print(f"Missing keys: {msg.missing_keys}\nUnexpected keys: {msg.unexpected_keys}\n"
                      f"=> loaded successfully '{self.pretrained}'")
        elif self.pretrained is None:
            self.apply(_init_weights)
        else:
            raise TypeError("pretrained must be a str or None")
        with torch.no_grad():
            for layer in self.encoder.layers:
                for adapter in (layer.S_Adapter, layer.T_Adapter, layer.MLP_Adapter):
                    adapter.D_fc2.weight.zero_()
                    adapter.D_fc2.bias.zero_()

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"image_adapter.pos_embed", "image_adapter.cls_embedding", "image_adapter.temporal_embedding"}

    def get_num_layers(self):
        return len(self.encoder.layers)

    def _rows(self, x):
        """-> (fp32 frame-major rows [B T N, d] after the last layer, B, T, N)."""
        ad = self.image_adapter
        side, T = ad.bucket_size, ad.num_frames
        if x is None or x.dim() != 5 or tuple(x.shape[1:]) != (3, T, 16 * side, 16 * side):
            raise ValueError(f"OnePeaceViT with num_frames {T} and bucket_size {side} takes [B, 3, {T}, {16 * side}, "
                             f"{16 * side}] clips, got {None if x is None else tuple(x.shape)}")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("OnePeaceViT: only evaluation is built; run under torch.no_grad() (mmaction's test "
                                      "loop does)")
        for layer in self.encoder.layers:
            layer.check_structure()
        B, N = x.shape[0], side * side + 1
        frames = x.transpose(1, 2).reshape(B * T, 3, 16 * side, 16 * side)
        if frames.dtype not in (torch.float32, torch.bfloat16):
            frames = frames.float()
        rows = ad.stem(frames.contiguous())
        self.encoder.run(rows, ad.lut_bias(), B, T, N)
        return rows, B, T, N

    def _final_norm(self):
        ln = self.encoder.image_layer_norm
        return f32(ln.weight), f32(ln.bias), ln.eps

    def forward_features(self, x=None):
        """-> image_layer_norm of every row, fp32 [N, B T, d] (onepeace.py:678-682)."""
        with torch.autocast("cuda", enabled=False):
            rows, B, T, N = self._rows(x)
            w, b, eps = self._final_norm()
            out = K.layernorm(rows, w, b, torch.empty_like(rows), eps=eps)
            return out.view(B * T, N, -1).transpose(0, 1)

    def forward(self, x=None):
        """-> image_layer_norm of the CLS rows, fp32 [B, d, T, 1, 1] (onepeace.py:684-691); autocast does not change it."""
        with torch.autocast("cuda", enabled=False):
            rows, B, T, N = self._rows(x)
            d = rows.shape[1]
            w, b, eps = self._final_norm()
            cls = K.layernorm(rows, w, b, torch.empty(B * T, d, dtype=torch.float32, device=rows.device), rows=B * T,
                              ld_in=N * d, ld_out=d, eps=eps)
            return cls.view(B, T, d).permute(0, 2, 1).contiguous()[..., None, None]
