"""Drop-in for the Kinetics-400 action-recognition backbone of the vision branch,
``one_peace_vision/video/mmaction_custom/models/backbones/onepeace.py`` (``OnePeaceViT``), as
``configs/recognition/onepeace_k400*.py`` builds it.

The module tree, parameter and buffer names, shapes, dtypes and registration order are the reference's, so
``onepeace_video_k400.pth`` loads through mmcv's ``load_checkpoint`` and the configs' ``paramwise_cfg`` keys match.
Evaluation (eval mode):

    input                           NCTHW clips, reordered to (b t) c h w frames (a copy)
    hMLP stem, CLS + positions      autograd.ImageEmbedFn (three patch GEMMs), then one row_gather adds temporal_embedding[t]
                                    to every row of frame t, CLS row included: ((patch + pos) + temporal) in fp32
    rows                            frame-major, row (b T + t) N + n with N = bucket^2 + 1, fp32 residual stream
    layers                          VideoLayer.forward_video: the temporal pass attends along t at a row stride of N
                                    (csrc/attention_temporal.cu), the spatial pass over the N rows of each frame with the
                                    shared relative-position table in LUT form; every LayerNorm is folded into the GEMM
                                    that reads it, as in TransformerEncoderLayer.forward_rows_fused
    output                          image_layer_norm of the CLS rows only -> fp32 [B, d, T, 1, 1] for mmaction's I3DHead

Fine-tuning (train mode, as mmaction's train_step runs it): ImageEmbedFn -> TemporalEmbedFn -> VideoStackFn ->
ClsNormFn (FinalNormFn for forward_features).  VideoStackFn runs video_layer_forward, the un-fused LayerNorm form of the
layer with the two passes' attention rows stacked, and its adjoint video_layer_backward (the temporal pass through
opb_attention_temporal_bwd, the spatial pass through opb_attention_bwd with the dense table from RelPosBiasFn, whose
gradient sums over the layers).  Drop-path draws one mask per frame for each of the three branches (draw_row_scales).
Activations are kept or recomputed per autograd.keep_activations.  Parameters with requires_grad=False get no gradient.

Refused in the constructor, as no config uses them: dropout, attention_dropout or activation_dropout > 0,
``rp_bias=True``, ``shared_rp_bias=False`` and ``num_tadapter=2``.  ``forward`` raises ValueError for an input that is
not [B, 3, num_frames, 16 bucket, 16 bucket] and, in eval mode, NotImplementedError when a gradient is required (the
evaluation path has no backward).
"""
import pickle

import torch
import torch.nn as nn

from .. import kernels as K
from .. import relpos
from . import _get_rank, resize_abs_pos_embed
from ..adapter.image import (geometric_sequence_interpolation, hmlp_stem, hmlp_stem_tensors, image_lut_bias,
                             make_image_bucket_position)
from ..autograd import (ImageEmbedFn, RelPosBiasFn, _dw, _dx, ffn_params, ffn_train_pack, keep_activations, shared_params,
                        shared_train_pack)
from ..autograd_general import FinalNormFn
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
        self.embed_images = hmlp_stem(embed_dim)
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
        x = ImageEmbedFn.apply(frames, self.pos_embed, *hmlp_stem_tensors(self.embed_images), self.cls_embedding)
        BT, N, d = x.shape
        idx = torch.arange(BT * N, dtype=torch.int64, device=x.device)
        return K.row_gather(x.view(BT * N, d), idx, add=self.temporal_rows(N))         # row (b T + t) N + n gains temporal[t]

    def temporal_rows(self, N):
        """fp32 [T N, d]: temporal_embedding[0, t] repeated over the N rows of frame t (rebuilt when the table changes)."""
        add = self._temporal_cache.get([self.temporal_embedding],
                                       lambda: f32(self.temporal_embedding[0]).repeat_interleave(N, dim=0).contiguous())
        assert add.shape[0] == self.num_frames * N
        return add

    def train_rows(self, frames, encoder):
        """Training forward of the stem, the temporal embedding and the layer stack: frames [B T, 3, R, R] clip-major ->
        autograd-tracked fp32 frame-major rows [B T N, d] after the last layer."""
        x = ImageEmbedFn.apply(frames, self.pos_embed, *hmlp_stem_tensors(self.embed_images), self.cls_embedding)
        BT, N, d = x.shape
        T = self.num_frames
        x = TemporalEmbedFn.apply(x.view(BT * N, d), self.temporal_embedding, self.temporal_rows(N), BT // T, T, N)
        bias = RelPosBiasFn.apply(self.rel_pos_table.weight, self.rp_bucket, N, encoder.num_attention_heads)
        params = [q for layer in encoder.layers for q in video_params(layer)]
        return VideoStackFn.apply(encoder, (BT // T, T, N, self.lut_bias(), torch.is_grad_enabled()), x, bias, *params)

    def lut_bias(self):
        """The shared table in LUT form for the spatial pass over S = bucket^2 + 1 rows (rebuilt when the table changes)."""
        S = self.bucket_size ** 2 + 1
        if S > K.ATTN_TC_MAX_S:
            raise NotImplementedError(f"OnePeaceViT: bucket_size {self.bucket_size} gives {S} tokens per frame; the LUT-form "
                                      f"attention is built for at most {K.ATTN_TC_MAX_S}")
        return image_lut_bias(self._lut_cache, self.rel_pos_table.weight, self.rp_bucket, self.bucket_size)


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


# ----------------------------------------------------------------------------------------------------------------
# training: un-fused forward and adjoint of one VideoLayer, the layer stack, and the Functions around it
# ----------------------------------------------------------------------------------------------------------------
def adapter_params(layer):
    """The 12 adapter parameters of a VideoLayer, T, S then MLP adapter, each fc1 weight, fc1 bias, fc2 weight, fc2 bias."""
    return [q for ad in (layer.T_Adapter, layer.S_Adapter, layer.MLP_Adapter)
            for q in (ad.D_fc1.weight, ad.D_fc1.bias, ad.D_fc2.weight, ad.D_fc2.bias)]


def video_params(layer):
    """Per layer, in the order video_layer_backward returns their gradients: the 15 shared_params, the 6 image FFN
    parameters, the 12 adapter_params."""
    return shared_params(layer) + ffn_params(layer, "image") + adapter_params(layer)


def adapter_train_pack(layer):
    cache = layer._cache.setdefault("_train_adapters", PackCache())
    ps = adapter_params(layer)

    def build():
        names = [f"{a}{k}" for a in "tsm" for k in ("1w", "1b", "2w", "2b")]
        pk = {n: (bf16(q) if n.endswith("w") else f32(q)) for n, q in zip(names, ps)}
        pk["scale"] = torch.full((layer.embed_dim,), float(layer.scale), dtype=torch.float32, device=ps[0].device)
        return pk
    return cache.get(ps, build)


def video_row_bytes(d, ffn, H):
    """Bytes per row that video_layer_forward keeps for the adjoint: both passes' h1, qkv, att, a2, o (bf16, 2 rows each),
    the adapters' pre-activations and activations (d / 4 wide, bf16), xt, s, h2, f, mo (bf16), y and x1 (fp32), the FFN's
    gl, u, u2 (bf16) and the spatial pass's log-sum-exp."""
    return 2 * 2 * 7 * d + 6 * 2 * (d // 4) + 5 * 2 * d + 2 * 4 * d + 4 * 2 * ffn + 4 * H


_IDX = {}


def _iota(M, device):
    key = (M, device)
    if key not in _IDX:
        _IDX[key] = torch.arange(M, dtype=torch.int64, device=device)
    return _IDX[key]


def video_layer_forward(layer, x, Bv, T, N, fast_bias, rs, keep):
    """x fp32 [Bv T N, d] frame-major rows -> (layer output fp32 [Bv T N, d], saved activations or None).  Un-fused
    LayerNorm form of onepeace.py:328-352 (num_tadapter = 1), so that every normalised operand of the dW GEMMs is in HBM:

        h1 = LN1(x);  a_t = out_proj(LN_in(TemporalAttn(QKV(h1))));   xt = T_Adapter(a_t);   y = x + rs[0] xt
        h1s = LN1(y); a_s = out_proj(LN_in(SpatialAttn(QKV(h1s))));  s = a_s + S_Adapter'(a_s)
        x1 = x + rs[1] gamma_1 s;  h2 = LN2(x1);  x_out = x1 + gamma_2 FFN(h2) + rs[2] scale MLP_Adapter(h2)

    rs: three fp32 [Bv T N] drop-path row scales (per frame) or Nones.  The two passes' QKV, attention, LN_in and out_proj
    rows are stacked, temporal first, in [2M, .] buffers, so that the adjoint forms each shared weight's gradient with one
    GEMM over 2M rows.  fast_bias: the shared table in LUT form for the spatial pass."""
    p, fp, ad = shared_train_pack(layer), ffn_train_pack(layer, "image"), adapter_train_pack(layer)
    d, F_, H = layer.embed_dim, layer.ffn_embed_dim, layer.self_attn.num_heads
    M, dh, dev = x.shape[0], ad["t1w"].shape[0], x.device
    eps1, eps_in, eps2 = layer.self_attn_layer_norm.eps, layer.self_attn.ln.eps, layer.final_layer_norm.eps

    def e(rows, n, dt=torch.bfloat16):
        return torch.empty(rows, n, dtype=dt, device=dev)
    h1, qkv, att, a2, o = e(2 * M, d), e(2 * M, 3 * d), e(2 * M, d), e(2 * M, d), e(2 * M, d)
    tp, sp = slice(0, M), slice(M, 2 * M)

    def attn_in(rows, part):
        K.layernorm(rows, p["ln1_w"], p["ln1_b"], h1[part], eps=eps1)
        K.gemm(h1[part], p["wqkv"], K.EPI_STORE_BF16, qkv[part], bias=p["bqkv"], colscale=p["qscale"])

    def attn_out(part):
        K.layernorm(att[part], p["lni_w"], p["lni_b"], a2[part], eps=eps_in)
        K.gemm(a2[part], p["wo"], K.EPI_STORE_BF16, o[part], bias=p["bo"])

    def fc1(a_in, w, b):
        z = K.gemm(a_in, w, K.EPI_STORE_BF16, e(M, dh), bias=b)
        return z, K.gelu_fwd(z, e(M, dh))
    # temporal pass
    attn_in(x, tp)
    K.attention_temporal(qkv[tp], Bv, T, N, H, out=att[tp], ln_stats=torch.empty(H, M, 2, device=dev))
    attn_out(tp)
    zt, ht = fc1(o[tp], ad["t1w"], ad["t1b"])
    xt = K.gemm(ht, ad["t2w"], K.EPI_STORE_BF16, e(M, d), bias=ad["t2b"])
    y = K.scale_resid_fwd(x, xt, None, rs[0], torch.empty_like(x))
    # spatial pass
    attn_in(y, sp)
    lse = torch.empty(M * H, dtype=torch.float32, device=dev)
    K.attention_tc(qkv[sp], fast_bias, None, Bv * T, N, H, out=att[sp], lse=lse)
    attn_out(sp)
    zs, hs = fc1(o[sp], ad["s1w"], ad["s1b"])
    s2 = K.gemm(hs, ad["s2w"], K.EPI_STORE_F32, e(M, d, torch.float32), bias=ad["s2b"])
    sb = K.row_gather(o[sp], _iota(M, dev), out=e(M, d), add=s2)                   # s = a_s + S_fc2(gelu(S_fc1(a_s)))
    x1 = K.scale_resid_fwd(x, sb, p["g1"], rs[1], torch.empty_like(x))
    # joint pass
    h2 = K.layernorm(x1, p["ln2_w"], p["ln2_b"], e(M, d), eps=eps2)
    gl = K.gemm(h2, fp["w01"], K.EPI_STORE_BF16, e(M, 2 * F_))
    u = K.geglu_fwd(gl, e(M, F_))
    u2 = K.layernorm(u, fp["lnf_w"], fp["lnf_b"], e(M, F_), eps=fp["lnf_eps"])
    f = K.gemm(u2, fp["w2"], K.EPI_STORE_BF16, e(M, d), bias=fp["b2"])
    zm, hm = fc1(h2, ad["m1w"], ad["m1b"])
    mo = K.gemm(hm, ad["m2w"], K.EPI_STORE_BF16, e(M, d), bias=ad["m2b"])
    x2 = K.scale_resid_fwd(x1, f, p["g2"], None, torch.empty_like(x))               # no drop-path on the FFN term
    x3 = K.scale_resid_fwd(x2, mo, ad["scale"], rs[2], torch.empty_like(x))
    saved = dict(h1=h1, qkv=qkv, att=att, a2=a2, o=o, lse=lse, zt=zt, ht=ht, xt=xt, y=y, zs=zs, hs=hs, sb=sb, x1=x1,
                 h2=h2, gl=gl, u=u, u2=u2, f=f, zm=zm, hm=hm, mo=mo) if keep else None
    return x3, saved


def video_layer_backward(layer, x, s, dx, Bv, T, N, bias, dbias, rs):
    """Adjoint of video_layer_forward.  dx fp32 [M, d] = dL/dx_out (overwritten); bias: the dense fp32 (H, N, N_pad) table
    of the spatial pass; dbias (same shape) accumulates its gradient.  Returns (dL/dx fp32 [M, d], the video_params
    gradients in each parameter's dtype)."""
    p, fp, ad = shared_train_pack(layer), ffn_train_pack(layer, "image"), adapter_train_pack(layer)
    d, F_, H = layer.embed_dim, layer.ffn_embed_dim, layer.self_attn.num_heads
    M, dh, dev = x.shape[0], ad["t1w"].shape[0], x.device
    idx = _iota(M, dev)
    tp, sp = slice(0, M), slice(M, 2 * M)
    sps = video_params(layer)

    def e(rows, n, dt=torch.bfloat16):
        return torch.empty(rows, n, dtype=dt, device=dev)

    def g(*n):
        return torch.empty(*n, dtype=torch.float32, device=dev)

    def adapter_bwd(dout, z, h, a_in, w1, w2, dx_out):
        """dout bf16 [M, d] = dL/d(fc2 output) -> fc2 weight, fc1 weight and bias gradients; dL/d(adapter input) into
        dx_out (fp32 or bf16)."""
        dW2 = _dw(dout, h, torch.float32)
        dz = K.gelu_bwd(z, _dx(dout, w2, dh), e(M, dh))
        db1 = K.colsum(dz, g(dh))
        dW1 = _dw(dz, a_in, torch.float32)
        _dx(dz, w1, d, out=dx_out)
        return dW1, db1, dW2
    # joint pass: x_out = x1 + gamma_2 f + rs[2] scale mo, both branches reading h2 = LN2(x1)
    dm2b, dg2, db2 = g(d), g(d), g(d)
    dmo = K.scale_resid_bwd(dx, s["mo"], ad["scale"], rs[2], e(M, d), dbias=dm2b)
    dh2m = g(M, d)
    dm1w, dm1b, dm2w = adapter_bwd(dmo, s["zm"], s["hm"], s["h2"], ad["m1w"], ad["m2w"], dh2m)
    df = K.scale_resid_bwd(dx, s["f"], p["g2"], None, e(M, d), dgamma=dg2, dbias=db2)
    dW2 = _dw(df, s["u2"], torch.float32)
    dlnf_w, dlnf_b = g(F_), g(F_)
    du = K.layernorm_bwd(s["u"], _dx(df, fp["w2"], F_), fp["lnf_w"], fp["lnf_b"], e(M, F_), eps=fp["lnf_eps"],
                         dgamma=dlnf_w, dbeta=dlnf_b)
    dgl = K.geglu_bwd(s["gl"], du, e(M, 2 * F_))
    dW01 = _dw(dgl, s["h2"], torch.float32)
    dh2 = K.row_gather(_dx(dgl, fp["w01"], d), idx, out=e(M, d), add=dh2m)             # FFN + MLP_Adapter shares
    dln2_w, dln2_b = g(d), g(d)
    K.layernorm_bwd(s["x1"], dh2, p["ln2_w"], p["ln2_b"], dx, eps=layer.final_layer_norm.eps, accumulate=True,
                    dgamma=dln2_w, dbeta=dln2_b)                                       # dx = dL/dx1
    # spatial pass: x1 = x + rs[1] gamma_1 s, s = a_s + S_Adapter'(a_s)
    dg1, ds2b = g(d), g(d)
    dsb = K.scale_resid_bwd(dx, s["sb"], p["g1"], rs[1], e(M, d), dgamma=dg1, dbias=ds2b)
    das = g(M, d)
    ds1w, ds1b, ds2w = adapter_bwd(dsb, s["zs"], s["hs"], s["o"][sp], ad["s1w"], ad["s2w"], das)
    do, da2, datt, dqkv, dh1 = e(2 * M, d), e(2 * M, d), e(2 * M, d), e(2 * M, 3 * d), e(2 * M, d)
    K.row_gather(dsb, idx, out=do[sp], add=das)                                        # the S_Adapter's skip term
    dlni, dln1 = g(2, 2, d), g(2, 2, d)                                                # [pass, (weight, bias), d]
    eps1, eps_in = layer.self_attn_layer_norm.eps, layer.self_attn.ln.eps

    def attn_bwd_to_datt(part, k):
        _dx(do[part], p["wo"], d, out=da2[part])
        K.layernorm_bwd(s["att"][part], da2[part], p["lni_w"], p["lni_b"], datt[part], eps=eps_in, dgamma=dlni[k, 0],
                        dbeta=dlni[k, 1])
    attn_bwd_to_datt(sp, 1)
    K.attention_bwd(s["qkv"][sp], s["att"][sp], datt[sp], bias, None, s["lse"], dqkv[sp], dbias, Bv * T, N, H,
                    layer.self_attn.scaling)
    _dx(dqkv[sp], p["wqkv"], d, out=dh1[sp])
    dy = K.layernorm_bwd(s["y"], dh1[sp], p["ln1_w"], p["ln1_b"], g(M, d), eps=eps1, dgamma=dln1[1, 0], dbeta=dln1[1, 1])
    dx = K.row_gather(dy, idx, out_dtype=torch.float32, add=dx)                         # y = x + rs[0] xt
    # temporal pass
    dt2b = g(d)
    dxt = K.scale_resid_bwd(dy, s["xt"], None, rs[0], e(M, d), dbias=dt2b)
    dt1w, dt1b, dt2w = adapter_bwd(dxt, s["zt"], s["ht"], s["o"][tp], ad["t1w"], ad["t2w"], do[tp])
    attn_bwd_to_datt(tp, 0)
    K.attention_temporal_bwd(s["qkv"][tp], s["att"][tp], datt[tp], Bv, T, N, H, layer.self_attn.scaling, dqkv=dqkv[tp])
    _dx(dqkv[tp], p["wqkv"], d, out=dh1[tp])
    K.layernorm_bwd(x, dh1[tp], p["ln1_w"], p["ln1_b"], dx, eps=eps1, accumulate=True, dgamma=dln1[0, 0],
                    dbeta=dln1[0, 1])
    # the weights both passes share: one reduction over the 2M stacked rows
    dWo, dbo = _dw(do, s["a2"], torch.float32), K.colsum(do, g(d))
    dWqkv, dbqkv = _dw(dqkv, s["h1"], torch.float32), K.colsum(dqkv, g(3 * d))
    dlni = K.batch_sum(dlni, g(2, d), 2, 2 * d, 2 * d)
    dln1 = K.batch_sum(dln1, g(2, d), 2, 2 * d, 2 * d)
    grads = [dWqkv[:d], dbqkv[:d], dWqkv[d:2 * d], dWqkv[2 * d:], dbqkv[2 * d:], dWo, dbo, dlni[0], dlni[1], dln1[0],
             dln1[1], dln2_w, dln2_b, dg1, dg2,
             dW01[:F_], dW01[F_:], dlnf_w, dlnf_b, dW2, db2,
             dt1w, dt1b, dt2w, dt2b, ds1w, ds1b, ds2w, ds2b, dm1w, dm1b, dm2w, dm2b]
    return dx, [gr if gr.dtype == prm.dtype else gr.to(prm.dtype) for gr, prm in zip(grads, sps)]


def draw_row_scales(layers, Bv, T, N, device):
    """Drop-path row scales of every layer in train mode (onepeace.py:328-352: drop_path with a (1, B T, 1) mask on the
    'n (b t) d' layout, i.e. one draw per frame).  Layer by layer, for each of the temporal, spatial and MLP-adapter
    branches in that order: one torch.rand(Bv T) on `device`, keep = draw < 1 - p, scale = keep / (1 - p) on the N rows of
    the frame.  Layers with drop_path_prob 0 draw nothing and get (None, None, None)."""
    out = []
    for layer in layers:
        pdrop = layer.drop_path_prob if layer.training else 0.0
        if pdrop <= 0:
            out.append((None, None, None))
            continue
        keep = 1.0 - pdrop
        out.append(tuple(((torch.rand(Bv * T, device=device) < keep).float() / keep).repeat_interleave(N).contiguous()
                         for _ in range(3)))
    return out


class VideoStackFn(torch.autograd.Function):
    """x0 fp32 [Bv T N, d] frame-major rows -> x_L through every VideoLayer (onepeace.py:409-414), with the dense
    relative-position table `bias` (H, N, N_pad) shared by the layers' spatial passes (its LUT form `fast` runs the
    forward).  meta = (Bv, T, N, fast, need_grad).  Activations are kept when they fit (autograd.keep_activations with
    video_row_bytes), otherwise each layer's input rows are kept and the layer is recomputed before its adjoint.  The
    table gradient is summed over the layers and projected onto zero row sums, as for EncoderStackFn's shared tables."""

    @staticmethod
    def forward(ctx, encoder, meta, x0, bias, *params):
        Bv, T, N, fast, need_grad = meta
        layers = list(encoder.layers)
        x = x0.contiguous()
        d, ffn, H = x.shape[1], encoder.cfg.ffn_embed_dim, encoder.num_attention_heads
        scales = draw_row_scales(layers, Bv, T, N, x.device)
        keep = need_grad and keep_activations(len(layers), x.shape[0], d, ffn, x.device, row_bytes=video_row_bytes(d, ffn, H))
        xs, saved_all = [], []
        for layer, rs in zip(layers, scales):
            if need_grad:
                xs.append(x)
            x, saved = video_layer_forward(layer, x, Bv, T, N, fast, rs, keep)
            saved_all.append(saved)
        ctx.encoder, ctx.meta, ctx.bias = encoder, meta, bias
        ctx.xs, ctx.scales, ctx.saved_all = xs, scales, saved_all
        if need_grad:
            encoder.activations = "keep" if keep else "recompute"      # the policy of the last training step, for reports
        return x

    @staticmethod
    def backward(ctx, grad_out):
        Bv, T, N, fast, _ = ctx.meta
        layers = list(ctx.encoder.layers)
        dx = grad_out.to(torch.float32).contiguous().clone()
        dbias = torch.zeros_like(ctx.bias)
        grads = [None] * len(layers)
        for i in reversed(range(len(layers))):
            saved, ctx.saved_all[i] = ctx.saved_all[i], None
            if saved is None:
                _, saved = video_layer_forward(layers[i], ctx.xs[i], Bv, T, N, fast, ctx.scales[i], True)
            dx, grads[i] = video_layer_backward(layers[i], ctx.xs[i], saved, dx, Bv, T, N, ctx.bias, dbias, ctx.scales[i])
            ctx.xs[i] = None
            del saved
        K.relpos_dbias_center(dbias)
        flat = [gr for lg in grads for gr in lg]
        flat = [gr if need else None for gr, need in zip(flat, ctx.needs_input_grad[4:])]
        return (None, None, dx, dbias if ctx.needs_input_grad[3] else None, *flat)


class TemporalEmbedFn(torch.autograd.Function):
    """x fp32 [Bv T N, d] + temporal_embedding[0, t] on every row of frame t, CLS row included (onepeace.py:199-201), by one
    row_gather.  Adjoint: dx passes through; d temporal [1, num_frames, d] is the sum of the rows of frame t over the clips
    and tokens: one row_gather into (b n, t) order, then one batch_sum over the Bv N groups of T rows."""

    @staticmethod
    def forward(ctx, x, temporal, add, Bv, T, N):
        ctx.meta = (Bv, T, N, temporal.shape, temporal.dtype)
        return K.row_gather(x, _iota(x.shape[0], x.device), add=add)

    @staticmethod
    def backward(ctx, dout):
        Bv, T, N, shape, dt = ctx.meta
        dout = dout.to(torch.float32).contiguous()
        d, dev = dout.shape[1], dout.device
        b = torch.arange(Bv, device=dev).view(Bv, 1, 1)
        n = torch.arange(N, device=dev).view(1, N, 1)
        t = torch.arange(T, device=dev).view(1, 1, T)
        by_token = K.row_gather(dout, ((b * T + t) * N + n).reshape(-1).contiguous())     # row (b N + n) T + t
        dtemp = torch.zeros(shape, dtype=torch.float32, device=dev)
        K.batch_sum(by_token, dtemp, Bv * N, T * d, T * d)
        return dout, dtemp.to(dt), None, None, None, None


class ClsNormFn(torch.autograd.Function):
    """image_layer_norm of the CLS rows of frame-major rows [Bv T N, d] (onepeace.py:684-691) -> fp32 [Bv T, d]; the adjoint
    writes the CLS rows only."""

    @staticmethod
    def forward(ctx, rows, w, b, eps, N):
        BT, d = rows.shape[0] // N, rows.shape[1]
        rows = rows.contiguous()
        out = K.layernorm(rows, f32(w), f32(b), torch.empty(BT, d, dtype=torch.float32, device=rows.device), rows=BT,
                          ld_in=N * d, ld_out=d, eps=eps)
        ctx.save_for_backward(rows, w, b)
        ctx.meta = (eps, N)
        return out

    @staticmethod
    def backward(ctx, dy):
        rows, w, b = ctx.saved_tensors
        eps, N = ctx.meta
        d = rows.shape[1]
        BT = rows.shape[0] // N
        dg = torch.empty(d, dtype=torch.float32, device=rows.device)
        db = torch.empty(d, dtype=torch.float32, device=rows.device)
        dx = torch.zeros_like(rows)
        K.layernorm_bwd(rows, dy.to(torch.float32).contiguous(), f32(w), f32(b), dx, eps=eps, dgamma=dg, dbeta=db, rows=BT,
                        dim=d, ldx=N * d, ld_dx=N * d)
        return dx, dg.to(w.dtype), db.to(b.dtype), None, None


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

    resize_abs_pos_embed = resize_abs_pos_embed

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
        if not self.training and torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("OnePeaceViT: the evaluation path has no backward; run it under torch.no_grad() "
                                      "(mmaction's test loop does), or train in train mode")
        for layer in self.encoder.layers:
            layer.check_structure()
        B, N = x.shape[0], side * side + 1
        frames = x.transpose(1, 2).reshape(B * T, 3, 16 * side, 16 * side)
        if frames.dtype not in (torch.float32, torch.bfloat16):
            frames = frames.float()
        if self.training:
            return ad.train_rows(frames.contiguous(), self.encoder), B, T, N
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
            if self.training:
                ln = self.encoder.image_layer_norm
                return FinalNormFn.apply(rows, ln.weight, ln.bias, ln.eps).view(B * T, N, -1).transpose(0, 1)
            w, b, eps = self._final_norm()
            out = K.layernorm(rows, w, b, torch.empty_like(rows), eps=eps)
            return out.view(B * T, N, -1).transpose(0, 1)

    def forward(self, x=None):
        """-> image_layer_norm of the CLS rows, fp32 [B, d, T, 1, 1] (onepeace.py:684-691); autocast does not change it."""
        with torch.autocast("cuda", enabled=False):
            rows, B, T, N = self._rows(x)
            d = rows.shape[1]
            if self.training:
                ln = self.encoder.image_layer_norm
                cls = ClsNormFn.apply(rows, ln.weight, ln.bias, ln.eps, N)
                return cls.view(B, T, d).permute(0, 2, 1).contiguous()[..., None, None]
            w, b, eps = self._final_norm()
            cls = K.layernorm(rows, w, b, torch.empty(B * T, d, dtype=torch.float32, device=rows.device), rows=B * T,
                              ld_in=N * d, ld_out=d, eps=eps)
            return cls.view(B, T, d).permute(0, 2, 1).contiguous()[..., None, None]
