"""Drop-in for ``TransformerEncoderLayer`` / ``GeGLU`` (models/transformer/transformer_layer.py:54-228).

Parameter names match the reference (self_attn.*, self_attn_layer_norm, {text,image,audio}_ffn.{0.wi_0,
0.wi_1,2,3}, final_layer_norm, gamma_1, gamma_2).  One layer forward (forward_rows_fused) = 4 wgmma GEMMs
+ 1 attention kernel: each of the four LayerNorms is folded into the GEMM that reads its output, with the row
statistics taken from the epilogue of the kernel that wrote the rows.  The residual stream stays fp32 in HBM and is
updated in place by the out_proj / fc2 GEMM epilogues (gamma * (acc + bias) + residual — `fused_dropout_res`, :70-88,
eval mode).  The training forward that keeps the normalised activations is autograd.layer_forward.
"""
import torch
import torch.nn as nn

from .. import kernels as K
from ..components import LayerNorm, Linear, PackCache, f32
from .multihead_attention import MultiheadAttention


class GeGLU(nn.Module):
    """models/transformer/transformer_layer.py:54-67 — parameter container (wi_0, wi_1: no bias)."""

    def __init__(self, embed_dim, ffn_dim):
        super().__init__()
        self.wi_0 = Linear(embed_dim, ffn_dim, bias=False)
        self.wi_1 = Linear(embed_dim, ffn_dim, bias=False)


class TransformerEncoderLayer(nn.Module):
    def __init__(self, cfg, drop_path_rate=0.0):
        super().__init__()
        self.cfg = cfg
        self.embed_dim = cfg.embed_dim
        self.ffn_embed_dim = cfg.ffn_embed_dim
        self.self_attn = MultiheadAttention(self.embed_dim, cfg.attention_heads, dropout=cfg.attention_dropout,
                                            scale_heads=cfg.scale_heads, magneto_scale_attn=cfg.magneto_scale_attn)
        self.self_attn_layer_norm = LayerNorm(self.embed_dim)
        self.dropout_prob = cfg.dropout
        self.drop_path_prob = drop_path_rate
        if cfg.use_text_moe:
            self.text_ffn = self.build_geglu_ffn(cfg)
        if cfg.use_image_moe:
            self.image_ffn = self.build_geglu_ffn(cfg)
        if cfg.use_audio_moe:
            self.audio_ffn = self.build_geglu_ffn(cfg)
        self.attn_ln = LayerNorm(self.embed_dim) if cfg.scale_attn else None
        self.final_layer_norm = LayerNorm(self.embed_dim)
        self.gamma_1 = None
        self.gamma_2 = None
        if cfg.use_layer_scale:
            self.gamma_1 = nn.Parameter(cfg.layer_scale_init_value * torch.ones((self.embed_dim)), requires_grad=True)
            self.gamma_2 = nn.Parameter(cfg.layer_scale_init_value * torch.ones((self.embed_dim)), requires_grad=True)
        self._cache = {}

    def build_geglu_ffn(self, cfg):
        # indices 0..3 match the reference Sequential (GeGLU, act-dropout, LayerNorm | Identity, Linear)
        return nn.Sequential(GeGLU(self.embed_dim, self.ffn_embed_dim), nn.Identity(),
                             LayerNorm(self.ffn_embed_dim) if cfg.scale_fc else nn.Identity(),
                             Linear(self.ffn_embed_dim, self.embed_dim))

    def check_structure(self):
        """The forward and backward kernels are built for the layer structure of the recipes; any other raises."""
        ffn_ok = all(isinstance(getattr(self, f"{m}_ffn")[2], nn.LayerNorm) for m in ("text", "image", "audio")
                     if hasattr(self, f"{m}_ffn"))
        if self.self_attn.ln is None or not ffn_ok or self.attn_ln is not None or self.self_attn.c_attn is not None:
            raise NotImplementedError("the encoder layer is built for the 4B layer structure (magneto_scale_attn, scale_fc on; "
                                      "scale_attn, scale_heads off — finetune_3B.yaml:114-132)")

    # ------------------------------------------------------------------------------------------------
    # fused-LayerNorm path: the four LayerNorms of the layer never run as kernels.  Each GEMM consumes the
    # UN-normalised bf16 rows and applies  rstd * (acc - mu * colsum) + bias'  in its epilogue (gemm.h); the row
    # statistics come from the epilogue of the kernel that produced those rows.
    # ------------------------------------------------------------------------------------------------

    @staticmethod
    def _fold(weights, ln, biases, interleave=False):
        """Folds LayerNorm `ln` into the Linear layers `weights` ([N_i, K] each, stacked along N; `interleave`: the GeGLU tile
        interleave of two weights) -> (bf16 W*diag(g) [sum N_i, K], colsum of the bf16 rows, bias' = W @ beta + b).
        One `opb_ln_fold` launch per source weight (csrc/pack.cu): the packs are rebuilt after every optimizer step."""
        dev = weights[0].device
        N, Kd = sum(w.shape[0] for w in weights), weights[0].shape[1]
        wg = torch.empty(N, Kd, dtype=torch.bfloat16, device=dev)
        colsum = torch.empty(N, dtype=torch.float32, device=dev)
        bias_out = torch.empty(N, dtype=torch.float32, device=dev)
        g, beta = f32(ln.weight), f32(ln.bias)
        off = 0
        for i, (w, b) in enumerate(zip(weights, biases)):
            wd = w.detach()
            if wd.dtype not in (torch.float32, torch.bfloat16):
                wd = wd.float()
            wd = wd.contiguous()
            bb = f32(b) if b is not None else None
            if interleave:
                K.ln_fold(wd, g, beta, bb, wg, colsum, bias_out, interleave=i + 1)
            else:
                n = w.shape[0]
                K.ln_fold(wd, g, beta, bb, wg[off:off + n], colsum[off:off + n], bias_out[off:off + n])
                off += n
        return wg, colsum, bias_out

    def _fused_attn_pack(self):
        cache = self._cache.setdefault("_fused_attn", PackCache())
        a = self.self_attn
        ps = [a.q_proj.weight, a.q_proj.bias, a.k_proj.weight, a.v_proj.weight, a.v_proj.bias, a.out_proj.weight,
              a.out_proj.bias, a.ln.weight, a.ln.bias, self.self_attn_layer_norm.weight, self.self_attn_layer_norm.bias] + \
             ([self.gamma_1] if self.gamma_1 is not None else [])

        def build():
            d = self.embed_dim
            dev = a.q_proj.weight.device
            w, c, dd = self._fold([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], self.self_attn_layer_norm,
                                  [a.q_proj.bias, None, a.v_proj.bias])
            qs = torch.ones(3 * d, device=dev)
            qs[:d] = a.scaling
            wo, co, do = self._fold([a.out_proj.weight], a.ln, [a.out_proj.bias])
            return dict(wqkv=w, cqkv=c, dqkv=dd, qscale=qs, wo=wo, co=co, do=do,
                        g1=f32(self.gamma_1) if self.gamma_1 is not None else None)
        return cache.get(ps, build)

    def _fused_ffn_pack(self, modality):
        cache = self._cache.setdefault("_fused_" + modality, PackCache())
        ffn = getattr(self, f"{modality}_ffn")
        ln2, lnf = self.final_layer_norm, ffn[2]
        ps = [ffn[0].wi_0.weight, ffn[0].wi_1.weight, ffn[3].weight, ffn[3].bias, lnf.weight, lnf.bias, ln2.weight,
              ln2.bias] + ([self.gamma_2] if self.gamma_2 is not None else [])

        def build():
            assert ffn[0].wi_0.weight.shape[0] % 128 == 0, "ffn_embed_dim must be a multiple of 128"
            w01, c01, d01 = self._fold([ffn[0].wi_0.weight, ffn[0].wi_1.weight], ln2, [None, None], interleave=True)
            w2, c2, d2 = self._fold([ffn[3].weight], lnf, [ffn[3].bias])
            return dict(w01=w01, c01=c01, d01=d01, w2=w2, c2=c2, d2=d2, lnf_eps=lnf.eps,
                        g2=f32(self.gamma_2) if self.gamma_2 is not None else None)
        return cache.get(ps, build)

    def forward_rows_fused(self, x, xb, ln1, ws, bias, key_pad, B, S, modality):
        """x fp32 [M,d] residual (in place), xb bf16 [M,d] copy of x, ln1 = LayerNorm-1 statistics of x: either
        dict(ln_mu=, ln_rstd=) (first layer) or dict(ln_partial=(records, parts, dim, eps)) (from the previous fc2).
        Returns the same for the layer output.  `ws` = workspace dict."""
        if self.training and (self.dropout_prob > 0 or self.drop_path_prob > 0):
            raise NotImplementedError("training-time dropout / drop-path: backward pass is not built yet")
        d, F_, H = self.embed_dim, self.ffn_embed_dim, self.self_attn.num_heads
        a = self._fused_attn_pack()
        f = self._fused_ffn_pack(modality)
        n_t = (d + 255) // 256
        # LN1 -> QKV (+bias, q scale)
        K.gemm_ln(xb, a["wqkv"], K.EPI_STORE_BF16, ws["qkv"], ln_colsum=a["cqkv"], bias=a["dqkv"], colscale=a["qscale"],
                  workspace=ws["tail"], **ln1)          # workspace: split-K slabs when M <= 256 (small batches)
        # attention; emits per-head partial statistics of its output rows (inner LN)
        self.self_attn.run_attention(ws["qkv"], bias, key_pad, B, S, out=ws["o"], ln_stats=ws["part_a"])
        # inner LN -> out_proj -> LayerScale + residual; emits x, xb and the partial statistics for LN2
        K.gemm_ln(ws["o"], a["wo"], K.EPI_RESID_F32, x, ln_partial=(ws["part_a"], H, d, self.self_attn.ln.eps),
                  ln_colsum=a["co"], bias=a["do"], gamma=a["g1"], resid=x, stats_out=ws["part_b"], out_bf16=xb,
                  workspace=ws["tail"])
        # LN2 -> GeGLU; emits u and the partial statistics for the FFN LayerNorm (96 records / row, reduced in the fc2 epilogue)
        K.gemm_ln(xb, f["w01"], K.EPI_GEGLU_BF16, ws["u"], ln_partial=(ws["part_b"], n_t, d, self.final_layer_norm.eps),
                  ln_colsum=f["c01"], bias=f["d01"], stats_out=ws["part_c"])
        # FFN LN -> fc2 -> LayerScale + residual; emits x, xb and the partial statistics for the next layer's LN1
        n_rec = 2 * ((2 * F_) // 256)                                                                     # 2 records / tile
        K.gemm_ln(ws["u"], f["w2"], K.EPI_RESID_F32, x, ln_partial=(ws["part_c"], n_rec, F_, f["lnf_eps"]), ln_colsum=f["c2"],
                  bias=f["d2"], gamma=f["g2"], resid=x, stats_out=ws["part_d"], out_bf16=xb, workspace=ws["tail"])
        return dict(ln_partial=(ws["part_d"], n_t, d, self.self_attn_layer_norm.eps))

    @staticmethod
    def fused_workspace(M, d, F_, H, device):
        n_t = (d + 255) // 256
        e = lambda *s, dt=torch.bfloat16: torch.empty(*s, dtype=dt, device=device)
        f32 = torch.float32
        return dict(qkv=e(M, 3 * d), o=e(M, d), u=e(M, F_), xb=e(M, d), part_a=e(H * M * 2, dt=f32),
                    part_b=e(n_t * M * 2, dt=f32), part_c=e(2 * ((2 * F_) // 256) * M * 2, dt=f32), part_d=e(n_t * M * 2, dt=f32),
                    tail=e(16 * 256 * d, dt=torch.float32),      # split-K slabs of the small-M GEMMs: one fp32 [M rounded up to 128, N] slab per piece
                    mu=e(M, dt=torch.float32), rstd=e(M, dt=torch.float32))
