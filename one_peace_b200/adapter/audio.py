"""Drop-in for ``AudioAdapter`` (models/adapter/audio.py:35-311): wav2vec-style conv feature extractor, conv
positional encoder, CLS, log-bucket relative-position bias.  Same parameter / buffer names
(embed_audios.0.conv_layers.N.{0,2.1}, embed_audios.{2,3}, embed_positions.{1..5}.0, cls_embedding,
cls_pos_embed, mask_embedding, rel_pos_table_list.N, rp_bucket).

Every convolution runs on the wgmma GEMM over channel-last activations (no transposes — the reference does
14 of them for the channel LayerNorms):
  * layer 0 (C_in = 1, k = 10, s = 5): a frame kernel writes the [frames, 16] bf16 operand (K padded 10 -> 16);
  * layers 1..6 (C = 512, k in {3, 2}, s = 2): the GEMM's A operand is an OVERLAPPING strided view of the previous
    layer's [frames, 512] output (row pitch s*512, row length k*512) — TMA reads it directly, nothing is
    materialised.  Per-clip frame buffers are allocated with pitch_k = 2 * pitch_{k+1} so that one uniform row
    stride covers the whole batch; the few slack rows compute garbage that no valid row ever reads;
  * the 5 positional convs (1536 ch, k = 19, pad 9, 16 groups) are grouped sliding-window GEMMs over a halo'd,
    group-padded (96 -> 128 channels) bf16 buffer; LayerNorm(no affine) + GELU re-emits that layout.
"""
import torch

from .. import kernels as K
from .. import relpos
from ..components import Embedding, LayerNorm, Linear, PackCache, bf16, f32, trunc_normal_
from .text import make_token_bucket_position


class TransposeLast(torch.nn.Module):
    """Kept only so that Sequential indices (and therefore parameter names) match the reference (audio.py:236-242)."""

    def forward(self, x):
        return x.transpose(-2, -1)


class SamePad(torch.nn.Module):
    def __init__(self, kernel_size):
        super().__init__()
        self.remove = 1 if kernel_size % 2 == 0 else 0


class ConvFeatureExtractionModel(torch.nn.Module):
    """Parameter container with the reference's names (audio.py:254-311): conv_layers.N = Sequential(conv,
    dropout, Sequential(TransposeLast, LayerNorm, TransposeLast), GELU)."""

    def __init__(self, conv_layers, conv_bias=False):
        super().__init__()
        in_d = 1
        self.conv_layers = torch.nn.ModuleList()
        for dim, k, stride in conv_layers:
            conv = torch.nn.Conv1d(in_d, dim, k, stride=stride, bias=conv_bias)
            torch.nn.init.kaiming_normal_(conv.weight)
            self.conv_layers.append(torch.nn.Sequential(
                conv, torch.nn.Dropout(p=0.0), torch.nn.Sequential(TransposeLast(), LayerNorm(dim), TransposeLast()),
                torch.nn.GELU()))
            in_d = dim


class AudioAdapter(torch.nn.Module):
    def __init__(self, cfg, embed_dim, attention_heads, num_layers=None):
        super().__init__()
        if cfg.layernorm_embedding or cfg.add_type_embedding or cfg.shrink_alpha != 1.0 or cfg.conv_pos_pre_ln:
            raise NotImplementedError("layernorm_embedding / add_type_embedding / shrink_alpha / conv_pos_pre_ln are off "
                                      "in the 4B config")
        if cfg.abs_pos_type not in ("conv", "fixed") or cfg.conv_bias:
            raise NotImplementedError("abs_pos_type must be 'conv' (encoder) or 'fixed' (decoder); conv_bias=False")
        self.embed_dim = embed_dim
        self.attention_heads = attention_heads
        self.abs_pos_type = cfg.abs_pos_type
        self._cache = PackCache()
        if cfg.feature_encoder_spec is None or cfg.abs_pos_type == "fixed":
            # decoder variant (pretrain_al_3B.yaml decoder.audio_adapter: no feature extractor, Embedding(1026, d) positions,
            # audio.py:44,87-88): only ever called with preserve_embed (the mask-token canvas)
            if cfg.feature_encoder_spec is not None or cfg.abs_pos_type != "fixed":
                raise NotImplementedError("decoder audio adapter = feature_encoder_spec None + abs_pos_type 'fixed'")
            self.spec = None
            self.embed_positions = Embedding(1024 + 2, embed_dim)
            self.cls_embedding = torch.nn.Parameter(torch.zeros(1, 1, embed_dim))
            self._init_bias_and_mask(cfg, attention_heads, num_layers)
            trunc_normal_(self.embed_positions.weight)
            return
        self.spec = eval(cfg.feature_encoder_spec)
        if self.spec[0][1:] != (10, 5) or any(s != 2 or c != self.spec[0][0] for c, _, s in self.spec[1:]):
            raise NotImplementedError("feature extractor kernels are built for [(C,10,5)] + [(C,k,2)]*n")
        feat = self.spec[-1][0]
        self.embed_audios = torch.nn.Sequential(ConvFeatureExtractionModel(self.spec), TransposeLast(),
                                                LayerNorm(feat), Linear(feat, embed_dim))
        self.pos_depth = cfg.conv_pos_depth
        self.pos_k = max(3, cfg.conv_pos_width // cfg.conv_pos_depth)
        self.pos_groups = cfg.conv_pos_groups
        if self.pos_k % 2 == 0:
            raise NotImplementedError("even conv-pos kernel (SamePad trimming) is not used by the 4B config (k = 19)")
        self.embed_positions = torch.nn.Sequential(
            TransposeLast(),
            *[torch.nn.Sequential(
                torch.nn.Conv1d(embed_dim, embed_dim, kernel_size=self.pos_k, padding=self.pos_k // 2, groups=self.pos_groups),
                SamePad(self.pos_k), TransposeLast(), torch.nn.LayerNorm(embed_dim, elementwise_affine=False),
                TransposeLast(), torch.nn.GELU()) for _ in range(self.pos_depth)],
            TransposeLast())
        self.cls_pos_embed = torch.nn.Parameter(torch.zeros(1, 1, embed_dim))
        trunc_normal_(self.cls_pos_embed)
        self.cls_embedding = torch.nn.Parameter(torch.zeros(1, 1, embed_dim))
        self._init_bias_and_mask(cfg, attention_heads, num_layers)

    def _init_bias_and_mask(self, cfg, attention_heads, num_layers):
        if cfg.use_attn_bias:
            num_rel_dis = 2 * cfg.bucket_size - 1
            rp_bucket = make_token_bucket_position(cfg.bucket_size, max_position=1024)
            rp_bucket[0, :] = num_rel_dis
            rp_bucket[:, 0] = num_rel_dis + 1
            rp_bucket[0, 0] = num_rel_dis + 2
            self.register_buffer("rp_bucket", rp_bucket)
            self.rel_pos_table_list = torch.nn.ModuleList(
                [Embedding(num_rel_dis + 3, attention_heads, zero_init=True) for _ in range(num_layers or 1)])
        else:
            self.rel_pos_table_list = None
        self.mask_embedding = torch.nn.Parameter(torch.zeros(1, self.embed_dim))
        trunc_normal_(self.cls_embedding)
        trunc_normal_(self.mask_embedding)

    # ------------------------------------------------------------------------------------------------
    def _pack(self):
        fe = self.embed_audios[0].conv_layers
        ps = [l[0].weight for l in fe] + [l[2][1].weight for l in fe] + [l[2][1].bias for l in fe] + \
             [self.embed_audios[2].weight, self.embed_audios[2].bias, self.embed_audios[3].weight, self.embed_audios[3].bias,
              self.cls_embedding, self.cls_pos_embed] + \
             [self.embed_positions[i + 1][0].weight for i in range(self.pos_depth)] + \
             [self.embed_positions[i + 1][0].bias for i in range(self.pos_depth)] + \
             ([t.weight for t in self.rel_pos_table_list] if self.rel_pos_table_list is not None else [])

        def build():
            d, G = self.embed_dim, self.pos_groups
            cg = d // G
            cpad = (cg + 63) // 64 * 64
            conv_w = []
            for i, l in enumerate(fe):
                w = l[0].weight.detach()                               # [C_out, C_in, k]
                if i == 0:
                    w16 = torch.zeros(w.shape[0], 16, dtype=torch.bfloat16, device=w.device)
                    w16[:, : w.shape[2]] = w[:, 0, :].to(torch.bfloat16)
                    conv_w.append(w16.contiguous())
                else:
                    conv_w.append(bf16(w.permute(0, 2, 1).reshape(w.shape[0], -1)))     # [out, (tap, c)]
            pos_w = []
            for i in range(self.pos_depth):
                w = self.embed_positions[i + 1][0].weight.detach()      # [d, cg, k]
                wp = torch.zeros(d, self.pos_k, cpad, dtype=torch.bfloat16, device=w.device)
                wp[:, :, :cg] = w.permute(0, 2, 1).to(torch.bfloat16)
                pos_w.append(wp.reshape(d, self.pos_k * cpad).contiguous())
            return dict(
                conv_w=conv_w, ln_w=[f32(l[2][1].weight) for l in fe], ln_b=[f32(l[2][1].bias) for l in fe],
                post_ln_w=f32(self.embed_audios[2].weight), post_ln_b=f32(self.embed_audios[2].bias),
                proj_w=bf16(self.embed_audios[3].weight), proj_b=f32(self.embed_audios[3].bias),
                pos_w=pos_w, pos_b=[f32(self.embed_positions[i + 1][0].bias) for i in range(self.pos_depth)],
                cls=f32(self.cls_embedding).view(-1), cls_pos=f32(self.cls_pos_embed).view(-1), cpad=cpad,
                tables=[f32(t.weight) for t in self.rel_pos_table_list] if self.rel_pos_table_list is not None else None)
        return self._cache.get(ps, build)

    def frame_counts(self, n_samples):
        out, L = [], n_samples
        for _, k, s in self.spec:
            L = (L - k) // s + 1
            out.append(L)
        return out

    def get_rel_pos_bias(self, seq_len):
        """One RelPosBias per table: LUT form for the attention kernel when S <= 384 (kernels.ATTN_TC_MAX_S), dense (H,S,S_pad) otherwise."""
        p = self._pack()
        if not hasattr(self, "_lut_cache"):
            self._lut_cache = relpos.LutCache()
        lut = self._lut_cache.get(seq_len, self.rp_bucket.device, self.rp_bucket, lambda S: relpos.text_codes(S)) if seq_len <= K.ATTN_TC_MAX_S else None
        out = []
        for t in p["tables"]:
            if lut is not None:
                out.append(K.RelPosBias(lut=K.relpos_lut_build(t, lut[0]), code_row=lut[1], code_col=lut[2]))
            else:
                out.append(K.RelPosBias(dense=K.relpos_bias_build(t, self.rp_bucket, seq_len, self.attention_heads)))
        return out

    def bias_source(self, n, ids=None):
        if self.rel_pos_table_list is None:
            return None
        return dict(tables=[t.weight for t in self.rel_pos_table_list], bucket=self.rp_bucket, n=n, ids=ids)

    def embed_general(self, src_audios, padding_mask, preserve_ids=None, preserve_embed=None, mask_token=None):
        """General (pretraining) form of forward (models/adapter/audio.py:136-207) -> (x fp32, pad uint8, bias source).
        preserve_ids (B,K) int64, -1 padded: encoder student pass — frame features gathered by id BEFORE the positional
        convolution (:184-189; padded slots read position K-1 as the reference does).  With preserve_embed (B,K,d): decoder
        canvas = mask token everywhere, preserved rows scattered to their positions, plus Embedding positions (:172-181)."""
        B, S = padding_mask.shape
        if preserve_embed is not None:
            from ..autograd_general import RowGatherFn
            from .text import canvas_index
            if self.abs_pos_type != "fixed":
                raise RuntimeError("the mask-token canvas needs abs_pos_type='fixed' (audio.py:173: embed_positions(position_ids))")
            d = self.embed_dim
            x = RowGatherFn.apply(preserve_embed.reshape(-1, d), canvas_index(preserve_ids, S), mask_token,
                                  self.embed_positions.weight[:S]).view(B, S, d)
            return x, padding_mask.to(torch.uint8).contiguous(), self.bias_source(S)
        if self.spec is None:
            raise RuntimeError("decoder audio adapter (no feature extractor) needs preserve_embed")
        if preserve_ids is not None:
            return self.forward_train(src_audios, padding_mask, preserve_ids)
        x, pad, _ = self.forward(src_audios, padding_mask)
        return x, pad, self.bias_source(x.shape[1])

    def forward(self, src_audios, padding_mask, preserve_ids=None, preserve_embed=None, mask_token=None):
        """src_audios (B, N) waveform, padding_mask (B, T+1) bool -> (x fp32 (B,T+1,d) with padded rows zeroed,
        padding_mask uint8, [bias (H,S,S_pad)])"""
        if preserve_ids is not None or preserve_embed is not None or self.spec is None:
            return self.embed_general(src_audios, padding_mask, preserve_ids, preserve_embed, mask_token)
        if torch.is_grad_enabled() and any(q.requires_grad for q in self.parameters()):
            return self.forward_train(src_audios, padding_mask)
        p = self._pack()
        B, N = src_audios.shape
        dev = src_audios.device
        d, C = self.embed_dim, self.spec[0][0]
        frames = self.frame_counts(N)
        T = frames[-1]
        S = T + 1
        if padding_mask.shape != (B, S):
            raise RuntimeError(f"audio_padding_masks must be (B, frames + 1) = ({B}, {S}), got {tuple(padding_mask.shape)}")
        nl = len(self.spec)
        # per-clip row pitch of every layer's frame buffer: pitch_k = 2^(nl-1-k) * P covers frames[k]
        P = max((frames[k] + (1 << (nl - 1 - k)) - 1) >> (nl - 1 - k) for k in range(nl))
        pitch = [P << (nl - 1 - k) for k in range(nl)]
        wav = src_audios if src_audios.dtype in (torch.float32, torch.bfloat16) else src_audios.float()
        a0 = torch.empty(B * pitch[0], 16, dtype=torch.bfloat16, device=dev)
        K.audio_frame10(wav.contiguous(), pitch[0], a0)
        slack = 4                                                   # rows read past the last clip by the widest window
        y = torch.zeros(B * pitch[0] + slack, C, dtype=torch.bfloat16, device=dev)
        K.gemm(a0, p["conv_w"][0], K.EPI_STORE_BF16, y, M=B * pitch[0])
        K.layernorm(y, p["ln_w"][0], p["ln_b"][0], y, rows=B * pitch[0], gelu=True)
        for k in range(1, nl):
            kw = self.spec[k][1]
            yn = torch.zeros(B * pitch[k] + slack, C, dtype=torch.bfloat16, device=dev)
            K.gemm(y, p["conv_w"][k], K.EPI_STORE_BF16, yn, M=B * pitch[k], K=kw * C, lda=2 * C)
            K.layernorm(yn, p["ln_w"][k], p["ln_b"][k], yn, rows=B * pitch[k], gelu=True)
            y = yn
        K.layernorm(y, p["post_ln_w"], p["post_ln_b"], y, rows=B * P)
        # features -> residual stream rows 1..T of every clip (fp32), slack rows (t >= T) dropped
        x = torch.empty(B, S, d, dtype=torch.float32, device=dev)
        K.gemm(y, p["proj_w"], K.EPI_STORE_F32, x.view(B * S, d), bias=p["proj_b"], M=B * P, out_group=P,
               out_group_stride=S, out_row_offset=1, out_group_valid=T)
        # conv positional encoder on the (un-normalised) features
        G, cg, cpad, kp = self.pos_groups, d // self.pos_groups, p["cpad"], self.pos_k
        halo = kp // 2
        Tp = T + 2 * halo
        bufs = [torch.zeros(B * Tp + kp, G, cpad, dtype=torch.bfloat16, device=dev) for _ in range(2)]
        K.pack_group_halo(x.view(B * S, d), bufs[0], B, T, S, 1, Tp, halo, d, cg, cpad)
        conv_out = torch.empty(B * Tp, d, dtype=torch.bfloat16, device=dev)
        for i in range(self.pos_depth):
            src, dst = bufs[i % 2], bufs[(i + 1) % 2]
            K.grouped_conv1d(src, p["pos_w"][i], p["pos_b"][i], conv_out, B * Tp, G, cpad, kp, cg)
            if i + 1 < self.pos_depth:
                # LN(no affine) + GELU -> next layer's halo'd / group-padded operand (valid rows only)
                K.layernorm(conv_out, None, None, dst.view(-1, G * cpad), rows=B * Tp, dim=d, gelu=True, row_period=Tp,
                            row_valid=T, out_period=Tp, out_row_shift=halo, group_in=cg, group_out=cpad)
            else:
                # last layer: x[b, 1 + t, :] += gelu(LN(conv))     (audio.py:194-199: x = feats + pos)
                K.layernorm(conv_out, None, None, x.view(B * S, d), rows=B * Tp, dim=d, gelu=True, row_period=Tp,
                            row_valid=T, out_period=S, out_row_shift=1, accumulate=True)
        K.cls_row_init(p["cls"], p["cls_pos"], x)
        pad = padding_mask.to(torch.uint8).contiguous()
        K.zero_padded_rows(x, pad)                                  # transformer_encoder.py:139-142
        bias = self.get_rel_pos_bias(S) if self.rel_pos_table_list is not None else None
        return x, pad, bias

    def _feat_params(self):
        fe = self.embed_audios[0].conv_layers
        return [l[0].weight for l in fe] + [l[2][1].weight for l in fe] + [l[2][1].bias for l in fe] + \
               [self.embed_audios[2].weight, self.embed_audios[2].bias, self.embed_audios[3].weight, self.embed_audios[3].bias]

    def _pos_params(self):
        return [self.embed_positions[i + 1][0].weight for i in range(self.pos_depth)] + \
               [self.embed_positions[i + 1][0].bias for i in range(self.pos_depth)] + [self.cls_embedding, self.cls_pos_embed]

    def forward_train(self, src_audios, padding_mask, preserve_ids=None):
        """Same outputs, recorded for autograd (autograd.AudioFeatFn -> [preserve_ids gather] -> AudioPosFn: materialised-window
        GEMMs + col2im adjoints).  With preserve_ids (B,K) the frame features are gathered BEFORE the positional convolution
        (models/adapter/audio.py:184-189) and the relative-position bias source carries the ids."""
        from ..autograd import AudioFeatFn, AudioPosFn, RelPosBiasFn, TrainBias
        B, N = src_audios.shape
        T = self.frame_counts(N)[-1]
        S = T + 1
        if padding_mask.shape != (B, S):
            raise RuntimeError(f"audio_padding_masks must be (B, frames + 1) = ({B}, {S}), got {tuple(padding_mask.shape)}")
        d = self.embed_dim
        feats = AudioFeatFn.apply(src_audios, (tuple(self.spec), d), *self._feat_params())            # fp32 [B*T, d]
        if preserve_ids is not None:
            from ..autograd_general import RowGatherFn
            Kk = preserve_ids.shape[1]
            # position_ids[:, 1:] - 1 with padded slots mapped to position K - 1 first (audio.py:150-153,186): frame K - 2
            pid = preserve_ids.masked_fill(preserve_ids.eq(-1), Kk - 1)[:, 1:] - 1
            flat = (pid + torch.arange(B, device=pid.device)[:, None] * T).reshape(-1).contiguous()
            feats = RowGatherFn.apply(feats, flat, None, None)
            x, pad = AudioPosFn.apply(feats, preserve_ids.eq(-1), (B, Kk - 1, self.pos_k, self.pos_groups, d), *self._pos_params())
            return x, pad, self.bias_source(Kk, preserve_ids.contiguous())
        x, pad = AudioPosFn.apply(feats, padding_mask, (B, T, self.pos_k, self.pos_groups, d), *self._pos_params())
        bias = None
        if self.rel_pos_table_list is not None:
            fast = self.get_rel_pos_bias(S)
            bias = [TrainBias(RelPosBiasFn.apply(t.weight, self.rp_bucket, S, self.attention_heads),
                              f if f.lut is not None else None) for t, f in zip(self.rel_pos_table_list, fast)]
        return x, pad, bias
