"""Drop-in for ``ImageAdapter`` (models/adapter/image.py:50-312): hMLP stem (3 stride==kernel convs with
LayerNorm2D + GELU between them), CLS + absolute positions (bicubic-resized pos_embed), 2-D relative
position bias.  Same parameter / buffer names.

The three convolutions have kernel == stride, so each is an exact GEMM over non-overlapping patches
(A.5 in SURVEY.md): a patchify kernel builds the K=48 operand of the first one, and the LayerNorm+GELU
kernel after each conv scatters its output rows straight into the 2x2-merged operand of the next.
The last GEMM's epilogue adds the conv bias and the positional table and writes behind the CLS slot.
"""
import torch
import torch.nn.functional as F

from .. import kernels as K
from .. import relpos
from ..components import Embedding, LayerNorm, PackCache, bf16, f32, trunc_normal_


def make_image_bucket_position(bucket_size, num_relative_distance):
    """BEiT-style 2-D relative index with 3 CLS ids — same index math as models/adapter/image.py:19-34."""
    coords = torch.stack(torch.meshgrid([torch.arange(bucket_size), torch.arange(bucket_size)], indexing="ij"))
    flat = torch.flatten(coords, 1)
    rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += bucket_size - 1
    rel[:, :, 1] += bucket_size - 1
    rel[:, :, 0] *= 2 * bucket_size - 1
    idx = torch.zeros(size=(bucket_size * bucket_size + 1,) * 2, dtype=rel.dtype)
    idx[1:, 1:] = rel.sum(-1)
    idx[0, 0:] = num_relative_distance - 3
    idx[0:, 0] = num_relative_distance - 2
    idx[0, 0] = num_relative_distance - 1
    return idx


class LayerNorm2D(torch.nn.Module):
    """Parameter container named like models/adapter/image.py:37-47 (embed_images.{1,4}.layer_norm.*)."""

    def __init__(self, embed_dim):
        super().__init__()
        self.layer_norm = LayerNorm(embed_dim)


class ImageAdapter(torch.nn.Module):
    def __init__(self, cfg, embed_dim, attention_heads, num_layers=None):
        super().__init__()
        if cfg.vision_encoder_type not in ("hmlp", "none"):
            raise NotImplementedError("only the hMLP stem (the 4B config) and 'none' (the pretraining decoder) are built")
        if cfg.layernorm_embedding or cfg.add_type_embedding or cfg.shrink_alpha != 1.0:
            raise NotImplementedError("layernorm_embedding / add_type_embedding / shrink_alpha are off in the 4B config")
        self.attention_heads = attention_heads
        self.embed_dim = embed_dim
        c4 = embed_dim // 4
        self.embed_images = None if cfg.vision_encoder_type == "none" else torch.nn.Sequential(
            torch.nn.Conv2d(3, c4, kernel_size=4, stride=4), LayerNorm2D(c4), torch.nn.GELU(),
            torch.nn.Conv2d(c4, c4, kernel_size=2, stride=2), LayerNorm2D(c4), torch.nn.GELU(),
            torch.nn.Conv2d(c4, embed_dim, kernel_size=2, stride=2))
        self.cls_embedding = torch.nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.bucket_size = cfg.bucket_size
        self.pos_embed = torch.nn.Parameter(torch.zeros(self.bucket_size ** 2 + 1, embed_dim))
        self.register_buffer("position_idx", torch.arange(self.bucket_size ** 2 + 1))
        if cfg.use_attn_bias:
            self.rel_bucket_size = cfg.rel_bucket_size
            num_rel_dis = (2 * self.rel_bucket_size - 1) ** 2 + 3
            self.register_buffer("rp_bucket", make_image_bucket_position(self.rel_bucket_size, num_rel_dis))
            self.rel_pos_table_list = torch.nn.ModuleList(
                [Embedding(num_rel_dis, attention_heads, zero_init=True) for _ in range(num_layers or 1)])
        else:
            self.rel_pos_table_list = None
        trunc_normal_(self.cls_embedding)
        trunc_normal_(self.pos_embed)
        self._cache = PackCache()
        self._pos_cache = {}

    def _pack(self):
        e = self.embed_images
        ps = [e[0].weight, e[0].bias, e[1].layer_norm.weight, e[1].layer_norm.bias, e[3].weight, e[3].bias,
              e[4].layer_norm.weight, e[4].layer_norm.bias, e[6].weight, e[6].bias, self.cls_embedding, self.pos_embed] + \
             ([t.weight for t in self.rel_pos_table_list] if self.rel_pos_table_list is not None else [])

        def build():
            self._pos_cache = {}
            c4 = e[0].weight.shape[0]
            return dict(
                w1=bf16(e[0].weight.reshape(c4, 48)), b1=f32(e[0].bias),
                ln1_w=f32(e[1].layer_norm.weight), ln1_b=f32(e[1].layer_norm.bias),
                # conv weight [out, c, ky, kx] -> [out, (ky, kx, c)] to match the pixel-merge scatter order
                w2=bf16(e[3].weight.permute(0, 2, 3, 1).reshape(c4, 4 * c4)), b2=f32(e[3].bias),
                ln2_w=f32(e[4].layer_norm.weight), ln2_b=f32(e[4].layer_norm.bias),
                w3=bf16(e[6].weight.permute(0, 2, 3, 1).reshape(self.embed_dim, 4 * c4)), b3=f32(e[6].bias),
                cls=f32(self.cls_embedding).view(-1),
                tables=[f32(t.weight) for t in self.rel_pos_table_list] if self.rel_pos_table_list is not None else None)
        return self._cache.get(ps, build)

    def get_embed_positions(self, window_size):
        """fp32 [w*w+1, d]; bicubic resize of the (bucket_size^2) grid part when the window differs
        (models/adapter/image.py:173-186 — parameter preprocessing, cached until pos_embed changes)."""
        if window_size not in self._pos_cache:
            pe = self.pos_embed.detach()
            if window_size != self.bucket_size:
                old = pe[1:].reshape(1, self.bucket_size, self.bucket_size, -1).permute(0, 3, 1, 2).float()
                new = F.interpolate(old, size=(window_size, window_size), mode="bicubic").type_as(pe)
                new = new.permute(0, 2, 3, 1).reshape(window_size ** 2, -1)
                pe = torch.cat([pe[:1], new], dim=0)
            self._pos_cache[window_size] = f32(pe)
        return self._pos_cache[window_size]

    def get_rel_pos_bias(self, seq_len):
        """One RelPosBias per table: LUT form for the attention kernel when S <= 384 (kernels.ATTN_TC_MAX_S), dense (H,S,S_pad) otherwise."""
        p = self._pack()
        if not hasattr(self, "_lut_cache"):
            self._lut_cache = relpos.LutCache()
        w = self.rel_bucket_size
        lut = self._lut_cache.get(seq_len, self.rp_bucket.device, self.rp_bucket, lambda S: relpos.image_codes(S, w)) \
            if seq_len <= K.ATTN_TC_MAX_S else None
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

    def _pos_table(self, w):
        """(w*w+1, d) positional table as an autograd function of pos_embed (bicubic resize as a cached linear operator)."""
        pe = self.pos_embed
        if w != self.bucket_size:
            new = (self._resize_matrix(w, pe.device) @ pe[1:].float()).type_as(pe)
            pe = torch.cat([pe[:1], new], dim=0)
        return pe

    def embed_general(self, src_images, preserve_ids=None, preserve_embed=None, mask_token=None):
        """General (pretraining) form of forward (models/adapter/image.py:206-260); see TextAdapter.embed_general."""
        from ..autograd_general import RowGatherFn
        from .text import canvas_index, flat_ids
        B, R = src_images.shape[0], src_images.shape[-1]
        w = R // 16
        S = w * w + 1
        d = self.embed_dim
        if preserve_embed is not None:
            x = RowGatherFn.apply(preserve_embed.reshape(-1, d), canvas_index(preserve_ids, S), mask_token,
                                  self._pos_table(w)).view(B, S, d)
            return x, None, self.bias_source(S)
        x, _, _ = self.forward(src_images)                   # full sequence (autograd-tracked when training)
        if preserve_ids is None:
            return x, None, self.bias_source(S)
        Kk = preserve_ids.shape[1]
        xg = RowGatherFn.apply(x.reshape(B * S, d), flat_ids(preserve_ids, S), None, None).view(B, Kk, d)
        return xg, preserve_ids.eq(-1).to(torch.uint8).contiguous(), self.bias_source(Kk, preserve_ids.contiguous())

    def forward(self, src_images, preserve_ids=None, preserve_embed=None, mask_token=None, is_second_image=False):
        """-> (x fp32 (B, w*w+1, d), None (images are never padded), [bias (H,S,S_pad)])"""
        if preserve_ids is not None or preserve_embed is not None:
            return self.embed_general(src_images, preserve_ids, preserve_embed, mask_token)
        if torch.is_grad_enabled() and any(q.requires_grad for q in self.parameters()):
            return self.forward_train(src_images)
        p = self._pack()
        B, _, R, _ = src_images.shape
        d, c4 = self.embed_dim, self.embed_dim // 4
        g1, g2, w = R // 4, R // 8, R // 16
        S = w * w + 1
        if self.rel_pos_table_list is not None and S != self.rp_bucket.shape[0]:
            raise RuntimeError("image size must match rel_bucket_size * 16 (one_peace_retrieval.py:128)")
        dev = src_images.device
        img = src_images if src_images.dtype in (torch.float32, torch.bfloat16) else src_images.float()
        a1 = K.image_patchify4(img.contiguous())
        y1 = torch.empty(B * g1 * g1, c4, dtype=torch.bfloat16, device=dev)
        K.gemm(a1, p["w1"], K.EPI_STORE_BF16, y1, bias=p["b1"])
        a2 = torch.empty(B * g2 * g2, 4 * c4, dtype=torch.bfloat16, device=dev)
        K.layernorm(y1, p["ln1_w"], p["ln1_b"], a2, gelu=True, merge_grid_w=g1)
        y2 = torch.empty(B * g2 * g2, c4, dtype=torch.bfloat16, device=dev)
        K.gemm(a2, p["w2"], K.EPI_STORE_BF16, y2, bias=p["b2"])
        a3 = torch.empty(B * w * w, 4 * c4, dtype=torch.bfloat16, device=dev)
        K.layernorm(y2, p["ln2_w"], p["ln2_b"], a3, gelu=True, merge_grid_w=g2)
        pos = self.get_embed_positions(w)
        x = torch.empty(B, S, d, dtype=torch.float32, device=dev)
        K.gemm(a3, p["w3"], K.EPI_RESID_F32, x.view(B * S, d), bias=p["b3"], resid=pos, out_group=w * w,
               out_group_stride=S, out_row_offset=1, resid_period=w * w, resid_row_offset=1)
        K.cls_row_init(p["cls"], pos, x)
        bias = self.get_rel_pos_bias(S) if self.rel_pos_table_list is not None else None
        return x, None, bias

    def _resize_matrix(self, w, device):
        key = (w, str(device))
        cache = self.__dict__.setdefault("_resize_cache", {})
        if key not in cache:
            n = self.bucket_size
            eye = torch.eye(n * n, dtype=torch.float32, device=device).reshape(n * n, 1, n, n)      # basis images
            cache[key] = F.interpolate(eye, size=(w, w), mode="bicubic").reshape(n * n, w * w).t().contiguous()
        return cache[key]

    def forward_train(self, src_images):
        """Same outputs, recorded for autograd (autograd.ImageEmbedFn / RelPosBiasFn); the positional table is resized
        by torch ops so its gradient reaches pos_embed through torch's own bicubic adjoint (parameter preprocessing)."""
        from ..autograd import ImageEmbedFn, RelPosBiasFn, TrainBias
        R = src_images.shape[-1]
        w = R // 16
        S = w * w + 1
        if self.rel_pos_table_list is not None and S != self.rp_bucket.shape[0]:
            raise RuntimeError("image size must match rel_bucket_size * 16 (one_peace_retrieval.py:128)")
        pe = self.pos_embed
        if w != self.bucket_size:
            # the bicubic resize (image.py:173-186) is linear in pos_embed: apply it as a cached [w*w, bucket^2] fp32
            # matrix (torch's bicubic kernels run single-CTA here: 2.9 ms forward + 0.9 ms backward per step)
            new = (self._resize_matrix(w, pe.device) @ pe[1:].float()).type_as(pe)
            pe = torch.cat([pe[:1], new], dim=0)
        e = self.embed_images
        x = ImageEmbedFn.apply(src_images, pe, e[0].weight, e[0].bias, e[1].layer_norm.weight, e[1].layer_norm.bias,
                               e[3].weight, e[3].bias, e[4].layer_norm.weight, e[4].layer_norm.bias, e[6].weight, e[6].bias,
                               self.cls_embedding)
        bias = None
        if self.rel_pos_table_list is not None:
            fast = self.get_rel_pos_bias(S)            # LUT form for the attention kernel (S <= 384), same values
            bias = [TrainBias(RelPosBiasFn.apply(t.weight, self.rp_bucket, S, self.attention_heads),
                              f if f.lut is not None else None) for t, f in zip(self.rel_pos_table_list, fast)]
        return x, None, bias
