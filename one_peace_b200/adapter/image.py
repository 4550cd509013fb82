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
from ..autograd import ImageEmbedFn, RelPosBiasFn, TrainBias, image_stem, pack_image_stem
from ..components import Embedding, LayerNorm, PackCache, f32, trunc_normal_


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


def geometric_sequence_interpolation(src_size, dst_size, sequence, num):
    """models/adapter/image.py:115-162: resample a (src_size x src_size) relative-position table [src_size^2, num] onto
    (dst_size x dst_size).  The source offsets are placed on a geometric sequence whose ratio q (bisection over [1.01, 1.5]
    down to 1e-6) stretches src_size // 2 steps to dst_size // 2, and every head is fitted by a bicubic interpolating spline
    evaluated on the integer offsets -t .. t.  The reference calls scipy.interpolate.interp2d(kind='cubic'), which SciPy 1.14
    removed; on gridded data it computed the s = 0 bicubic spline of RectBivariateSpline(y, x, z), which is what runs here
    (z is [len(y), len(x)])."""
    import numpy as np
    from scipy.interpolate import RectBivariateSpline

    half_src, half_dst = src_size // 2, dst_size // 2
    lo, hi = 1.01, 1.5
    while hi - lo > 1e-6:                      # sum_{k<half_src} q^k against half_dst
        q = (lo + hi) / 2.0
        lo, hi = (lo, q) if (1.0 - q ** half_src) / (1.0 - q) > half_dst else (q, hi)
    pos = [1]
    for k in range(1, half_src):
        pos.append(pos[-1] + q ** k)
    grid = np.array([-v for v in pos[::-1]] + [0] + pos, dtype=np.float64)
    t = dst_size // 2.0
    target = np.arange(-t, t + 0.1, 1.0)
    heads = []
    for h in range(num):
        z = sequence[:, h].view(src_size, src_size).float().numpy()
        spline = RectBivariateSpline(grid, grid, z, kx=3, ky=3, s=0)       # axis 0 = y (rows of z), axis 1 = x
        heads.append(torch.tensor(spline(target, target), dtype=torch.float32).reshape(-1, 1).to(sequence))
    return torch.cat(heads, dim=-1)


class LayerNorm2D(torch.nn.Module):
    """Parameter container named like models/adapter/image.py:37-47 (embed_images.{1,4}.layer_norm.*)."""

    def __init__(self, embed_dim):
        super().__init__()
        self.layer_norm = LayerNorm(embed_dim)


def hmlp_stem(embed_dim):
    """`embed_images` of models/adapter/image.py:66-75: conv 4x4/4, LayerNorm2D, GELU, conv 2x2/2, LayerNorm2D, GELU,
    conv 2x2/2, with embed_dim / 4 channels between the convs.  autograd.image_stem runs it."""
    c4 = embed_dim // 4
    return torch.nn.Sequential(
        torch.nn.Conv2d(3, c4, kernel_size=4, stride=4), LayerNorm2D(c4), torch.nn.GELU(),
        torch.nn.Conv2d(c4, c4, kernel_size=2, stride=2), LayerNorm2D(c4), torch.nn.GELU(),
        torch.nn.Conv2d(c4, embed_dim, kernel_size=2, stride=2))


def hmlp_stem_tensors(e):
    """The 10 parameters of an hmlp_stem `e` in the order of autograd.pack_image_stem and ImageEmbedFn.apply."""
    return [e[0].weight, e[0].bias, e[1].layer_norm.weight, e[1].layer_norm.bias, e[3].weight, e[3].bias,
            e[4].layer_norm.weight, e[4].layer_norm.bias, e[6].weight, e[6].bias]


def image_lut_bias(cache, table, bucket, side):
    """One relative-position table over a side x side image grid plus its CLS row (S = side^2 + 1 rows) as a
    kernels.RelPosBias in LUT form; `cache` is the caller's relpos.LutCache of its `bucket`."""
    lut = cache.get(side * side + 1, bucket.device, bucket, lambda n: relpos.image_codes(n, side))
    return K.RelPosBias(lut=K.relpos_lut_build(f32(table), lut[0]), code_row=lut[1], code_col=lut[2])


class ImageAdapter(torch.nn.Module):
    def __init__(self, cfg, embed_dim, attention_heads, num_layers=None):
        super().__init__()
        if cfg.vision_encoder_type not in ("hmlp", "none"):
            raise NotImplementedError("only the hMLP stem (the 4B config) and 'none' (the pretraining decoder) are built")
        if cfg.layernorm_embedding or cfg.add_type_embedding or cfg.shrink_alpha != 1.0:
            raise NotImplementedError("layernorm_embedding / add_type_embedding / shrink_alpha are off in the 4B config")
        self.attention_heads = attention_heads
        self.embed_dim = embed_dim
        self.embed_images = None if cfg.vision_encoder_type == "none" else hmlp_stem(embed_dim)
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
        stem = hmlp_stem_tensors(self.embed_images)
        ps = stem + [self.cls_embedding, self.pos_embed] + \
            ([t.weight for t in self.rel_pos_table_list] if self.rel_pos_table_list is not None else [])

        def build():
            self._pos_cache = {}
            return dict(pack_image_stem(*stem), cls=f32(self.cls_embedding).view(-1),
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
        w = src_images.shape[-1] // 16
        S = w * w + 1
        if self.rel_pos_table_list is not None and S != self.rp_bucket.shape[0]:
            raise RuntimeError("image size must match rel_bucket_size * 16 (one_peace_retrieval.py:128)")
        x, _ = image_stem(p, src_images, self.get_embed_positions(w), p["cls"])
        bias = self.get_rel_pos_bias(S) if self.rel_pos_table_list is not None else None
        return x, None, bias

    def upgrade_state_dict_named(self, state_dict, name):
        """Resize a checkpoint's image tables to this adapter (models/adapter/image.py:262-305): a relative-position table
        smaller than (2 * rel_bucket_size - 1)^2 + 3 rows (a 256^2 checkpoint loaded for 384^2 fine-tuning) is interpolated
        onto the larger grid, and pos_embed is resized bicubically when it has fewer than bucket_size^2 + 1 rows.  Runs on the
        host, once per load.  Copying table 0 to every layer is left to the model (one_peace_classify)."""
        prefix = f"{name}." if name else ""
        key = prefix + "rel_pos_table_list.0.weight"
        if prefix + "rel_pos_table.weight" in state_dict:
            state_dict[key] = state_dict.pop(prefix + "rel_pos_table.weight")
        if self.rel_pos_table_list is not None and key in state_dict and \
                (2 * self.rel_bucket_size - 1) ** 2 + 3 > state_dict[key].shape[0]:
            table = state_dict[key]
            src = int((table.shape[0] - 3) ** 0.5)
            new = geometric_sequence_interpolation(src, 2 * self.rel_bucket_size - 1, table[:-3].cpu(), table.shape[1])
            state_dict[key] = torch.cat([new.to(table), table[-3:]], dim=0)
            state_dict[prefix + "rp_bucket"] = self.rp_bucket.clone()
        pk = prefix + "pos_embed"
        if pk in state_dict and self.bucket_size ** 2 + 1 > state_dict[pk].shape[0]:
            pe = state_dict[pk]
            n = int((pe.shape[0] - 1) ** 0.5)
            old = pe[1:].reshape(1, n, n, -1).permute(0, 3, 1, 2)
            new = F.interpolate(old, size=(self.bucket_size, self.bucket_size), mode="bicubic")
            state_dict[pk] = torch.cat([pe[:1], new.permute(0, 2, 3, 1).reshape(self.bucket_size ** 2, -1)], dim=0)
            state_dict[prefix + "position_idx"] = self.position_idx.clone()

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
        x = ImageEmbedFn.apply(src_images, pe, *hmlp_stem_tensors(self.embed_images), self.cls_embedding)
        bias = None
        if self.rel_pos_table_list is not None:
            fast = self.get_rel_pos_bias(S)            # LUT form for the attention kernel (S <= 384), same values
            bias = [TrainBias(RelPosBiasFn.apply(t.weight, self.rp_bucket, S, self.attention_heads),
                              f if f.lut is not None else None) for t, f in zip(self.rel_pos_table_list, fast)]
        return x, None, bias
