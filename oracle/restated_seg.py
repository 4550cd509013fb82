"""TEST INFRASTRUCTURE.  A torch restatement of the segmentation backbone's forward
(one_peace_vision/seg/mmseg_custom/models/backbones/onepeace_adapter.py with its adapter_modules.py and onepeace.py: eval
BatchNorm, rp_bias=True, with_cffn, add_vit_feature), written for this project from the reference's documented
computation and pinned to the reference by tests/golden/seg.pt.  It takes a state dict of the reference's names and runs on
any device in the dtype of that state dict, so the GPU tests use it in fp32 as the yardstick of the 40-layer backbone and
scripts/bench_seg.py runs it in bf16 as the eager baseline.  The deformable attention is the grid_sample form of the
reference's ms_deform_attn_core_pytorch.
"""
import torch
import torch.nn.functional as F

from restated_video import _attn, _lin, _ln

LN_EPS = 1e-6


def _bn(x, sd, p, eps=1e-5):
    """Eval BatchNorm on NCHW x."""
    v = lambda n: sd[f"{p}.{n}"].to(x.dtype).view(1, -1, 1, 1)
    return (x - v("running_mean")) * torch.rsqrt(v("running_var") + eps) * v("weight") + v("bias")


def level_shapes(side):
    return [(2 * side, 2 * side), (side, side), (side // 2, side // 2)]


def reference_points(shapes, device, dtype):
    out = []
    for h, w in shapes:
        y, x = torch.meshgrid(torch.linspace(0.5, h - 0.5, h, dtype=torch.float64, device=device),
                              torch.linspace(0.5, w - 0.5, w, dtype=torch.float64, device=device), indexing="ij")
        out.append(torch.stack((x.reshape(-1) / w, y.reshape(-1) / h), -1))
    return torch.cat(out, 0).to(dtype)[None, :, None]                     # [1, Lq, 1, 2]


def msda(sd, p, query, ref, feat, shapes, heads, points):
    """MSDeformAttn (ops/modules/ms_deform_attn.py) with ms_deform_attn_core_pytorch: query [N, Lq, d], ref [1, Lq, 1, 2],
    feat [N, S_in, d] -> [N, Lq, d]."""
    N, Lq, _ = query.shape
    L = len(shapes)
    value = _lin(feat, sd, p + ".value_proj")
    Dh = value.shape[-1] // heads
    value = value.view(N, -1, heads, Dh)
    off = _lin(query, sd, p + ".sampling_offsets").view(N, Lq, heads, L, points, 2)
    aw = _lin(query, sd, p + ".attention_weights").view(N, Lq, heads, L * points).softmax(-1).view(N, Lq, heads, L, points)
    norm = torch.tensor([[w, h] for h, w in shapes], dtype=query.dtype, device=query.device)
    grid = 2 * (ref[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]) - 1
    out, start = 0, 0
    for l, (h, w) in enumerate(shapes):
        v = value[:, start:start + h * w].permute(0, 2, 3, 1).reshape(N * heads, Dh, h, w)
        g = grid[:, :, :, l].permute(0, 2, 1, 3, 4).reshape(N * heads, Lq, points, 2)
        smp = F.grid_sample(v, g, mode="bilinear", padding_mode="zeros", align_corners=False)
        out = out + (smp * aw[:, :, :, l].permute(0, 2, 1, 3).reshape(N * heads, 1, Lq, points)).sum(-1)
        start += h * w
    out = out.view(N, heads, Dh, Lq).permute(0, 3, 1, 2).reshape(N, Lq, heads * Dh)
    return _lin(out, sd, p + ".output_proj")


def spm(sd, img):
    """SpatialPriorModule -> c1 map [B, d, 4s, 4s] and the c2, c3, c4 rows [B, h w, d] before level_embed."""
    x = img
    for conv, bn, stride in ((0, 1, 2), (3, 4, 1), (6, 7, 1)):
        x = F.relu(_bn(F.conv2d(x, sd[f"spm.stem.{conv}.weight"], stride=stride, padding=1), sd, f"spm.stem.{bn}"))
    feats = [F.max_pool2d(x, kernel_size=3, stride=2, padding=1)]
    for i in (2, 3, 4):
        feats.append(F.relu(_bn(F.conv2d(feats[-1], sd[f"spm.conv{i}.0.weight"], stride=2, padding=1), sd, f"spm.conv{i}.1")))
    outs = [F.conv2d(f, sd[f"spm.fc{i + 1}.weight"], sd[f"spm.fc{i + 1}.bias"]) for i, f in enumerate(feats)]
    return outs[0], [o.flatten(2).transpose(1, 2) for o in outs[1:]]


def stem(sd, img):
    """hMLP stem + CLS + pos_embed -> [B, s^2 + 1, d]."""
    p = "image_adapter.embed_images"
    y = img
    for i, (conv, ln) in enumerate(((0, 1), (3, 4))):
        y = F.conv2d(y, sd[f"{p}.{conv}.weight"], sd[f"{p}.{conv}.bias"], stride=4 if i == 0 else 2)
        y = F.gelu(_ln(y.permute(0, 2, 3, 1), sd, f"{p}.{ln}.layer_norm").permute(0, 3, 1, 2))
    y = F.conv2d(y, sd[f"{p}.6.weight"], sd[f"{p}.6.bias"], stride=2).flatten(2).transpose(1, 2)
    return torch.cat([sd["image_adapter.cls_embedding"].expand(y.shape[0], -1, -1), y], 1) + sd["image_adapter.pos_embed"]


def layer(sd, p, x, heads):
    """onepeace.py TransformerEncoderLayer (rp_bias=True) on x [B, S, d]."""
    bias = F.embedding(sd[p + ".rp_bucket"], sd[p + ".rel_pos_table.weight"]).permute(2, 0, 1)
    x = x + sd[p + ".gamma_1"] * _attn(_ln(x, sd, p + ".self_attn_layer_norm"), sd, p + ".self_attn", heads, bias)
    xn = _ln(x, sd, p + ".final_layer_norm")
    f = p + ".image_ffn"
    h = F.gelu(F.linear(xn, sd[f + ".0.wi_0.weight"])) * F.linear(xn, sd[f + ".0.wi_1.weight"])
    return x + sd[p + ".gamma_2"] * _lin(_ln(h, sd, f + ".2"), sd, f + ".3")


def conv_ffn(sd, p, x, shapes):
    h = _lin(x, sd, p + ".fc1")
    B, _, C = h.shape
    parts, start = [], 0
    for hh, ww in shapes:
        g = h[:, start:start + hh * ww].transpose(1, 2).reshape(B, C, hh, ww)
        g = F.conv2d(g, sd[p + ".dwconv.dwconv.weight"], sd[p + ".dwconv.dwconv.bias"], padding=1, groups=C)
        parts.append(g.flatten(2).transpose(1, 2))
        start += hh * ww
    return _lin(F.gelu(torch.cat(parts, 1)), sd, p + ".fc2")


def extractor(sd, p, c, x, ref_c, side, shapes, heads, points):
    c = c + msda(sd, p + ".attn", _ln(c, sd, p + ".query_norm", LN_EPS), ref_c, _ln(x, sd, p + ".feat_norm", LN_EPS),
                 [(side, side)], heads, points)
    return c + conv_ffn(sd, p + ".ffn", _ln(c, sd, p + ".ffn_norm", LN_EPS), shapes)


def forward(sd, img, heads, deform_heads, n_points, interaction_indexes):
    """img [B, 3, 16 s, 16 s] -> [f1, f2, f3, f4] NCHW, in the dtype of sd."""
    B = img.shape[0]
    side = img.shape[-1] // 16
    shapes = level_shapes(side)
    dev, dt = img.device, img.dtype
    ref_x = reference_points([(side, side)], dev, dt)
    ref_c = reference_points(shapes, dev, dt)
    c1, cs = spm(sd, img)
    c = torch.cat([cl + sd["level_embed"][i] for i, cl in enumerate(cs)], 1)
    x = stem(sd, img)
    d = x.shape[-1]
    cls, x = x[:, :1], x[:, 1:]
    outs = []
    for i, (lo, hi) in enumerate(interaction_indexes):
        p = f"interactions.{i}"
        x = x + sd[p + ".injector.gamma"] * msda(sd, p + ".injector.attn", _ln(x, sd, p + ".injector.query_norm", LN_EPS),
                                                 ref_x, _ln(c, sd, p + ".injector.feat_norm", LN_EPS), shapes, deform_heads,
                                                 n_points)
        x = torch.cat((cls, x), 1)
        for j in range(lo, hi + 1):
            x = layer(sd, f"encoder.layers.{j}", x, heads)
        cls, x = x[:, :1], x[:, 1:]
        exts = [p + ".extractor"] + ([f"{p}.extra_extractors.{k}" for k in range(2)]
                                     if i == len(interaction_indexes) - 1 else [])
        for e in exts:
            c = extractor(sd, e, c, x, ref_c, side, shapes, deform_heads, n_points)
        outs.append(x.transpose(1, 2).reshape(B, d, side, side))
    maps, start = [], 0
    for h, w in shapes:
        maps.append(c[:, start:start + h * w].transpose(1, 2).reshape(B, d, h, w))
        start += h * w
    c1 = F.conv_transpose2d(maps[0], sd["up.weight"], sd["up.bias"], stride=2) + c1
    x1 = F.interpolate(outs[0], scale_factor=4, mode="bilinear", align_corners=False)
    x2 = F.interpolate(outs[1], scale_factor=2, mode="bilinear", align_corners=False)
    x4 = F.interpolate(outs[3], scale_factor=0.5, mode="bilinear", align_corners=False)
    fs = [c1 + x1, maps[0] + x2, maps[1] + outs[2], maps[2] + x4]
    return [_bn(f, sd, f"norm{i + 1}") for i, f in enumerate(fs)]
