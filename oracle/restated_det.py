"""TEST INFRASTRUCTURE — the fp32 oracle of the detection backbone.  Not product code; only tests/ and
scripts/bench_det.py may import it.

A plain PyTorch restatement of ``OnePeace.forward`` (one_peace_vision/det/models/onepeace.py:146-157, 194-216, 304-331,
383-409, 624-629) with rp_bias=False, shared_rp_bias=True and use_decomposed_rel_pos=True, written against a state dict
with the reference's parameter names.  detectron2's window_partition / window_unpartition / add_decomposed_rel_pos are
restated from their documented semantics (square windows, equal query and key grids).  tests/test_det_host_logic.py
pins it to tests/golden/det.pt, which oracle/make_golden_det.py produced from the reference's own file.

``dtype=torch.bfloat16`` runs the same arithmetic with bf16 weights and activations (the soft-max in fp32), the eager
baseline of scripts/bench_det.py; ``sdpa=True`` hands the bias and the decomposed terms to
F.scaled_dot_product_attention as a float mask instead of the explicit soft-max.
"""
import torch
import torch.nn.functional as F


def make_image_bucket_position(bucket_size, num_relative_distance):
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


def shared_bias(table, pretrain_bucket, side):
    """get_rel_pos_bias (onepeace.py:123-144): [H, side^2, side^2] from the shared table, bicubically resized when
    2 side - 1 differs from 2 pretrain_bucket - 1."""
    src, dst = 2 * pretrain_bucket - 1, 2 * side - 1
    bucket = make_image_bucket_position(side, dst * dst + 3)[1:, 1:].to(table.device)
    if src != dst:
        body = table[:-3].view(1, src, src, -1).permute(0, 3, 1, 2)
        body = F.interpolate(body, size=(dst, dst), mode="bicubic")
        table = torch.cat((body.permute(0, 2, 3, 1).reshape(dst * dst, -1), table[-3:]), dim=0)
    return F.embedding(bucket, table).permute(2, 0, 1).contiguous()


def window_partition(x, ws):
    B, H, W, C = x.shape
    x = x.view(B, H // ws, ws, W // ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).reshape(-1, ws, ws, C)


def window_unpartition(win, ws, hw):
    H, W = hw
    B = win.shape[0] // (H * W // ws // ws)
    x = win.view(B, H // ws, W // ws, ws, ws, -1)
    return x.permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, -1)


def decomposed_terms(q, rel_pos_h, rel_pos_w, hw):
    """detectron2 add_decomposed_rel_pos terms for equal query / key grids: q [N, h*w, c] (unscaled) ->
    rel_h [N, h, w, h], rel_w [N, h, w, w]."""
    h, w = hw
    Rh = rel_pos_h[(torch.arange(h)[:, None] - torch.arange(h)[None, :] + h - 1).to(rel_pos_h.device)]
    Rw = rel_pos_w[(torch.arange(w)[:, None] - torch.arange(w)[None, :] + w - 1).to(rel_pos_w.device)]
    r_q = q.reshape(q.shape[0], h, w, -1)
    return torch.einsum("bhwc,hkc->bhwk", r_q, Rh), torch.einsum("bhwc,wkc->bhwk", r_q, Rw)


def attention(sd, p, x, bias, heads, sdpa=False):
    """onepeace.py:194-216 on x [N, h, w, d]; bias [H, L, L]."""
    N, h, w, d = x.shape
    L, hd = h * w, d // heads
    lin = lambda name, t: F.linear(t, sd[p + name + ".weight"], sd.get(p + name + ".bias"))
    split = lambda t: t.reshape(N, L, heads, hd).permute(0, 2, 1, 3).reshape(N * heads, L, hd)
    q, k, v = split(lin("q_proj", x)), split(lin("k_proj", x)), split(lin("v_proj", x))
    rel_h, rel_w = decomposed_terms(q, sd[p + "rel_pos_h"], sd[p + "rel_pos_w"], (h, w))
    full_bias = bias.unsqueeze(0).expand(N, -1, -1, -1).reshape(N * heads, L, L)
    if sdpa:
        dec = (rel_h[:, :, :, :, None] + rel_w[:, :, :, None, :]).reshape(N * heads, L, L)
        o = F.scaled_dot_product_attention(q.view(N, heads, L, hd), k.view(N, heads, L, hd), v.view(N, heads, L, hd),
                                           attn_mask=(full_bias + dec).view(N, heads, L, L).to(q.dtype))
    else:
        attn = (q * hd ** -0.5) @ k.transpose(-2, -1)
        attn = (attn + full_bias).view(N * heads, h, w, h, w)
        attn = (attn + rel_h[:, :, :, :, None] + rel_w[:, :, :, None, :]).view(N * heads, L, L)
        o = attn.softmax(dim=-1, dtype=torch.promote_types(attn.dtype, torch.float32)).to(v.dtype) @ v
    o = o.reshape(N, heads, h, w, hd).permute(0, 2, 3, 1, 4).reshape(N, h, w, d)
    o = F.layer_norm(o, (d,), sd[p + "ln.weight"], sd[p + "ln.bias"])
    return lin("out_proj", o)


def layer(sd, p, x, bias, bias_window, heads, window, sdpa=False):
    """onepeace.py:304-331 (eval: dropout and drop-path are identities)."""
    d = x.shape[-1]
    ln = lambda name, t, n=d: F.layer_norm(t, (n,), sd[p + name + ".weight"], sd[p + name + ".bias"])
    shortcut = x
    y = ln("self_attn_layer_norm", x)
    B, H, W, _ = y.shape
    if window > 0:
        y = window_partition(y, window)
        bias = bias_window
    y = attention(sd, p + "self_attn.", y, bias, heads, sdpa)
    if window > 0:
        y = window_unpartition(y, window, (H, W))
    x = shortcut + sd[p + "gamma_1"] * y
    y = ln("final_layer_norm", x)
    f = p + "image_ffn."
    u = F.gelu(F.linear(y, sd[f + "0.wi_0.weight"])) * F.linear(y, sd[f + "0.wi_1.weight"])
    u = F.layer_norm(u, (u.shape[-1],), sd[f + "2.weight"], sd[f + "2.bias"])
    return x + sd[p + "gamma_2"] * F.linear(u, sd[f + "3.weight"], sd[f + "3.bias"])


def stem(sd, img):
    """ImageAdaptor.forward (onepeace.py:146-152) -> [B, h, w, d]."""
    p = "image_adapter."
    x = F.conv2d(img, sd[p + "embed_images.0.weight"], sd[p + "embed_images.0.bias"], stride=4)
    for i, conv in ((1, 3), (4, 6)):
        c = x.shape[1]
        x = F.layer_norm(x.permute(0, 2, 3, 1), (c,), sd[f"{p}embed_images.{i}.layer_norm.weight"],
                         sd[f"{p}embed_images.{i}.layer_norm.bias"]).permute(0, 3, 1, 2)
        x = F.conv2d(F.gelu(x), sd[f"{p}embed_images.{conv}.weight"], sd[f"{p}embed_images.{conv}.bias"], stride=2)
    x = x.permute(0, 2, 3, 1)
    h, w = x.shape[1:3]
    return x + sd[p + "pos_embed"][1:].unsqueeze(0).reshape(1, h, w, -1)


def forward(sd, img, heads, layers, bucket_size, window_size, window_block_indexes, pretrain_bucket_size=16,
            dtype=torch.float32, sdpa=False):
    """OnePeace.forward -> last_feat [B, d, bucket, bucket] (fp32 for dtype=torch.float32).  pretrain_bucket_size is the
    ImageAdaptor's (the reference builds it with its default 16)."""
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    table = sd["image_adapter.rel_pos_table.weight"]
    bias = shared_bias(table, pretrain_bucket_size, bucket_size)
    bias_window = shared_bias(table, pretrain_bucket_size, window_size)
    x = stem(sd, img.to(dtype))
    for i in range(layers):
        x = layer(sd, f"encoder.layers.{i}.", x, bias, bias_window, heads,
                  window_size if i in window_block_indexes else 0, sdpa)
    return x.permute(0, 3, 1, 2).contiguous()
