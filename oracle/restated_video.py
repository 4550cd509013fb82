"""TEST INFRASTRUCTURE.  An fp32 restatement of the Kinetics-400 video backbone's evaluation forward
(one_peace_vision/video/mmaction_custom/models/backbones/onepeace.py, num_tadapter=1, rp_bias=False, shared table), written
for this project from the reference's documented computation and pinned to the reference by tests/golden/video.pt.  It
takes a state dict of the reference's names and runs on any device, so the GPU tests use it as the fp32 yardstick of the
40-layer backbone.
"""
import torch
import torch.nn.functional as F


def _ln(x, sd, p, eps=1e-5):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], eps)


def _lin(x, sd, p, bias=True):
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias") if bias else None)


def _adapter(x, sd, p, skip):
    y = _lin(F.gelu(_lin(x, sd, p + ".D_fc1")), sd, p + ".D_fc2")
    return x + y if skip else y


def _attn(x, sd, p, heads, bias=None):
    """x [B, L, d] -> attention with the inner LayerNorm and out_proj (q scaled after its bias)."""
    B, L, d = x.shape
    hd = d // heads
    q = (_lin(x, sd, p + ".q_proj") * hd ** -0.5).view(B, L, heads, hd).transpose(1, 2)
    k = _lin(x, sd, p + ".k_proj", bias=False).view(B, L, heads, hd).transpose(1, 2)
    v = _lin(x, sd, p + ".v_proj").view(B, L, heads, hd).transpose(1, 2)
    s = q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    o = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, L, d)
    return _lin(_ln(o, sd, p + ".ln"), sd, p + ".out_proj")


def stem(sd, frames, T):
    """frames [B T, 3, R, R] clip-major -> ((patch + pos) + temporal[t]) fp32 [B T, N, d]."""
    p = "image_adapter.embed_images"
    y = frames
    for i, (conv, ln) in enumerate(((0, 1), (3, 4))):
        y = F.conv2d(y, sd[f"{p}.{conv}.weight"], sd[f"{p}.{conv}.bias"], stride=4 if i == 0 else 2)
        y = F.gelu(_ln(y.permute(0, 2, 3, 1), sd, f"{p}.{ln}.layer_norm").permute(0, 3, 1, 2))
    y = F.conv2d(y, sd[f"{p}.6.weight"], sd[f"{p}.6.bias"], stride=2).flatten(2).transpose(1, 2)
    BT, _, d = y.shape
    x = torch.cat([sd["image_adapter.cls_embedding"].expand(BT, -1, -1), y], dim=1) + sd["image_adapter.pos_embed"]
    N = x.shape[1]
    x = x.view(BT // T, T, N, d) + sd["image_adapter.temporal_embedding"][0, :T].view(1, T, 1, d)
    return x.view(BT, N, d)


def layer(sd, p, x, T, heads, bias, scale):
    """One layer on x [B T, N, d] (frame-major)."""
    BT, N, d = x.shape
    B = BT // T
    xt = x.view(B, T, N, d).transpose(1, 2).reshape(B * N, T, d)                 # (b n) t d
    xt = _adapter(_attn(_ln(xt, sd, p + ".self_attn_layer_norm"), sd, p + ".self_attn", heads), sd, p + ".T_Adapter", False)
    y = x + xt.view(B, N, T, d).transpose(1, 2).reshape(BT, N, d)
    a = _adapter(_attn(_ln(y, sd, p + ".self_attn_layer_norm"), sd, p + ".self_attn", heads, bias), sd, p + ".S_Adapter", True)
    x = x + sd[p + ".gamma_1"] * a
    xn = _ln(x, sd, p + ".final_layer_norm")
    f = p + ".image_ffn"
    h = F.gelu(F.linear(xn, sd[f + ".0.wi_0.weight"])) * F.linear(xn, sd[f + ".0.wi_1.weight"])
    ffn = _lin(_ln(h, sd, f + ".2"), sd, f + ".3")
    return x + sd[p + ".gamma_2"] * ffn + scale * _adapter(xn, sd, p + ".MLP_Adapter", False)


def features(sd, clips, heads, layers, scale=0.5):
    """clips [B, 3, T, R, R] -> the last layer's rows fp32 [B T, N, d] before image_layer_norm."""
    B, _, T, R, _ = clips.shape
    x = stem(sd, clips.transpose(1, 2).reshape(B * T, 3, R, R), T)
    bias = sd["image_adapter.rel_pos_table.weight"][sd["image_adapter.rp_bucket"]].permute(2, 0, 1)
    for i in range(layers):
        x = layer(sd, f"encoder.layers.{i}", x, T, heads, bias, scale)
    return x


def forward(sd, clips, heads, layers, scale=0.5):
    """-> image_layer_norm of the CLS rows, fp32 [B, d, T, 1, 1]."""
    B, _, T = clips.shape[:3]
    x = _ln(features(sd, clips, heads, layers, scale)[:, 0], sd, "encoder.image_layer_norm")
    return x.view(B, T, -1).permute(0, 2, 1)[..., None, None]
