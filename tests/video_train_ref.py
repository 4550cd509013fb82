"""Train-mode restatement of the video backbone for the tests: oracle/restated_video.py's layer with the reference's three
drop-path terms (onepeace.py:328-352) given as explicit per-frame scales, so that torch autograd through it is the
yardstick of OnePeaceViT's training forward and adjoint.  Masks are regenerated from an RNG state by
``row_scales``, in the order one_peace_b200.vision.video.draw_row_scales documents."""
import torch
import torch.utils.checkpoint as cp

import restated_video as RV


def layer(sd, p, x, T, heads, bias, scale, rs=(None, None, None)):
    """One layer on x [B T, N, d] (frame-major); rs: three per-frame scales [B T] or None (no drop-path)."""
    BT, N, d = x.shape
    B = BT // T
    m = [None if r is None else r.view(BT, 1, 1).to(x.dtype) for r in rs]
    xt = x.view(B, T, N, d).transpose(1, 2).reshape(B * N, T, d)
    xt = RV._adapter(RV._attn(RV._ln(xt, sd, p + ".self_attn_layer_norm"), sd, p + ".self_attn", heads), sd, p + ".T_Adapter",
                     False)
    xt = xt.view(B, N, T, d).transpose(1, 2).reshape(BT, N, d)
    y = x + (xt if m[0] is None else m[0] * xt)
    a = RV._adapter(RV._attn(RV._ln(y, sd, p + ".self_attn_layer_norm"), sd, p + ".self_attn", heads, bias), sd,
                    p + ".S_Adapter", True)
    a = sd[p + ".gamma_1"] * a
    x = x + (a if m[1] is None else m[1] * a)
    xn = RV._ln(x, sd, p + ".final_layer_norm")
    f = p + ".image_ffn"
    h = torch.nn.functional.gelu(torch.nn.functional.linear(xn, sd[f + ".0.wi_0.weight"])) * \
        torch.nn.functional.linear(xn, sd[f + ".0.wi_1.weight"])
    ffn = RV._lin(RV._ln(h, sd, f + ".2"), sd, f + ".3")
    mlp = scale * RV._adapter(xn, sd, p + ".MLP_Adapter", False)
    return x + sd[p + ".gamma_2"] * ffn + (mlp if m[2] is None else m[2] * mlp)


def rows(sd, clips, heads, layers, scale=0.5, masks=None, checkpoint=False):
    """clips [B, 3, T, R, R] -> the last layer's rows [B T, N, d]; masks: per layer a triple of [B T] scales or None."""
    B, _, T, R, _ = clips.shape
    x = RV.stem(sd, clips.transpose(1, 2).reshape(B * T, 3, R, R), T)
    bias = sd["image_adapter.rel_pos_table.weight"][sd["image_adapter.rp_bucket"]].permute(2, 0, 1)
    for i in range(layers):
        rs = masks[i] if masks is not None else (None, None, None)
        fn = lambda x_, i=i, rs=rs: layer(sd, f"encoder.layers.{i}", x_, T, heads, bias, scale, rs)
        x = cp.checkpoint(fn, x, use_reentrant=False) if checkpoint else fn(x)
    return x


def forward(sd, clips, heads, layers, scale=0.5, masks=None, checkpoint=False):
    """-> image_layer_norm of the CLS rows [B, d, T, 1, 1]."""
    B, _, T = clips.shape[:3]
    x = RV._ln(rows(sd, clips, heads, layers, scale, masks, checkpoint)[:, 0], sd, "encoder.image_layer_norm")
    return x.view(B, T, -1).permute(0, 2, 1)[..., None, None]


def row_scales(drop_probs, BT, rng_state, device):
    """The per-frame drop-path scales of each layer, drawn again from the CUDA RNG state saved before the forward: per
    layer with p > 0, three torch.rand(B T) (temporal, spatial, MLP adapter), keep = draw < 1 - p, scale = keep / (1 - p)."""
    out = []
    with torch.random.fork_rng(devices=[device]):
        torch.cuda.set_rng_state(rng_state, device)
        for p in drop_probs:
            if p <= 0:
                out.append((None, None, None))
                continue
            keep = 1.0 - p
            out.append(tuple((torch.rand(BT, device=device) < keep).float() / keep for _ in range(3)))
    return out
