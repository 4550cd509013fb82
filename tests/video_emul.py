"""fp64 emulation of VideoLayer.forward_video's launch sequence, with the kernels' bf16 rounding points (the bf16 weights,
and every bf16 buffer the sequence writes: xb, qkv, o, a, h, yb, u), and seven planted mistakes that each tests must tell
apart from it.  The oracle is oracle/restated_video.features in fp64, the reference's computation without rounding."""
import torch
import torch.nn.functional as F

import restated_video as RV

MISTAKES = ("resid_from_y", "t_b_grouping", "temporal_skips_cls", "scale_on_ffn", "no_gamma1_on_a", "t_adapter_skip",
            "ln2_after_mlp")


def rb(t):
    return t.to(torch.bfloat16).to(torch.float64)


def _lin(x, w, b=None):
    return x @ rb(w).t() + (b if b is not None else 0.0)


def _ln_lin(x, ln_w, ln_b, w, b=None, eps=1e-5):
    """LayerNorm folded into the GEMM: statistics of the fp32 rows, the bf16 copy as A, bf16 W diag(g), fp64 W beta + b."""
    mu = x.mean(-1, keepdim=True)
    rstd = (x.var(-1, unbiased=False, keepdim=True) + eps).rsqrt()
    return ((rb(x) - mu) * rstd) @ rb(w * ln_w).t() + (w @ ln_b + (b if b is not None else 0.0))


def _attn(qkv, heads, bias=None):
    """qkv [B, L, 3d] (bf16 values) -> softmax(q k^T + bias) v, [B, L, d]"""
    B, L, d3 = qkv.shape
    d = d3 // 3
    q, k, v = (t.view(B, L, heads, d // heads).transpose(1, 2) for t in qkv.split(d, -1))
    s = q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    return (s.softmax(-1) @ v).transpose(1, 2).reshape(B, L, d)


def layer(sd, p, x, T, heads, bias, scale, mistake=None):
    """x fp64 [B T, N, d] frame-major -> the layer output, as the launch sequence computes it."""
    BT, N, d = x.shape
    B = BT // T
    g = lambda n: sd[f"{p}.{n}"]
    a_ = f"{p}.self_attn"
    wqkv = torch.cat([g("self_attn.q_proj.weight"), g("self_attn.k_proj.weight"), g("self_attn.v_proj.weight")])
    bqkv = torch.cat([g("self_attn.q_proj.bias"), torch.zeros(d, dtype=x.dtype), g("self_attn.v_proj.bias")])
    qs = torch.ones(3 * d, dtype=x.dtype)
    qs[:d] = (d // heads) ** -0.5
    ln1 = (g("self_attn_layer_norm.weight"), g("self_attn_layer_norm.bias"))
    lni = (sd[a_ + ".ln.weight"], sd[a_ + ".ln.bias"])

    def qkv_of(rows):
        return rb(_ln_lin(rows, *ln1, wqkv, bqkv) * qs)

    def out_proj(o):
        return rb(_ln_lin(o, *lni, sd[a_ + ".out_proj.weight"], sd[a_ + ".out_proj.bias"]))

    def fc1(t, ad):
        return rb(F.gelu(_lin(t, g(f"{ad}.D_fc1.weight"), g(f"{ad}.D_fc1.bias"))))

    def fc2(h, ad):
        return _lin(h, g(f"{ad}.D_fc2.weight"), g(f"{ad}.D_fc2.bias"))

    # temporal pass: attention along t for every (b, n)
    qkv = qkv_of(x)
    if mistake == "t_b_grouping":            # frames grouped as (t b): sequences over the clips of one frame index
        seq = qkv.view(B, T, N, 3 * d).permute(1, 2, 0, 3).reshape(T * N, B, 3 * d)
        o = rb(_attn(seq, heads)).view(T, N, B, d).permute(2, 0, 1, 3).reshape(BT, N, d)
    else:
        seq = qkv.view(B, T, N, 3 * d).transpose(1, 2).reshape(B * N, T, 3 * d)
        o = rb(_attn(seq, heads)).view(B, N, T, d).transpose(1, 2).reshape(BT, N, d)
    at = out_proj(o)
    xt = fc2(fc1(at, "T_Adapter"), "T_Adapter")
    if mistake == "t_adapter_skip":
        xt = xt + at
    y = x + xt
    # spatial pass
    a = out_proj(rb(_attn(qkv_of(y), heads, bias)))
    s = fc2(fc1(a, "S_Adapter"), "S_Adapter")
    resid = y if mistake == "resid_from_y" else x
    x = resid + g("gamma_1") * (s + (a / g("gamma_1") if mistake == "no_gamma1_on_a" else a))
    # joint pass
    ln2 = (g("final_layer_norm.weight"), g("final_layer_norm.bias"))
    f = f"{p}.image_ffn"
    wi = _ln_lin(x, *ln2, torch.cat([sd[f + ".0.wi_0.weight"], sd[f + ".0.wi_1.weight"]]))
    u = rb(F.gelu(wi[..., :wi.shape[-1] // 2]) * wi[..., wi.shape[-1] // 2:])
    ffn = _ln_lin(u, sd[f + ".2.weight"], sd[f + ".2.bias"], sd[f + ".3.weight"], sd[f + ".3.bias"])
    hm = rb(F.gelu(_ln_lin(x, *ln2, g("MLP_Adapter.D_fc1.weight"), g("MLP_Adapter.D_fc1.bias"))))
    if mistake == "scale_on_ffn":
        return x + scale * g("gamma_2") * ffn + fc2(hm, "MLP_Adapter")
    x = x + g("gamma_2") * ffn
    if mistake == "ln2_after_mlp":
        hm = rb(F.gelu(_ln_lin(x, *ln2, g("MLP_Adapter.D_fc1.weight"), g("MLP_Adapter.D_fc1.bias"))))
    return x + scale * fc2(hm, "MLP_Adapter")


def features(sd, clips, heads, layers, scale=0.5, mistake=None):
    """clips [B, 3, T, R, R] -> fp64 rows [B T, N, d] after the last layer, through the emulated launch sequence."""
    B, _, T, R, _ = clips.shape
    x = RV.stem(sd, clips.transpose(1, 2).reshape(B * T, 3, R, R), T)
    if mistake == "temporal_skips_cls":
        x = x.clone()
        x[:, 0] -= sd["image_adapter.temporal_embedding"][0, :T].repeat(B, 1)
    bias = sd["image_adapter.rel_pos_table.weight"][sd["image_adapter.rp_bucket"]].permute(2, 0, 1)
    for i in range(layers):
        x = layer(sd, f"encoder.layers.{i}", x, T, heads, bias, scale, mistake)
    return x
