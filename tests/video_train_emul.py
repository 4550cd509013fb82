"""fp64 emulation of the video backbone's training launch sequence, forward and adjoint: TemporalEmbedFn,
video_layer_forward / video_layer_backward for every layer (one_peace_b200/vision/video.py) and ClsNormFn, with the
kernels' bf16 rounding points (`rb`: the bf16 weights and every bf16 buffer the sequence writes) and eight planted
mistakes that the tests must tell apart from it.  The yardstick is torch fp64 autograd through the train-mode
restatement tests/video_train_ref.py with the same explicit per-frame drop-path scales.

The input is the stem's output before the temporal embedding (patch + positions, [B T, N, d]); the stem's own adjoint is
ImageEmbedFn's, which tests/test_stem_ref.py covers."""
import torch
import torch.nn.functional as F

import restated_video as RV
import video_train_ref as VT

MISTAKES = ("per_clip_masks", "drop_path_on_ffn", "x1_from_y", "temporal_share_dropped", "no_s_adapter_skip",
            "no_mlp_dh2", "temporal_grad_wrong_axis", "final_norm_patch_rows")


def rb(t):
    return t.to(torch.bfloat16).to(torch.float64)


def _ln(x, w, b, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    rstd = (x.var(-1, unbiased=False, keepdim=True) + eps).rsqrt()
    return (x - mu) * rstd * w + b


def _ln_bwd(x, dy, w, eps=1e-5):
    """-> (dx, dw, db)"""
    mu = x.mean(-1, keepdim=True)
    rstd = (x.var(-1, unbiased=False, keepdim=True) + eps).rsqrt()
    xh = (x - mu) * rstd
    g = dy * w
    dx = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    return dx, (dy * xh).sum(0), dy.sum(0)


def _gelu_grad(z):
    return 0.5 * (1 + torch.erf(z / 2 ** 0.5)) + z * torch.exp(-0.5 * z * z) / (2 * torch.pi) ** 0.5


def _split(qkv, heads):
    B, L, d3 = qkv.shape
    d = d3 // 3
    return [t.view(B, L, heads, d // heads).transpose(1, 2) for t in qkv.split(d, -1)]


def _attn(qkv, heads, bias=None):
    """qkv [B, L, 3d] (q scaled) -> (o [B, L, d], P)"""
    q, k, v = _split(qkv, heads)
    s = q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    p = s.softmax(-1)
    B, L = qkv.shape[:2]
    return (p @ v).transpose(1, 2).reshape(B, L, -1), p


def _attn_bwd(qkv, o, do, p, heads, q_scale):
    """-> (dqkv [B, L, 3d] with dq times q_scale, dS [B, H, L, L])"""
    q, k, v = _split(qkv, heads)
    B, L, d = o.shape
    oh = o.view(B, L, heads, -1).transpose(1, 2)
    doh = do.view(B, L, heads, -1).transpose(1, 2)
    ds = p * (doh @ v.transpose(-1, -2) - (doh * oh).sum(-1, keepdim=True))
    rows = lambda t: t.transpose(1, 2).reshape(B, L, d)
    return torch.cat([rows(q_scale * ds @ k), rows(ds.transpose(-1, -2) @ q), rows(p.transpose(-1, -2) @ doh)], -1), ds


def _to_seq(x, B, T, N):
    """frame-major [B T N, c] -> [(b n), t, c]"""
    return x.view(B, T, N, -1).transpose(1, 2).reshape(B * N, T, -1)


def _from_seq(x, B, T, N):
    return x.view(B, N, T, -1).transpose(1, 2).reshape(B * T * N, -1)


def layer_fwd(sd, pfx, x, B, T, N, heads, bias, scale, rs, mistake):
    """x fp64 [M, d] frame-major -> (x_out, saved); rs: three [M] row scales (or 1.0)."""
    g = lambda n: sd[f"{pfx}.{n}"]
    d = x.shape[1]
    M = x.shape[0]
    qs = torch.ones(3 * d, dtype=x.dtype)
    qs[:d] = (d // heads) ** -0.5
    wqkv = torch.cat([g("self_attn.q_proj.weight"), g("self_attn.k_proj.weight"), g("self_attn.v_proj.weight")])
    bqkv = torch.cat([g("self_attn.q_proj.bias"), torch.zeros(d, dtype=x.dtype), g("self_attn.v_proj.bias")])
    ln1 = (g("self_attn_layer_norm.weight"), g("self_attn_layer_norm.bias"))
    lni = (g("self_attn.ln.weight"), g("self_attn.ln.bias"))
    s = dict(qs=qs, wqkv=wqkv)

    def lin(a, w, b=None):
        return a @ rb(w).t() + (b if b is not None else 0.0)

    def attn_in(rows):
        h1 = rb(_ln(rows, *ln1))
        return h1, rb(lin(h1, wqkv, bqkv) * qs)

    def attn_out(att):
        a2 = rb(_ln(att, *lni))
        return a2, rb(lin(a2, g("self_attn.out_proj.weight"), g("self_attn.out_proj.bias")))

    def fc1(a, ad):
        z = rb(lin(a, g(f"{ad}.D_fc1.weight"), g(f"{ad}.D_fc1.bias")))
        return z, rb(F.gelu(z))
    s["h1t"], s["qkvt"] = attn_in(x)
    att, s["pt"] = _attn(_to_seq(s["qkvt"], B, T, N), heads)
    s["att_t"] = rb(_from_seq(att, B, T, N))
    s["a2t"], s["ot"] = attn_out(s["att_t"])
    s["zt"], s["ht"] = fc1(s["ot"], "T_Adapter")
    s["xt"] = rb(lin(s["ht"], g("T_Adapter.D_fc2.weight"), g("T_Adapter.D_fc2.bias")))
    s["y"] = x + rs[0] * s["xt"]
    s["h1s"], s["qkvs"] = attn_in(s["y"])
    att, s["ps"] = _attn(s["qkvs"].view(B * T, N, -1), heads, bias)
    s["att_s"] = rb(att.reshape(M, d))
    s["a2s"], s["os"] = attn_out(s["att_s"])
    s["zs"], s["hs"] = fc1(s["os"], "S_Adapter")
    s["sb"] = rb(s["os"] + lin(s["hs"], g("S_Adapter.D_fc2.weight"), g("S_Adapter.D_fc2.bias")))
    s["x1"] = (s["y"] if mistake == "x1_from_y" else x) + rs[1] * g("gamma_1") * s["sb"]
    s["h2"] = rb(_ln(s["x1"], g("final_layer_norm.weight"), g("final_layer_norm.bias")))
    f = f"{pfx}.image_ffn"
    s["gl"] = rb(lin(s["h2"], torch.cat([sd[f + ".0.wi_0.weight"], sd[f + ".0.wi_1.weight"]])))
    F_ = s["gl"].shape[1] // 2
    s["u"] = rb(F.gelu(s["gl"][:, :F_]) * s["gl"][:, F_:])
    s["u2"] = rb(_ln(s["u"], sd[f + ".2.weight"], sd[f + ".2.bias"]))
    s["f"] = rb(lin(s["u2"], sd[f + ".3.weight"], sd[f + ".3.bias"]))
    s["zm"], s["hm"] = fc1(s["h2"], "MLP_Adapter")
    s["mo"] = rb(lin(s["hm"], g("MLP_Adapter.D_fc2.weight"), g("MLP_Adapter.D_fc2.bias")))
    ffn_rs = rs[2] if mistake == "drop_path_on_ffn" else 1.0
    return s["x1"] + ffn_rs * g("gamma_2") * s["f"] + rs[2] * scale * s["mo"], s


def layer_bwd(sd, pfx, x, s, dx, B, T, N, heads, scale, rs, mistake):
    """-> (dx_in, {parameter name: gradient}, dbias [H, N, N])"""
    g = lambda n: sd[f"{pfx}.{n}"]
    M, d = dx.shape
    gr = {}

    def put(n, v):
        gr[f"{pfx}.{n}"] = v

    def dxw(dy, w):
        return dy @ rb(w)

    def adapter(dout, z, h, a_in, ad, skip=None):
        put(f"{ad}.D_fc2.weight", dout.t() @ h)
        put(f"{ad}.D_fc2.bias", dout.sum(0))
        dz = rb(rb(dxw(dout, g(f"{ad}.D_fc2.weight"))) * _gelu_grad(z))
        put(f"{ad}.D_fc1.weight", dz.t() @ a_in)
        put(f"{ad}.D_fc1.bias", dz.sum(0))
        return dxw(dz, g(f"{ad}.D_fc1.weight"))
    # joint pass
    dmo = rb(rs[2] * scale * dx)
    dh2m = adapter(dmo, s["zm"], s["hm"], s["h2"], "MLP_Adapter")
    ffn_rs = rs[2] if mistake == "drop_path_on_ffn" else 1.0
    put("gamma_2", (ffn_rs * dx * s["f"]).sum(0))
    df = rb(ffn_rs * g("gamma_2") * dx)
    f = f"{pfx}.image_ffn"
    gr[f + ".3.weight"], gr[f + ".3.bias"] = df.t() @ s["u2"], df.sum(0)
    du, gr[f + ".2.weight"], gr[f + ".2.bias"] = _ln_bwd(s["u"], rb(dxw(df, sd[f + ".3.weight"])), sd[f + ".2.weight"])
    du = rb(du)
    F_ = s["u"].shape[1]
    gg, gl = s["gl"][:, :F_], s["gl"][:, F_:]
    dgl = rb(torch.cat([du * gl * _gelu_grad(gg), du * F.gelu(gg)], 1))
    w01 = torch.cat([sd[f + ".0.wi_0.weight"], sd[f + ".0.wi_1.weight"]])
    dW01 = dgl.t() @ s["h2"]
    gr[f + ".0.wi_0.weight"], gr[f + ".0.wi_1.weight"] = dW01[:F_], dW01[F_:]
    dh2 = rb(rb(dxw(dgl, w01)) + (0.0 if mistake == "no_mlp_dh2" else dh2m))
    d1, dw, db = _ln_bwd(s["x1"], dh2, g("final_layer_norm.weight"))
    put("final_layer_norm.weight", dw)
    put("final_layer_norm.bias", db)
    dx = dx + d1
    # spatial pass
    put("gamma_1", (rs[1] * dx * s["sb"]).sum(0))
    dsb = rb(rs[1] * g("gamma_1") * dx)
    das = adapter(dsb, s["zs"], s["hs"], s["os"], "S_Adapter")
    do_s = rb(das + (0.0 if mistake == "no_s_adapter_skip" else dsb))

    def attn_back(do, att, qkv_seq, o_seq, p, to_seq, from_seq):
        da2 = rb(dxw(do, g("self_attn.out_proj.weight")))
        datt, dlw, dlb = _ln_bwd(att, da2, g("self_attn.ln.weight"))
        dqkv, ds = _attn_bwd(qkv_seq, o_seq, to_seq(rb(datt)), p, heads, (d // heads) ** -0.5)
        dqkv = rb(from_seq(dqkv))
        return dqkv, rb(dxw(dqkv, s["wqkv"])), dlw, dlb, ds
    dqkv_s, dh1s, dlw_s, dlb_s, ds = attn_back(do_s, s["att_s"], s["qkvs"].view(B * T, N, -1), s["att_s"].view(B * T, N, -1),
                                               s["ps"], lambda t: t.view(B * T, N, -1), lambda t: t.reshape(M, -1))
    dbias = ds.sum(0)
    dy, d1w_s, d1b_s = _ln_bwd(s["y"], dh1s, g("self_attn_layer_norm.weight"))
    if mistake == "x1_from_y":               # x reaches x1 only through y
        dy = dy + dx
        dx = dy
    else:
        dx = dx + dy
    # temporal pass
    dxt = rb(rs[0] * dy)
    do_t = rb(adapter(dxt, s["zt"], s["ht"], s["ot"], "T_Adapter"))
    dqkv_t, dh1t, dlw_t, dlb_t, _ = attn_back(do_t, s["att_t"], _to_seq(s["qkvt"], B, T, N), _to_seq(s["att_t"], B, T, N),
                                              s["pt"], lambda t: _to_seq(t, B, T, N), lambda t: _from_seq(t, B, T, N))
    d1, d1w_t, d1b_t = _ln_bwd(x, dh1t, g("self_attn_layer_norm.weight"))
    dx = dx + d1
    # the shared weights: both passes' rows
    k = 0.0 if mistake == "temporal_share_dropped" else 1.0
    do = torch.cat([k * do_t, do_s])
    a2 = torch.cat([s["a2t"], s["a2s"]])
    dqkv = torch.cat([k * dqkv_t, dqkv_s])
    h1 = torch.cat([s["h1t"], s["h1s"]])
    put("self_attn.out_proj.weight", do.t() @ a2)
    put("self_attn.out_proj.bias", do.sum(0))
    dW, dbq = dqkv.t() @ h1, dqkv.sum(0)
    put("self_attn.q_proj.weight", dW[:d])
    put("self_attn.k_proj.weight", dW[d:2 * d])
    put("self_attn.v_proj.weight", dW[2 * d:])
    put("self_attn.q_proj.bias", dbq[:d])
    put("self_attn.v_proj.bias", dbq[2 * d:])
    put("self_attn.ln.weight", k * dlw_t + dlw_s)
    put("self_attn.ln.bias", k * dlb_t + dlb_s)
    put("self_attn_layer_norm.weight", k * d1w_t + d1w_s)
    put("self_attn_layer_norm.bias", k * d1b_t + d1b_s)
    return dx, gr, dbias


def step(sd, p0, T, heads, layers, rs_frames, cot, scale=0.5, mistake=None):
    """p0 fp64 [B T, N, d] (stem rows before the temporal embedding); rs_frames: per layer three per-frame scales [B T];
    cot [B, d, T, 1, 1].  -> (out [B, d, T, 1, 1], {name: gradient}, dp0)."""
    BT, N, d = p0.shape
    B, M = BT // T, BT * N
    if mistake == "per_clip_masks":
        rs_frames = [tuple(r.view(B, T)[:, :1].expand(B, T).reshape(-1) for r in trip) for trip in rs_frames]
    rows = lambda r: r.repeat_interleave(N)[:, None]
    temporal = sd["image_adapter.temporal_embedding"][0, :T]
    x = p0.reshape(M, d) + temporal.repeat_interleave(N, 0).repeat(B, 1)
    bias = sd["image_adapter.rel_pos_table.weight"][sd["image_adapter.rp_bucket"]].permute(2, 0, 1)
    xs, saved = [], []
    for i in range(layers):
        xs.append(x)
        x, s = layer_fwd(sd, f"encoder.layers.{i}", x, B, T, N, heads, bias, scale, [rows(r) for r in rs_frames[i]], mistake)
        saved.append(s)
    lw, lb = sd["encoder.image_layer_norm.weight"], sd["encoder.image_layer_norm.bias"]
    cls = x.view(BT, N, d)[:, 0]
    out = _ln(cls, lw, lb).view(B, T, d).permute(0, 2, 1)[..., None, None]
    # adjoint
    dcls = cot[..., 0, 0].permute(0, 2, 1).reshape(BT, d)
    dcls_x, dlw, dlb = _ln_bwd(cls, dcls, lw)
    grads = {"encoder.image_layer_norm.weight": dlw, "encoder.image_layer_norm.bias": dlb}
    dx = torch.zeros(BT, N, d, dtype=x.dtype)
    dx[:, 1 if mistake == "final_norm_patch_rows" else 0] = dcls_x
    dx = dx.view(M, d)
    dbias = torch.zeros_like(bias)
    for i in reversed(range(layers)):
        dx, gr, db = layer_bwd(sd, f"encoder.layers.{i}", xs[i], saved[i], dx, B, T, N, heads, scale,
                               [rows(r) for r in rs_frames[i]], mistake)
        grads.update(gr)
        dbias = dbias + db
    dtable = torch.zeros_like(sd["image_adapter.rel_pos_table.weight"])
    dtable.index_put_((sd["image_adapter.rp_bucket"].flatten(),), dbias.permute(1, 2, 0).reshape(N * N, -1), accumulate=True)
    grads["image_adapter.rel_pos_table.weight"] = dtable
    dtemp = torch.zeros_like(sd["image_adapter.temporal_embedding"])
    r = torch.arange(M)
    frame = (r // (T * N)) % T if mistake == "temporal_grad_wrong_axis" else (r // N) % T     # wrong: the clip index
    dtemp[0].index_add_(0, frame, dx)
    grads["image_adapter.temporal_embedding"] = dtemp
    return out, grads, dx.view(BT, N, d)


def reference(sd, p0, T, heads, layers, rs_frames, cot, scale=0.5):
    """torch fp64 autograd through tests/video_train_ref.py on the same input and masks."""
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    p0 = p0.clone().requires_grad_(True)
    BT, N, d = p0.shape
    B = BT // T
    x = (p0.view(B, T, N, d) + sdg["image_adapter.temporal_embedding"][0, :T].view(1, T, 1, d)).view(BT, N, d)
    bias = sdg["image_adapter.rel_pos_table.weight"][sdg["image_adapter.rp_bucket"]].permute(2, 0, 1)
    for i in range(layers):
        x = VT.layer(sdg, f"encoder.layers.{i}", x, T, heads, bias, scale, rs_frames[i])
    out = RV._ln(x[:, 0], sdg, "encoder.image_layer_norm").view(B, T, -1).permute(0, 2, 1)[..., None, None]
    (out * cot).sum().backward()
    grads = {k: v.grad for k, v in sdg.items() if torch.is_tensor(v) and v.requires_grad and v.grad is not None}
    return out.detach(), grads, p0.grad
