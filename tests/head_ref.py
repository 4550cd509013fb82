"""fp64 references of the training Functions around the encoder stack: the classification heads and criteria
(one_peace_b200/autograd_classify.py: ``ClassifyHeadFn``, ``ClassifyLossFn``, ``RefcocoLossFn``, ``VitHeadFn``) and the
pretraining-path pieces (one_peace_b200/autograd_general.py: ``BlockBiasFn``, ``RowGatherFn``, ``ZeroPadFn``,
``LinearFn``, ``FinalNormFn``, ``DclLossFn``), forward and adjoint, stage by stage, with an error bound for every output
element.

Plain PyTorch on whatever device the inputs live on; nothing here calls the extension.  The method is tests/stem_ref.py's
and so are its helpers (``anchor``, ``vjp``, ``kernel_calls``, ``ln_bwd_of``, ``ln_stage``, ``share``).

Reference
---------
fp64 torch autograd of the reference model's own operations with bf16-rounded weights: ``MultiheadAttentionPooling`` and
``OnePeaceClassifyHead`` (one_peace_base.py:132-230: ``k_proj`` without bias, an unscaled ``q``, softmax over the keys
that are not padding, ``norm``, the pooler's tanh(Linear), the two passes of ``use_two_images`` concatenated along the
features, Linear -> LayerNorm -> GELU -> Linear), the ViT head (models_vit.py:431-434), ``compute_dcl_loss``
(image_text_pretrain_loss.py:187-208, ``adjust_label_smoothed_nll_loss``), ``F.linear``, ``F.layer_norm``, gathers and
masked fills.  The criteria's references are the fp64 closed forms of test_classify_host_logic.py and grounding_ref.py,
which their own tests hold to torch's criteria and autograd.

Forward: the reference is anchored to the activations the Function saved, ``v = v_ref + (v_dev - v_ref).detach()``, and
each saved stage is checked against the reference operation applied to the device's previous stage.  The pooler's tanh
is anchored at the device's pre-activation atanh(t_dev), so that its derivative is the 1 - t^2 the device uses.

Adjoint: each stage is checked from the cotangent the device handed it (dl, dg, dh, dcin, dt, dzn, dy, do, dkv; da;
grad_n, dx32; read from the kernel calls, ``kernel_calls`` and ``ln_bwd_of``).  A bound then carries the error of one
kernel, plus, where the Function itself rounds, that one rounding:
  bf16 dl on entry to a head backward         a stage of its own: bf16(dlogits), bound 0 (+ u_out)
  dt = bf16(dpool * (1 - t*t)) in fp32        |dpool| (u t^2 + 2u |1 - t^2|) (+ u_out)
  (dl * g_loss) and (dx32 * g_loss) in fp32   u |value|
Single-kernel bounds come from their own modules: GEMMs tau |A| |B| (kernel_ref.TAU), LayerNorm ``ln_stage`` /
``layernorm_ref``, attention pooling ``pool_fwd_ref`` / ``pool_bwd_ref`` and the criteria ``loss_ref``
(test_classify_host_logic.py), ``refcoco`` (grounding_ref.py), ``head_fwd`` / ``head_bwd`` (vit_ref.py), ``infonce_ref`` /
``infonce_grad_ref`` / ``l2_normalize_ref`` / ``l2_normalize_bwd_ref`` / ``scatter_ref`` (kernel_ref.py).  Column sums
(bias gradients) are tau sum |terms|.

Where the reference is exactly zero the bound is zero, so the device value must be exactly zero: dfeats on the CLS row,
dkv on padded keys, the ViT CLS form's dx off the CLS rows, padded rows of ZeroPadFn, student rows outside stu_idx,
bias-table rows no bucket uses, unused rows of a gathered source, the padded columns of a classifier's dl.
"""
import torch
import torch.nn.functional as F

from grounding_ref import refcoco
from kernel_ref import (TAU, U32, infonce_grad_ref, infonce_ref, l2_normalize_bwd_ref, l2_normalize_ref, layernorm_ref,
                        scatter_ref)
from stem_ref import BF, F32, _f32, anchor, b64, kernel_calls, leaf, ln_bwd_of, ln_stage, vjp
from test_classify_host_logic import HARD, HINGE, MULTI, SOFT, loss_ref, pool_bwd_ref, pool_fwd_ref
from vit_ref import head_bwd, head_fwd

TANH_ULP = 2            # torch's fp32 tanh: CUDA's tanhf is within 2 ulp (CUDA C++ Programming Guide, math functions)


def dx_of(log, dy):
    """result of the ``_dx(dy, W, ...)`` GEMM of a recorded backward: the gemm_t call that contracts dy (as given) with an
    MN-major weight"""
    hits = [r for a, kw, r in kernel_calls(log, "gemm_t") if a[0] is dy and kw.get("b_mn") and not kw.get("a_mn")]
    assert len(hits) == 1, f"{len(hits)} dX GEMMs read this gradient"
    return hits[0]


def _zeros(t):
    return torch.zeros(t.shape, dtype=torch.float64, device=t.device)


def _linear_mag(x, w, b=None):
    """|x| |W|^T (+ |b|): the magnitude a GEMM's tau bound multiplies"""
    m = x.detach().double().abs() @ w.detach().double().abs().t()
    return m if b is None else m + b.detach().double().abs()


def _pool(kv, q, valid, N, T):
    """MultiheadAttentionPooling.forward before out_proj (one_peace_base.py:146-172) on the k | v rows [N*T, 2d]: the
    unscaled q [H, 64] against k, softmax over the keys that are not padding, the weights on v -> [N, d]"""
    H = q.shape[0]
    k, v = kv.view(N, T, 2, H, 64).unbind(2)
    s = torch.einsum("nthe,he->nht", k, q).masked_fill(~valid[:, None, :], float("-inf"))
    return torch.einsum("nht,nthe->nhe", torch.softmax(s, -1), v).reshape(N, H * 64)


# ----------------------------------------------------------------------------------------------------------------------
# ClassifyHeadFn: attention pooling, out_proj, norm, pooler, [pass 1 | pass 2], Linear, LayerNorm + GELU, Linear
# ----------------------------------------------------------------------------------------------------------------------
CLASSIFY_GRADS = ("nw", "nb", "q", "wk", "wv", "bv", "wo", "bo", "wp", "bp", "w0", "b0", "g1", "be1", "w3", "b3")


def classify_head_ref(feats, key_pad, eps_n, eps_c, params, saved, dlogits, log):
    """feats: (f1,) or (f1, f2) [B, S, d] as given; key_pad [B, S] (nonzero = padding) or None; params: the 16
    ``head_params`` (None for an absent pooler); saved: ``ctx.saved``; dlogits [B, n_cls] the upstream gradient; log: the
    kernel calls of the backward.  Returns (checks, got): checks[name] = (reference, bound, out dtype) for the forward
    stages, the backward intermediates and the gradients (f1, f2 and CLASSIFY_GRADS); got[name] = the device's forward
    stages and backward intermediates."""
    P = len(feats)
    B, S, d = feats[0].shape
    T, H, N = S - 1, d // 64, len(feats) * B
    nw, nb, q, wk, wv, bv, wo, bo, wp, bp, w0, b0, g1, be1, w3, b3 = params
    pool = wp is not None
    n_cls, inner = w3.shape[0], w0.shape[0]
    s = saved
    Xs = [leaf(f) for f in feats]
    Nw, Nb, Q, Wk, Wv, Bv, Wo, Bo = (leaf(nw), leaf(nb), leaf(q), leaf(b64(wk)), leaf(b64(wv)), leaf(bv), leaf(b64(wo)),
                                     leaf(bo))
    W0, B0, G1, Be1, W3, B3 = leaf(b64(w0)), leaf(b0), leaf(g1), leaf(be1), leaf(b64(w3)), leaf(b3)
    q64 = Q.reshape(H, 64)
    dev = feats[0].device
    # forward_features of each pass reads padding_masks[:, 1:] (one_peace_base.py:218-219): the same mask for both passes
    valid = (torch.ones(B, T, dtype=torch.bool, device=dev) if key_pad is None else key_pad[:, 1:] == 0).repeat(P, 1)
    kp_ref = (~valid).to(torch.uint8)
    chk, got = {}, {k: s[k] for k in ("xb", "kv", "o", "lse", "y", "zn", "cin", "h", "g")}

    xb_r = torch.cat([X[:, 1:] for X in Xs]).reshape(N * T, d)
    xb = anchor(xb_r, s["xb"])
    kv_r = torch.cat([F.linear(xb, Wk), F.linear(xb, Wv, Bv)], 1)
    kv = anchor(kv_r, s["kv"])
    o_r = _pool(kv, q64, valid, N, T)
    o = anchor(o_r, s["o"])
    y_r = F.linear(o, Wo, Bo)
    y = anchor(y_r, s["y"])
    zn_r = F.layer_norm(y, (d,), Nw, Nb, eps_n)
    zn = anchor(zn_r, s["zn"])
    if pool:
        Wp, Bp = leaf(b64(wp)), leaf(bp)
        t_dev = s["t"].double()
        assert (t_dev.abs() < 1).all(), "a pooler unit saturated to +-1 in fp32: its derivative cannot be anchored"
        pre = anchor(F.linear(zn, Wp, Bp), torch.atanh(t_dev))
        pooled = torch.tanh(pre)
        got["t"] = s["t"]
    else:
        pooled = zn
    cin_r = pooled if P == 1 else torch.cat([pooled[:B], pooled[B:]], 1)
    cin = anchor(cin_r, s["cin"])
    h_r = F.linear(cin, W0, B0)
    h = anchor(h_r, s["h"])
    g_r = F.gelu(F.layer_norm(h, (inner,), G1, Be1, eps_c))
    g = anchor(g_r, s["g"])
    l_r = F.linear(g, W3, B3)
    with torch.no_grad():
        chk["xb"] = (xb_r.detach(), _zeros(xb_r), BF)
        mk = TAU * torch.cat([_linear_mag(s["xb"], Wk), _linear_mag(s["xb"], Wv, Bv)], 1)
        chk["kv"] = (kv_r.detach(), mk, BF)
        _, lse_r, b_o, b_lse = pool_fwd_ref(s["kv"], q64.detach(), kp_ref, N, T)
        chk["o"] = (o_r.detach(), b_o, F32)                          # b_o holds the bf16 rounding
        chk["lse"] = (lse_r, b_lse, F32)
        chk["y"] = (y_r.detach(), TAU * _linear_mag(s["o"], Wo, Bo), F32)
        chk["zn"] = (zn_r.detach(), layernorm_ref(s["y"], _f32(nw), _f32(nb), eps_n).err, BF)
        if pool:
            t_r = torch.tanh(F.linear(s["zn"].double(), Wp, Bp))
            e = TAU * _linear_mag(s["zn"], Wp, Bp)                    # |tanh'| <= 1 - t^2 + e within e of the point
            chk["t"] = (t_r, e * (1 - t_r * t_r + e) + TANH_ULP * U32 * t_r.abs(), F32)
        chk["cin"] = (cin_r.detach(), _zeros(cin_r), BF)
        chk["h"] = (h_r.detach(), TAU * _linear_mag(s["cin"], W0, B0), F32)
        chk["g"] = (g_r.detach(), layernorm_ref(s["h"], _f32(g1), _f32(be1), eps_c, gelu=True).err, BF)
        chk["logits"] = (l_r.detach(), TAU * _linear_mag(s["g"], W3, B3), F32)

    # the device's backward intermediates
    dl = kernel_calls(log, "colsum")[0][0][0]
    dg, dh, _ = ln_bwd_of(log, s["h"])
    dzn, dy, _ = ln_bwd_of(log, s["y"])
    ((pa, _, (dkv, _)),) = kernel_calls(log, "attn_pool_bwd")
    do, dcin = pa[4], dx_of(log, dh)
    got.update(dl=dl, dg=dg, dh=dh, dcin=dcin, dzn=dzn, dy=dy, do=do, dkv=dkv)
    n_pad = dl.shape[1]
    ref, bound = {}, {}
    dlc = dl[:, :n_cls]
    chk["dl"] = (F.pad(dlogits.double(), (0, n_pad - n_cls)), torch.zeros(B, n_pad, dtype=torch.float64, device=dev), BF)
    ref["w3"], ref["b3"], r = vjp(l_r, [W3, B3, g], dlc)
    a = dlc.double().abs()
    bound["w3"], bound["b3"] = TAU * (a.t() @ s["g"].double().abs()), TAU * a.sum(0)
    chk["dg"] = (r, TAU * (a @ W3.abs()), BF)
    r, ref["g1"], ref["be1"] = vjp(g_r, [h, G1, Be1], dg)
    ex, bound["g1"], bound["be1"] = ln_stage(s["h"], dg, _f32(g1), _f32(be1), eps_c, True)
    chk["dh"] = (r, ex, BF)
    ref["w0"], ref["b0"], r = vjp(h_r, [W0, B0, cin], dh)
    a = dh.double().abs()
    bound["w0"], bound["b0"] = TAU * (a.t() @ s["cin"].double().abs()), TAU * a.sum(0)
    chk["dcin"] = (r, TAU * (a @ W0.abs()), BF)
    if pool:
        dt = kernel_calls(log, "colsum")[2][0][0]
        got["dt"] = dt
        r_dt, dpool = vjp(cin_r, [pre, pooled], dcin)               # dpool: dcin split back into the passes (exact)
        tt = t_dev * t_dev
        chk["dt"] = (r_dt, dpool.abs() * (U32 * tt + 2 * U32 * (1 - tt).abs()), BF)
        ref["wp"], ref["bp"], r = vjp(pre, [Wp, Bp, zn], dt)
        a = dt.double().abs()
        bound["wp"], bound["bp"] = TAU * (a.t() @ s["zn"].double().abs()), TAU * a.sum(0)
        chk["dzn"] = (r, TAU * (a @ Wp.abs()), BF)
    else:
        (r,) = vjp(cin_r, [zn], dcin)
        chk["dzn"] = (r, _zeros(r), BF)
    r, ref["nw"], ref["nb"] = vjp(zn_r, [y, Nw, Nb], dzn)
    ex, bound["nw"], bound["nb"] = ln_stage(s["y"], dzn, _f32(nw), _f32(nb), eps_n, False)
    chk["dy"] = (r, ex, BF)
    ref["wo"], ref["bo"], r = vjp(y_r, [Wo, Bo, o], dy)
    a = dy.double().abs()
    bound["wo"], bound["bo"] = TAU * (a.t() @ s["o"].double().abs()), TAU * a.sum(0)
    chk["do"] = (r, TAU * (a @ Wo.abs()), BF)
    r, ref["q"] = vjp(o_r, [kv, Q], do)
    _, _, b_dkv, bound["q"] = pool_bwd_ref(s["kv"], q64.detach(), kp_ref, do, N, T)
    chk["dkv"] = (r, b_dkv, F32)                                     # b_dkv holds the bf16 rounding
    gs = vjp(kv_r, [Wk, Wv, Bv] + Xs, dkv)
    ref["wk"], ref["wv"], ref["bv"] = gs[:3]
    a, xa = dkv.double().abs(), s["xb"].double().abs()
    bound["wk"], bound["wv"] = TAU * (a[:, :d].t() @ xa), TAU * (a[:, d:].t() @ xa)
    bound["bv"] = TAU * a[:, d:].sum(0)
    mag = (TAU * (a[:, :d] @ Wk.abs() + a[:, d:] @ Wv.abs())).view(P, B, T, d)
    for p in range(P):
        e = torch.zeros(B, S, d, dtype=torch.float64, device=dev)      # the CLS row gets no gradient
        e[:, 1:] = mag[p]
        chk[f"f{p + 1}"] = (gs[3 + p], e, BF)                         # fp32 copies of the bf16 dX
    for k, prm in zip(CLASSIFY_GRADS, params):
        if prm is not None:
            chk[k] = (ref[k], bound[k].reshape(ref[k].shape), prm.dtype)
    return chk, got


# ----------------------------------------------------------------------------------------------------------------------
# VitHeadFn: mean over the patch rows -> fc_norm, or LayerNorm of the CLS row; then the head Linear
# ----------------------------------------------------------------------------------------------------------------------
VIT_GRADS = ("x", "nw", "nb", "w", "b")


def vit_head_ref(x, nw, nb, w, b, pool, eps, saved, a_dev, dlogits, log):
    """x fp32 [B, S, d]; saved: ``ctx.saved`` ((m, mean, rstd) pooled, (x,) CLS form) and a_dev ``ctx.a``, both taken
    before the backward; dlogits [B, n_cls]; log: the kernel calls of the backward.  Returns (checks, got)."""
    B, S, d = x.shape
    n_cls = w.shape[0]
    X, Nw, Nb, W, Bb = leaf(x), leaf(nw), leaf(nb), leaf(b64(w)), leaf(b)
    nw32, nb32 = _f32(nw), _f32(nb)
    chk, got = {}, {"a": a_dev}
    if pool:                                       # models_vit.py:431-432: x[:, 1:].mean(1), then fc_norm
        m, mean, rstd = saved
        f = head_fwd(x, nw32, nb32, eps)
        for k, v in (("m", m), ("mean", mean), ("rstd", rstd)):
            chk[k] = (f[k], f["b_" + k], F32)
            got[k] = v
        a_r = F.layer_norm(X[:, 1:].mean(1), (d,), Nw, Nb, eps)
        a_b = f["b_y"]                              # holds the bf16 rounding
    else:                                          # :434: encoder.layer_norm, then the CLS row
        a_r = F.layer_norm(X[:, 0], (d,), Nw, Nb, eps)
        a_b = layernorm_ref(x[:, 0], nw32, nb32, eps).err
    chk["a"] = (a_r.detach(), a_b, F32 if pool else BF)
    a = anchor(a_r, a_dev)
    l_r = F.linear(a, W, Bb)
    chk["logits"] = (l_r.detach(), TAU * _linear_mag(a_dev, W, Bb), F32)

    dl = kernel_calls(log, "colsum")[0][0][0]
    da = dx_of(log, dl)
    got.update(dl=dl, da=da)
    n_pad = dl.shape[1]
    chk["dl"] = (F.pad(dlogits.double(), (0, n_pad - n_cls)), torch.zeros(B, n_pad, dtype=torch.float64, device=x.device), BF)
    ref, bound = {}, {}
    dlc = dl[:, :n_cls]
    ref["w"], ref["b"], r = vjp(l_r, [W, Bb, a], dlc)
    g = dlc.double().abs()
    bound["w"], bound["b"] = TAU * (g.t() @ a_dev.double().abs()), TAU * g.sum(0)
    chk["da"] = (r, TAU * (g @ W.abs()), F32)                         # fp32 GEMM output
    if pool:       # the adjoint of LayerNorm(mean) at the kernel's own m, mean and rstd, as vit_ref bounds it
        hb = head_bwd(da, m, mean, rstd, nw32, S)
        ref["x"], ref["nw"], ref["nb"] = hb["dx"], hb["dgamma"], hb["dbeta"]
        bound["x"], bound["nw"], bound["nb"] = hb["b_dx"], hb["b_dgamma"], hb["b_dbeta"]
    else:
        ref["x"], ref["nw"], ref["nb"] = vjp(a_r, [X, Nw, Nb], da)
        ex, bound["nw"], bound["nb"] = ln_stage(x[:, 0], da, nw32, nb32, eps, False)
        bound["x"] = _zeros(X)
        bound["x"][:, 0] = ex
    for k, prm in zip(VIT_GRADS, (x, nw, nb, w, b)):
        chk[k] = (ref[k], bound[k].reshape(ref[k].shape), prm.dtype)
    return chk, got


# ----------------------------------------------------------------------------------------------------------------------
# ClassifyLossFn and RefcocoLossFn: the kernels' gradients, scaled by the upstream gradient in fp32
# ----------------------------------------------------------------------------------------------------------------------
def _criterion(z, mode, labels, targets, eps, num_choices):
    """The reference criteria in fp64 on the logits z [rows, C] (classify_loss.py, hinge_loss.py), summed over rows"""
    if mode == HARD:
        return F.cross_entropy(z, labels, label_smoothing=eps, reduction="sum")
    if mode == SOFT:
        return -(targets.double() * F.log_softmax(z, 1)).sum()
    if mode == MULTI:
        return F.binary_cross_entropy_with_logits(z, targets.double(), reduction="sum")
    zg = z[:, 0].view(-1, num_choices)
    assert mode == HINGE
    return (1 + zg - zg.gather(1, labels[:, None])).clamp_min(0).sum()


def classify_loss_ref(logits, mode, labels, targets, eps, num_choices, g):
    """logits [rows, C] as given (bf16 or fp32, any row pitch); g: the upstream gradient of the loss.  Returns checks
    for loss, n_correct, row_correct (``loss_ref``) and dlogits = g d loss / d logits."""
    C = logits.shape[1]
    r = loss_ref(logits.detach().float(), C, mode, labels=labels, targets=targets, eps=eps, num_choices=num_choices)
    Z = leaf(logits)
    (dz,) = vjp(_criterion(Z, mode, labels, targets, eps, num_choices), [Z], torch.ones((), dtype=torch.float64))
    gv = float(g)
    ref = gv * dz
    bd = r["b_dlogits"].reshape(dz.shape)
    return dict(loss=(r["loss"].reshape(1), r["b_loss"].reshape(1), F32),
                n_correct=(r["n_correct"].reshape(1), r["b_n_correct"].reshape(1), F32),
                row_correct=(r["row_correct"], r["b_row_correct"], F32),
                dlogits=(ref, abs(gv) * bd + U32 * ref.abs(), logits.dtype))


def refcoco_loss_ref(logits, targets, ns, g):
    """logits [B, 4] as given, targets [B, 4], ns; g: the upstream gradient of the loss.  Returns checks for loss, l1,
    n_valid (``refcoco``) and dlogits = g d loss / d logits."""
    r = refcoco(logits.detach().float(), targets, ns)
    assert not r["unsure"].any(), "a row's validity is within the fp32 error of its box"
    gv = float(g)
    ref = gv * r["dlogits"]
    dev = logits.device
    nv = torch.tensor([float(r["n_valid"])], dtype=torch.float64, device=dev)
    return dict(loss=(r["loss"].reshape(1), r["b_loss"].reshape(1), F32), l1=(r["l1"].reshape(1), r["b_l1"].reshape(1), F32),
                n_valid=(nv, torch.zeros_like(nv), F32),
                dlogits=(ref, abs(gv) * r["b_dlogits"] + U32 * ref.abs(), logits.dtype))


# ----------------------------------------------------------------------------------------------------------------------
# DclLossFn: masked student rows against every teacher row, label-smoothed InfoNCE, mean over the student rows
# ----------------------------------------------------------------------------------------------------------------------
def dcl_ref(student, teacher, stu_idx, tea_idx, scale, eps, g, fwd_log, log):
    """student / teacher [R, d] as given; stu_idx [n_m], tea_idx [n_t] (``dcl_indices``); g: the upstream gradient of the
    loss; fwd_log / log: the kernel calls of the forward (the Function computes the gradient there) and of the backward.
    Returns (checks, got) for the stages s_rows, t_rows, s_n, t_n, a3, b3, lse, loss, grad_n, dx32, gdx (= dx32 * g) and
    the student's gradient."""
    n_m, n_t = stu_idx.numel(), tea_idx.numel()
    d = student.shape[1]
    (_, _, s_rows), (_, _, t_rows) = kernel_calls(fwd_log, "row_gather")
    s_n, t_n = [r for _, _, r in kernel_calls(fwd_log, "l2_normalize_rows")]
    ((_, _, (a3, b3)),) = kernel_calls(fwd_log, "split_bf16x3")
    ((_, _, ((lse,), out)),) = kernel_calls(fwd_log, "infonce_forward")
    ((_, _, (grad_n, _)),) = kernel_calls(fwd_log, "infonce_grad")
    ((_, _, (_, dx32)),) = kernel_calls(fwd_log, "l2_normalize_bwd")
    ((sa, _, _),) = kernel_calls(log, "row_scatter_add")
    got = dict(s_rows=s_rows, t_rows=t_rows, s_n=s_n, t_n=t_n, a3=a3, b3=b3, lse=lse, loss=out[:1], grad_n=grad_n,
               dx32=dx32, gdx=sa[0])
    n8 = t_rows.shape[0]
    chk = {}
    St = leaf(student)
    s_rows_r = St[stu_idx]
    t_rows_r = F.pad(teacher.detach().double()[tea_idx], (0, 0, 0, n8 - n_t))        # zero rows past n_t
    chk["s_rows"] = (s_rows_r.detach(), _zeros(s_rows_r), F32)
    chk["t_rows"] = (t_rows_r, _zeros(t_rows_r), F32)
    Sr = anchor(s_rows_r, s_rows)
    sn_r = F.normalize(Sr, dim=1)
    chk["s_n"] = l2_normalize_ref(s_rows) + (F32,)
    chk["t_n"] = l2_normalize_ref(t_rows) + (F32,)
    for name, x, side in (("a3", s_n, 0), ("b3", t_n, 1)):           # hi = bf16(x), lo = bf16(x - hi): exact
        hi = x.to(BF)
        lo = (x - hi.float()).to(BF)
        v = torch.cat([hi, hi, lo] if side == 0 else [hi, lo, hi], 1).double()
        chk[name] = (v, _zeros(v), F32)
    Sn = anchor(sn_r, s_n)
    Tn = t_n.double()[:n_t]
    # compute_dcl_loss: log_softmax(scale s t^T), adjust_label_smoothed_nll_loss with targets 0..n_m-1, mean
    scale = float(scale)
    lp = F.log_softmax(scale * Sn @ Tn.t(), 1)
    eps_i = eps / (n_t - 1)
    rows = torch.arange(n_m, device=student.device)
    loss = ((1 - eps - eps_i) * -lp[rows, rows] + eps_i * -lp.sum(1)).mean()
    r = infonce_ref(s_n, t_n, scale, 0, eps, n_valid=n_t)
    chk["lse"] = (r.lse, r.dlse, F32)
    chk["loss"] = (loss.detach().reshape(1), ((r.dloss.sum() + 2.0 ** -16 * r.loss.abs().sum()) / n_m).reshape(1), F32)
    (r_g,) = vjp(loss, [Sn], torch.ones((), dtype=torch.float64))
    hi = b3[:n_t, :d].double()
    _, tol = infonce_grad_ref(r, b3[:, :d], scale, 1.0 / n_m)
    # the kernel contracts G with the bf16 hi part of the teacher rows, the reference with the rows
    chk["grad_n"] = (r_g, tol + scale / n_m * (r.G.abs() @ (Tn - hi).abs()), F32)
    (r_dx,) = vjp(sn_r, [Sr], grad_n)
    chk["dx32"] = (r_dx, l2_normalize_bwd_ref(s_rows, grad_n)[1], F32)
    gdx = dx32.double() * float(g)
    chk["gdx"] = (gdx, U32 * gdx.abs(), F32)
    (r_ds,) = vjp(s_rows_r, [St], sa[0])
    chk["student"] = (r_ds, scatter_ref(_zeros(student), stu_idx, sa[0])[1], student.dtype)
    return chk, got


# ----------------------------------------------------------------------------------------------------------------------
# RowGatherFn, ZeroPadFn, BlockBiasFn, LinearFn, FinalNormFn
# ----------------------------------------------------------------------------------------------------------------------
def row_gather_fn_ref(src, idx, fill, add, dout):
    """out[r] = src[idx[r]] (idx >= 0) else fill (or 0), + add[r % period] (one fp32 addition); the gradients of src
    (scatter-add), fill (sum over the fill rows) and add (sum over the periods) for the upstream dout.  Returns checks."""
    rows, dim = idx.numel(), src.shape[1]
    Src = leaf(src)
    ins, names = [Src], ["src"]
    keep = (idx >= 0)[:, None]
    base = torch.zeros(rows, dim, dtype=torch.float64, device=src.device)
    if fill is not None:
        Fl = leaf(fill)
        base = Fl.reshape(1, dim).expand(rows, dim)
        ins.append(Fl)
        names.append("fill")
    out = torch.where(keep, Src[idx.clamp_min(0)], base)
    if add is not None:
        Ad = leaf(add)
        period = Ad.numel() // dim
        out = out + Ad.reshape(period, dim)[torch.arange(rows, device=src.device) % period]
        ins.append(Ad)
        names.append("add")
    chk = {"out": (out.detach(), U32 * out.detach().abs() if add is not None else _zeros(out), F32)}
    D = dout.double()
    for nm, t, r in zip(names, ins, vjp(out, ins, D)):
        if nm == "src":
            e = scatter_ref(_zeros(t), idx, D)[1]
        elif nm == "fill":
            e = scatter_ref(torch.zeros(1, dim, dtype=torch.float64, device=D.device), torch.where(idx < 0, 0, -1), D)[1]
        else:
            e = scatter_ref(torch.zeros(period, dim, dtype=torch.float64, device=D.device),
                            torch.arange(rows, device=D.device) % period, D)[1]
        prm = {"src": src, "fill": fill, "add": add}[nm]
        chk[nm] = (r, e.reshape(r.shape), prm.dtype)
    return chk


def zero_pad_ref(x, pad_rows, dout):
    """x * (1 - padding_mask) (transformer_encoder.py:139-142) and its gradient: both exact"""
    keep = (pad_rows.reshape(-1, 1) == 0).double()
    out, dx = x.double() * keep, dout.double() * keep
    return dict(out=(out, _zeros(out), F32), x=(dx, _zeros(dx), F32))


def block_bias_ref(H, S, blocks, tables, dbias):
    """The bias canvas [Bb, H, S, S_pad]: zero, and each table's block table[bucket[p_i, p_j]] at rows and columns
    lo..lo+n of every canvas, p = ids[bb] (-1 -> n - 1, relpos_bias_block_ref) or 0..n-1 (a block shared by every
    sample).  Returns checks for the canvas (exact) and each table's gradient t0, t1, ... (fp32 scatter-adds)."""
    Bb = max([1] + [ids.shape[0] for _, ids, _, _ in blocks if ids is not None])
    s_pad = (S + 7) // 8 * 8
    Ts = [leaf(t) for t in tables]
    dev = tables[0].device
    canvas = torch.zeros(Bb, H, S, s_pad, dtype=torch.float64, device=dev)
    dests = []
    for Tb, (bucket, ids, n, lo) in zip(Ts, blocks):
        p = torch.arange(n, device=dev).expand(Bb, n) if ids is None else torch.where(ids < 0, n - 1, ids)
        dest = bucket[p[:, :, None], p[:, None, :]]                    # [Bb, n, n]
        blk = Tb[dest].permute(0, 3, 1, 2)
        canvas = canvas + F.pad(blk, (lo, s_pad - lo - n, lo, S - lo - n))
        dests.append((dest, n, lo))
    chk = {"bias": (canvas.detach(), _zeros(canvas), F32)}
    D = dbias.double()
    for i, (t, r, (dest, n, lo)) in enumerate(zip(tables, vjp(canvas, Ts, D), dests)):
        src = D[:, :, lo:lo + n, lo:lo + n].permute(0, 2, 3, 1).reshape(-1, H)
        chk[f"t{i}"] = (r, scatter_ref(_zeros(t), dest.reshape(-1), src)[1], t.dtype)
    return chk


def linear_fn_ref(x, w, b, saved, dy, log):
    """F.linear (components.py:29-35) on the bf16 copy of x the Function saved; saved: (xb, w, b); dy: the upstream
    gradient; log: the kernel calls of the backward.  Returns (checks, got)."""
    xb = saved[0]
    X, W = leaf(x), leaf(b64(w))
    ins, Bv = [X, W], None
    if b is not None:
        Bv = leaf(b)
        ins.append(Bv)
    xa = anchor(X, xb)
    y = F.linear(xa, W, Bv)
    ((_, _, dyb),) = kernel_calls(log, "row_gather")
    got = dict(xb=xb, dyb=dyb)
    chk = dict(xb=(X.detach(), _zeros(X), BF), y=(y.detach(), TAU * _linear_mag(xb, W, Bv), F32),
               dyb=(dy.double(), _zeros(dy), BF))
    gs = vjp(y, ins, dyb)
    a = dyb.double().abs()
    chk["x"] = (gs[0], TAU * (a @ W.abs()), x.dtype)                  # fp32 GEMM output
    chk["w"] = (gs[1], TAU * (a.t() @ xb.double().abs()), w.dtype)
    if b is not None:
        chk["b"] = (gs[2], TAU * a.sum(0), b.dtype)
    return chk, got


def final_norm_ref(x, w, b, eps, dy):
    """F.layer_norm over the rows (transformer_encoder.py:201-220), fp32 out, and its adjoint for the upstream dy"""
    X, Wl, Bl = leaf(x), leaf(w), leaf(b)
    y = F.layer_norm(X, (x.shape[1],), Wl, Bl, eps)
    dx, dw, db = vjp(y, [X, Wl, Bl], dy)
    ex, ew, eb = ln_stage(x, dy.float(), _f32(w), _f32(b), eps, False)
    return dict(out=(y.detach(), layernorm_ref(x, _f32(w), _f32(b), eps).err, F32), x=(dx, ex, x.dtype),
                w=(dw, ew, w.dtype), b=(db, eb, b.dtype))
