"""fp64 references of the embedding stems and the retrieval head of the training path (one_peace_b200/autograd.py:
``ImageEmbedFn``, ``AudioFeatFn``, ``AudioPosFn``, ``TextEmbedFn``, ``RelPosBiasFn``, ``HeadFn``), forward and adjoint, stage
by stage, with an error bound for every output element.

Plain PyTorch on whatever device the inputs live on; nothing here calls the extension.  The bounds are ``kernel_ref``'s
single-kernel bounds with its constants (TAU, U32, the LayerNorm bounds); nothing here adds a tolerance.

Reference
---------
fp64 torch autograd of the reference model's own operations (``oracle/restated.py``): ``F.conv2d`` on NCHW images,
``F.conv1d`` (strided, or grouped with ``padding = k // 2``), ``F.layer_norm``, ``F.gelu``, ``F.linear``, ``F.normalize``,
``F.embedding``.  It is not a restatement of the kernels' row layouts: device rows are mapped onto the reference's tensors
(``nchw_rows``, ``nchw_merged``, ``to_ct``) only to read what the device computed.  Weights are rounded to bf16 as the
Functions' packs round them.

Forward: the reference is anchored to the activations the Function saved for its backward, ``v = v_ref + (v_dev -
v_ref).detach()``, and each saved stage is checked against the reference operation applied to the device's previous
stage.  That checks the layout equivalence of each stage, for example a 2 x 2 pixel merge against a stride-2 ``conv2d``.

Adjoint: each stage of the device backward is checked on its own.  Its reference is the vjp of the stage's reference
operation, at the anchored forward point, of the cotangent the DEVICE handed to that stage: the bf16 intermediates
(dy3, da3, dy2, da2, dy1; dfb, dyP, dz_k, dy_k; dp_i, dc_i; dlog, dcls), read from the kernel calls the Function made
(``kernel_calls``).  A bound then never carries an error through more than one kernel, and it stays as tight at the real
widths as in a single-kernel test.  Chained through the stages, the checks still cover the whole adjoint: every output
is checked, and every stage's input is a checked output of the stage before.

Bounds, per element (|got - ref| <= bound + u_out |ref|; u_out = 2^-8 for a bf16 output):
  dW = dY^T X (GEMM over rows)   tau conv*_weight(|X|, |dY|), plus, where the kernel reads a bf16 copy of an fp32 forward
                                 operand X (the image, the waveform, the audio features), the exact |X - bf16(X)|^T |dY|
  dX = dY W                      tau conv*_input(|W|, |dY|); a col2im (window_scatter) of per-tap bf16 products adds
                                 (2^-8 + kw u) conv*_input(|W|, |dY|) and tau 2^-8 of the same
  LayerNorm (+ GELU) backward    ``layernorm_bwd_ref`` on the device's x and dy
  bf16 copies of fp32 values     u_out only;  column sums ``colsum_ref`` / (tau + 2u) sum |v| over fp32 values;
  batch sums, scatter-adds       (count + 1) u (|init| + sum |terms|) (``scatter_ref``)
Where the reference is exactly zero (a padding token's embedding row, an unused vocabulary row or relative-position
bucket, the head's dx past the CLS row, padded rows) the bound is zero, so the device value must be exactly zero.
"""
import torch
import torch.nn.functional as F
from torch.nn.grad import conv1d_input, conv1d_weight, conv2d_input, conv2d_weight

from kernel_ref import (TAU, U32, l2_normalize_bwd_ref, l2_normalize_ref, layernorm_bwd_ref, layernorm_ref,
                        scatter_ref)

BF, F32 = torch.bfloat16, torch.float32
R8 = 2.0 ** -8          # bf16 round-to-nearest, the u_out of kernel_ref


def b64(t):
    """the bf16 rounding of t as the packs make it, in fp64"""
    return t.detach().to(BF).double()


def anchor(ref, dev):
    """ref with the value of the device's saved activation and the gradient of the reference graph"""
    return ref + (dev.double() - ref).detach()


def leaf(t):
    return t.detach().double().requires_grad_()


def vjp(out, inputs, cot):
    gs = torch.autograd.grad(out, inputs, cot.double(), retain_graph=True, allow_unused=True)
    return [(g if g is not None else torch.zeros_like(i)).detach() for g, i in zip(gs, inputs)]


def nchw_rows(t, B, g):
    """device rows (b, y, x) x C -> [B, C, g, g]"""
    return t.reshape(B, g, g, -1).permute(0, 3, 1, 2)


def rows_nchw(t):
    """[B, C, g, g] -> rows (b, y, x) x C"""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def nchw_merged(t, B, go):
    """2 x 2 merged rows (b, Y, X) x (ky, kx, c) on a go x go grid -> [B, C, 2 go, 2 go]"""
    C = t.shape[1] // 4
    return t.reshape(B, go, go, 2, 2, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, 2 * go, 2 * go)


def to_ct(t, B):
    """device rows (b, t) x C -> [B, C, T]"""
    return t.reshape(B, -1, t.shape[-1]).transpose(1, 2)


def ct_rows(t):
    """[B, C, T] -> rows (b, t) x C"""
    return t.transpose(1, 2).reshape(-1, t.shape[1])


def kernel_calls(log, name):
    """(args, kwargs, result) of each call of kernel ``name`` in a recorded log of (name, args, kwargs, result)"""
    return [(a, kw, r) for n, a, kw, r in log if n == name]


def ln_bwd_of(log, x):
    """(dy, dx, kwargs) of the layernorm_bwd call that read the forward rows x (matched by address)"""
    hits = [(a[1], r, kw) for a, kw, r in kernel_calls(log, "layernorm_bwd") if a[0].data_ptr() == x.data_ptr()]
    assert len(hits) == 1, f"{len(hits)} layernorm_bwd calls read these rows"
    return hits[0]


def ln_stage(x_rows, dy_rows, gamma, beta, eps, gelu):
    """bounds of a LayerNorm backward on the device's own operands: (dx, dgamma, dbeta)"""
    r = layernorm_bwd_ref(x_rows, dy_rows, gamma, beta, eps, gelu=gelu)
    return r.dx_err, r.dgamma_err, r.dbeta_err


def _lngelu(y, lw, lb, eps):
    """LayerNorm over the channel dimension of [B, C, ...] followed by GELU, as the reference's LayerNorm2D / conv stacks"""
    t = y.movedim(1, -1)
    return F.gelu(F.layer_norm(t, (t.shape[-1],), lw, lb, eps)).movedim(-1, 1)


def _f32(t):
    return t.detach().float() if t is not None else None


# ----------------------------------------------------------------------------------------------------------------------
# ImageEmbedFn: hMLP stem (conv 4x4/4, LN+GELU, conv 2x2/2, LN+GELU, conv 2x2/2), CLS row, positions
# ----------------------------------------------------------------------------------------------------------------------
IMAGE_GRADS = ("pos", "w1", "b1", "ln1w", "ln1b", "w2", "b2", "ln2w", "ln2b", "w3", "b3", "cls")


def image_embed_ref(img, params, saved, dx, log, eps=1e-5):
    """img [B, 3, R, R] as given; params: the 12 tensors after img in ImageEmbedFn.apply's order; saved: its saved
    tensors (im, ln1w, ln1b, ln2w, ln2b, w1, w2, w3, y1, a2, y2, a3); dx: the upstream gradient [B, S, d]; log: the kernel
    calls of its backward.

    Returns (checks, got): checks[name] = (reference, bound, out dtype) for the forward stages (y1, a2, y2, a3, x), the
    backward intermediates (dy3, da3, dy2, da2, dy1) and the gradients of IMAGE_GRADS; got[name] = what the device made
    for the intermediates and forward stages, in the reference's layout."""
    pos, w1, b1, ln1w, ln1b, w2, b2, ln2w, ln2b, w3, b3, cls = params
    y1d, a2d, y2d, a3d = saved[8:12]
    B, _, R, _ = img.shape
    g1, g2, w = R // 4, R // 8, R // 16
    d = w3.shape[0]
    a1 = b64(img)                                                       # the operand patchify4 gives the GEMM
    P = [leaf(pos), leaf(b64(w1)), leaf(b1), leaf(ln1w), leaf(ln1b), leaf(b64(w2)), leaf(b2), leaf(ln2w), leaf(ln2b),
         leaf(b64(w3)), leaf(b3), leaf(cls)]
    Pos, W1, B1, L1w, L1b, W2, B2, L2w, L2b, W3, B3, Cls = P
    y1n, a2n, y2n, a3n = nchw_rows(y1d, B, g1), nchw_merged(a2d, B, g2), nchw_rows(y2d, B, g2), nchw_merged(a3d, B, w)
    chk, got = {}, dict(y1=y1n, a2=a2n, y2=y2n, a3=a3n)

    y1_r = F.conv2d(img.double(), W1, B1, stride=4)
    y1 = anchor(y1_r, y1n)
    a2_r = _lngelu(y1, L1w, L1b, eps)
    a2 = anchor(a2_r, a2n)
    y2_r = F.conv2d(a2, W2, B2, stride=2)
    y2 = anchor(y2_r, y2n)
    a3_r = _lngelu(y2, L2w, L2b, eps)
    a3 = anchor(a3_r, a3n)
    y3 = F.conv2d(a3, W3, B3, stride=2).flatten(2).transpose(1, 2)
    x = torch.cat([Cls.reshape(1, 1, d).expand(B, 1, d), y3], 1) + Pos[None]
    with torch.no_grad():
        cb = lambda bb: bb.abs()[:, None, None]
        chk["y1"] = (F.conv2d(a1, W1, B1, stride=4), TAU * (F.conv2d(a1.abs(), W1.abs(), stride=4) + cb(B1)), BF)
        e = layernorm_ref(rows_nchw(y1n), _f32(ln1w), _f32(ln1b), eps, gelu=True).err
        chk["a2"] = (a2_r.detach(), nchw_rows(e, B, g1), BF)
        chk["y2"] = (y2_r.detach(), TAU * (F.conv2d(a2n.double().abs(), W2.abs(), stride=2) + cb(B2)), BF)
        e = layernorm_ref(rows_nchw(y2n), _f32(ln2w), _f32(ln2b), eps, gelu=True).err
        chk["a3"] = (a3_r.detach(), nchw_rows(e, B, g2), BF)
        m3 = (F.conv2d(a3n.double().abs(), W3.abs(), stride=2) + cb(B3)).flatten(2).transpose(1, 2)
        mag = torch.cat([Cls.abs().reshape(1, 1, d).expand(B, 1, d), m3], 1) + Pos.abs()[None]
        chk["x"] = (x.detach(), TAU * mag, F32)

    # device intermediates of the backward
    (dy3,) = [r for _, kw, r in kernel_calls(log, "scale_resid_bwd")]
    da3, dy2, _ = ln_bwd_of(log, y2d)
    da2, dy1, _ = ln_bwd_of(log, y1d)
    dy3n, da3n, dy2n, da2n, dy1n = (dy3.reshape(B, w * w, d), nchw_merged(da3, B, w), nchw_rows(dy2, B, g2),
                                    nchw_merged(da2, B, g2), nchw_rows(dy1, B, g1))
    got.update(dy3=dy3n, da3=da3n, dy2=dy2n, da2=da2n, dy1=dy1n)
    D = dx.double()
    ref = dict(zip(("pos", "cls", "b3"), vjp(x, [Pos, Cls, B3], D)))
    bound = {"pos": (B + 1) * U32 * D.abs().sum(0), "cls": (B + 1) * U32 * D[:, 0].abs().sum(0),
             "b3": (TAU + 2 * U32) * D[:, 1:].abs().sum((0, 1))}
    chk["dy3"] = (D[:, 1:], torch.zeros_like(D[:, 1:]), BF)
    # conv3: dW3, da3 from dy3
    ref["w3"], r_da3 = vjp(y3, [W3, a3], dy3n)
    g = dy3n.double().abs().transpose(1, 2).reshape(B, d, w, w)
    bound["w3"] = TAU * conv2d_weight(a3n.double().abs(), W3.shape, g, stride=2)
    chk["da3"] = (r_da3, TAU * conv2d_input(a3.shape, W3.abs(), g, stride=2), BF)
    # LN2 + GELU: dy2, dln2 from da3
    r_dy2, ref["ln2w"], ref["ln2b"] = vjp(a3_r, [y2, L2w, L2b], da3n)
    ex, bound["ln2w"], bound["ln2b"] = ln_stage(rows_nchw(y2n), rows_nchw(da3n), _f32(ln2w), _f32(ln2b), eps,
                                                True)
    chk["dy2"] = (r_dy2, nchw_rows(ex, B, g2), BF)
    # conv2: dW2, db2, da2 from dy2
    r_da2, ref["w2"], ref["b2"] = vjp(y2_r, [a2, W2, B2], dy2n)
    g = dy2n.double().abs()
    bound["w2"] = TAU * conv2d_weight(a2n.double().abs(), W2.shape, g, stride=2)
    bound["b2"] = TAU * g.sum((0, 2, 3))
    chk["da2"] = (r_da2, TAU * conv2d_input(a2.shape, W2.abs(), g, stride=2), BF)
    # LN1 + GELU: dy1, dln1 from da2
    r_dy1, ref["ln1w"], ref["ln1b"] = vjp(a2_r, [y1, L1w, L1b], da2n)
    ex, bound["ln1w"], bound["ln1b"] = ln_stage(rows_nchw(y1n), rows_nchw(da2n), _f32(ln1w), _f32(ln1b), eps, True)
    chk["dy1"] = (r_dy1, nchw_rows(ex, B, g1), BF)
    # conv1: dW1, db1 from dy1 (the GEMM reads bf16(img), the reference img)
    ref["w1"], ref["b1"] = vjp(y1_r, [W1, B1], dy1n)
    g = dy1n.double().abs()
    bound["w1"] = (TAU * conv2d_weight(a1.abs(), W1.shape, g, stride=4)
                   + conv2d_weight((img.double() - a1).abs(), W1.shape, g, stride=4))
    bound["b1"] = TAU * g.sum((0, 2, 3))
    for k, p in zip(IMAGE_GRADS, params):
        chk[k] = (ref[k], bound[k].reshape(ref[k].shape), p.dtype)
    return chk, got


# ----------------------------------------------------------------------------------------------------------------------
# HeadFn: CLS row -> LayerNorm -> Linear (fp32) -> l2-normalize
# ----------------------------------------------------------------------------------------------------------------------
HEAD_GRADS = ("x", "ln_w", "ln_b", "w", "b")


def head_ref(x, ln_w, ln_b, w, b, eps, saved, dy, log):
    """x [B, S, d] fp32; saved: HeadFn's saved tensors (x, ln_w, ln_b, w, b, cls, logits); dy [B, n]; log: the kernel calls
    of its backward.  Returns (checks, got) as ``image_embed_ref`` does."""
    cls_d, log_d = saved[5], saved[6]
    X, Lw, Lb, W, Bb = leaf(x), leaf(ln_w), leaf(ln_b), leaf(b64(w)), leaf(b)
    c_r = F.layer_norm(X[:, 0], (X.shape[2],), Lw, Lb, eps)
    c = anchor(c_r, cls_d)
    l_r = F.linear(c, W, Bb)
    lg = anchor(l_r, log_d)
    y = F.normalize(lg, dim=1)
    chk = {}
    with torch.no_grad():
        chk["cls"] = (c_r.detach(), layernorm_ref(x[:, 0], _f32(ln_w), _f32(ln_b), eps).err, BF)
        chk["logits"] = (l_r.detach(), TAU * (cls_d.double().abs() @ W.abs().t() + Bb.abs()), F32)
        chk["y"] = (y.detach(), l2_normalize_ref(log_d)[1], F32)
    (dlog,) = [r for _, _, r in kernel_calls(log, "l2_normalize_bwd")]
    dcls, _, _ = ln_bwd_of(log, x)
    got = dict(cls=cls_d, logits=log_d, dlog=dlog, dcls=dcls)
    (r,) = vjp(y, [lg], dy)
    chk["dlog"] = (r, l2_normalize_bwd_ref(log_d, dy.float())[1], BF)
    ref, bound = {}, {}
    ref["w"], ref["b"], r = vjp(l_r, [W, Bb, c], dlog)
    g = dlog.double().abs()
    bound["w"], bound["b"] = TAU * (g.t() @ cls_d.double().abs()), TAU * g.sum(0)
    chk["dcls"] = (r, TAU * (g @ W.abs()), BF)
    ref["x"], ref["ln_w"], ref["ln_b"] = vjp(c_r, [X, Lw, Lb], dcls)
    ex, bound["ln_w"], bound["ln_b"] = ln_stage(x[:, 0], dcls, _f32(ln_w), _f32(ln_b), eps, False)
    bound["x"] = torch.zeros_like(X)
    bound["x"][:, 0] = ex
    for k, p in zip(HEAD_GRADS, (x, ln_w, ln_b, w, b)):
        chk[k] = (ref[k], bound[k], p.dtype)
    return chk, got


# ----------------------------------------------------------------------------------------------------------------------
# TextEmbedFn and RelPosBiasFn
# ----------------------------------------------------------------------------------------------------------------------
def text_embed_fn_ref(tokens, table, pos, cls, pad_idx, dx):
    """The reference model's (cat(cls, embedding(tokens)) + pos) with padded rows zeroed, in fp64: the forward (one fp32
    addition of fp32 operands per element: u |x|) and the gradients of table, pos, cls (fp32 scatter-adds).
    Returns (checks, pad mask)."""
    B, T = tokens.shape
    pad = torch.cat([torch.zeros(B, 1, dtype=torch.bool, device=tokens.device), tokens == pad_idx], 1)
    Tb, Pp, Cc = leaf(table if table.dtype in (F32, BF) else table.float()), leaf(pos.float()), leaf(cls.float())
    d = Tb.shape[1]
    emb = F.embedding(tokens, Tb, padding_idx=pad_idx)
    x = (torch.cat([Cc.reshape(1, 1, d).expand(B, 1, d), emb], 1) + Pp[:T + 1][None]) * (~pad)[..., None].double()
    gt, gp, gc = vjp(x, [Tb, Pp, Cc], dx)
    D = dx.double() * (~pad)[..., None].double()
    tok = torch.where(tokens == pad_idx, torch.full_like(tokens, -1), tokens)
    _, et = scatter_ref(torch.zeros_like(gt), tok.reshape(-1), D[:, 1:].reshape(B * T, d))
    pidx = torch.arange(T + 1, device=dx.device).expand(B, T + 1)
    _, ep = scatter_ref(torch.zeros_like(gp), torch.where(pad, -1, pidx).reshape(-1), D.reshape(-1, d))
    ec = (B + 1) * U32 * D[:, 0].abs().sum(0)
    chk = dict(x=(x.detach(), U32 * x.detach().abs(), F32), table=(gt, et, table.dtype), pos=(gp, ep, pos.dtype),
               cls=(gc, ec.reshape(gc.shape), cls.dtype))
    return chk, pad.to(torch.uint8)


def relpos_fn_ref(table, bucket, S, dbias):
    """table[bucket[:S, :S]].permute(2, 0, 1) with zero padding columns up to S_pad (exact), and the table gradient for
    the upstream dbias [H, S, S_pad] (its padding columns carry none)"""
    Tb = leaf(table)
    H = table.shape[1]
    b = F.pad(Tb[bucket[:S, :S]].permute(2, 0, 1), (0, (S + 7) // 8 * 8 - S))
    (gt,) = vjp(b, [Tb], dbias)
    # every (h, i, j) adds one term to row bucket[i, j], column h
    src = dbias[..., :S].double().permute(1, 2, 0).reshape(S * S, H)
    _, e = scatter_ref(torch.zeros_like(gt), bucket[:S, :S].reshape(-1), src)
    return dict(bias=(b.detach(), torch.zeros_like(b.detach()), F32), table=(gt, e, table.dtype))


# ----------------------------------------------------------------------------------------------------------------------
# AudioPosFn: grouped conv positional encoder (k = 19, 16 groups, 5 layers), residual, CLS, padded rows zeroed
# ----------------------------------------------------------------------------------------------------------------------
def audio_pos_ref(feats, pad, meta, params, saved, dxs, dfeats, log, eps=1e-5):
    """feats fp32 [B*T, d]; pad bool [B, T+1]; meta (B, T, k, groups, d); params: the Function's tensors after meta (pos
    conv weights, pos conv biases, cls_embedding, cls_pos_embed); saved: ``ctx.saved``; dxs [B, T+1, d] the upstream
    gradient; dfeats the device's gradient of feats; log: the kernel calls of its backward.  Returns (checks, got); the
    gradients are named feats, w0.., b0.., cls, cls_pos."""
    B, T, k, G, d = meta
    n = (len(params) - 2) // 2
    p_ins, cs = saved["p_ins"], saved["cs"]
    Fe = leaf(feats)
    Ws = [leaf(b64(params[i])) for i in range(n)]
    Bs = [leaf(params[n + i]) for i in range(n)]
    Cl, Cp = leaf(params[-2]), leaf(params[-1])
    keep = (~pad.bool())[..., None].double()
    conv = lambda x, i: F.conv1d(x, Ws[i], Bs[i], padding=k // 2, groups=G)
    chk, got = {}, {}
    got["p_in0"] = p_ins[0]
    chk["p_in0"] = (feats.double(), torch.zeros(feats.shape, dtype=torch.float64, device=feats.device), BF)
    pin = to_ct(Fe, B)
    pins, c_rs, outs = [], [], []
    for i in range(n):
        if i > 0:
            got[f"p_in{i}"] = to_ct(p_ins[i], B)
            chk[f"p_in{i}"] = (pin.detach(), to_ct(layernorm_ref(cs[i - 1], None, None, eps, gelu=True).err, B), BF)
            pin = anchor(pin, to_ct(p_ins[i], B))
        xin = to_ct(p_ins[i], B).double()
        with torch.no_grad():
            mag = F.conv1d(xin.abs(), Ws[i].abs(), padding=k // 2, groups=G) + Bs[i].abs()[:, None]
            chk[f"c{i}"] = (conv(xin, i), TAU * mag, BF)
        got[f"c{i}"] = to_ct(cs[i], B)
        c_r = conv(pin, i)
        pins.append(pin)
        c_rs.append(c_r)
        pin = _lngelu(anchor(c_r, to_ct(cs[i], B)), None, None, eps)
        outs.append(pin)
    posb = pin.transpose(1, 2)
    body = Fe.reshape(B, T, d) + posb
    x = torch.cat([(Cl + Cp).reshape(1, 1, d).expand(B, 1, d), body], 1) * keep
    with torch.no_grad():
        e5 = layernorm_ref(cs[-1], None, None, eps, gelu=True).err.reshape(B, T, d)
        eb = e5 + R8 * (posb.abs() + e5) + U32 * body.abs()
        ec = U32 * (Cl + Cp).abs().reshape(1, 1, d).expand(B, 1, d)
        chk["x"] = (x.detach(), torch.cat([ec, eb], 1) * keep, F32)

    ref, bound = {}, {}
    D = dxs.double() * keep
    ref["cls"], ref["cls_pos"], r_dp = vjp(x, [Cl, Cp, posb], dxs)
    bound["cls"] = bound["cls_pos"] = ((B + 1) * U32 * D[:, 0].abs().sum(0)).reshape(ref["cls"].shape)
    direct = D[:, 1:].reshape(B * T, d)
    dps = [ln_bwd_of(log, cs[i]) for i in range(n)]                      # (dp_i, dc_i) per layer
    r_dp = r_dp.transpose(1, 2)                                           # [B, d, T]
    e_dp = torch.zeros_like(r_dp)                                         # dp of the last layer: bf16(dxs rows) alone
    for i in reversed(range(n)):
        dp, dc, _ = dps[i]
        got[f"dp{i}"], got[f"dc{i}"] = to_ct(dp, B), to_ct(dc, B)
        chk[f"dp{i}"] = (r_dp, e_dp, BF)
        (r_dc,) = vjp(outs[i], [c_rs[i]], to_ct(dp, B))
        chk[f"dc{i}"] = (r_dc, to_ct(ln_stage(cs[i], dp, None, None, eps, True)[0], B), BF)
        r_dp, ref[f"w{i}"], ref[f"b{i}"] = vjp(c_rs[i], [pins[i], Ws[i], Bs[i]], to_ct(dc, B))
        g = to_ct(dc, B).double().abs()
        xin = to_ct(p_ins[i], B).double()
        bound[f"w{i}"] = TAU * conv1d_weight(xin.abs(), Ws[i].shape, g, padding=k // 2, groups=G)
        if i == 0:                                  # the GEMM reads bf16(feats), the reference feats
            bound["w0"] = bound["w0"] + conv1d_weight((to_ct(feats, B).double() - xin).abs(), Ws[0].shape, g,
                                                      padding=k // 2, groups=G)
        bound[f"b{i}"] = TAU * g.sum((0, 2))
        mag = conv1d_input(xin.shape, Ws[i].abs(), g, padding=k // 2, groups=G)
        e_dp = (TAU * (1 + R8) + R8 + k * U32) * mag                        # per-tap bf16 products, col2im, bf16
    # dfeats = direct term + the positional branch's bf16 dp (one fp32 addition)
    r_df = direct + ct_rows(r_dp)
    e_df = ct_rows(e_dp + R8 * (r_dp.abs() + e_dp)) + U32 * r_df.abs()
    ref["feats"], bound["feats"] = r_df, e_df
    got["feats"] = dfeats
    names = ["feats"] + [f"w{i}" for i in range(n)] + [f"b{i}" for i in range(n)] + ["cls", "cls_pos"]
    dts = [F32] + [p.dtype for p in params]
    for nm, dt in zip(names, dts):
        chk[nm] = (ref[nm], bound[nm].reshape(ref[nm].shape), dt)
    return chk, got


# ----------------------------------------------------------------------------------------------------------------------
# AudioFeatFn: wav2vec feature extractor (7 strided convs, LN + GELU), post LayerNorm, Linear
# ----------------------------------------------------------------------------------------------------------------------
def audio_feat_ref(wav, spec, d, params, saved, feats_dev, log, eps=1e-5):
    """wav [B, N] as given; spec ((C, k, s), ...); params: the Function's tensors after (wav, meta); saved: ``ctx.saved``
    (a0, wk, ys, zs, yP); feats_dev: its output; log: the kernel calls of its backward.  Returns (checks, got); the
    gradients are named conv0.., lnw0.., lnb0.., post_w, post_b, proj_w, proj_b."""
    n = len(spec)
    B = wav.shape[0]
    C = spec[0][0]
    ys, zs, yP = saved["ys"], saved["zs"], saved["yP"]
    Ws = [leaf(b64(params[i])) for i in range(n)]
    Lw = [leaf(params[n + i]) for i in range(n)]
    Lb = [leaf(params[2 * n + i]) for i in range(n)]
    Pw, Pb, Jw, Jb = leaf(params[3 * n]), leaf(params[3 * n + 1]), leaf(b64(params[3 * n + 2])), leaf(params[3 * n + 3])
    wav64, a1 = wav.double(), b64(wav)
    chk, got = {}, {}
    k0, s0 = spec[0][1], spec[0][2]
    win = a1.unfold(1, k0, s0)                                           # [B, T0, k0]: the first conv's windows
    got["a0"] = saved["a0"].reshape(B, -1, 16)
    chk["a0"] = (F.pad(win, (0, 16 - k0)), torch.zeros(win.shape[:2] + (16,), dtype=torch.float64, device=wav.device), BF)
    y_r, zr, z_in = [], [], [wav64[:, None]]
    z = wav64[:, None]
    for i, (_, kk, st) in enumerate(spec):
        xin = a1[:, None] if i == 0 else to_ct(zs[i - 1], B).double()
        with torch.no_grad():
            chk[f"y{i}"] = (F.conv1d(xin, Ws[i], stride=st), TAU * F.conv1d(xin.abs(), Ws[i].abs(), stride=st), BF)
        got[f"y{i}"] = to_ct(ys[i], B)
        yr = F.conv1d(z, Ws[i], stride=st)
        y_r.append(yr)
        zi = _lngelu(anchor(yr, to_ct(ys[i], B)), Lw[i], Lb[i], eps)
        zr.append(zi)
        with torch.no_grad():
            chk[f"z{i}"] = (zi.detach(), to_ct(layernorm_ref(ys[i], _f32(params[n + i]), _f32(params[2 * n + i]), eps,
                                                             gelu=True).err, B), BF)
        got[f"z{i}"] = to_ct(zs[i], B)
        z = anchor(zi, to_ct(zs[i], B))
        z_in.append(z)
    zl = z.transpose(1, 2)                                               # [B, T, C]
    yP_r = F.layer_norm(zl, (C,), Pw, Pb, eps)
    yPa = anchor(yP_r, yP.reshape(B, -1, C))
    f_r = F.linear(yPa, Jw, Jb)
    with torch.no_grad():
        chk["yP"] = (yP_r.detach(), layernorm_ref(zs[-1], _f32(params[3 * n]), _f32(params[3 * n + 1]), eps).err
                     .reshape(yP_r.shape), BF)
        chk["feats_fwd"] = (f_r.detach(), TAU * (yP.double().abs() @ Jw.abs().t() + Jb.abs()).reshape(f_r.shape), F32)
    got["yP"], got["feats_fwd"] = yP.reshape(B, -1, C), feats_dev.reshape(f_r.shape)

    ((a, kw, dfb),) = [c for c in kernel_calls(log, "scale_resid_bwd") if c[1].get("dbias") is not None]
    dfeats = a[0].reshape(f_r.shape)
    T = dfeats.shape[1]
    ref, bound = {}, {}
    (ref["proj_b"],) = vjp(f_r, [Jb], dfeats)
    bound["proj_b"] = (TAU + 2 * U32) * dfeats.double().abs().sum((0, 1))
    got["dfb"] = dfb.reshape(f_r.shape)
    chk["dfb"] = (dfeats.double(), torch.zeros(f_r.shape, dtype=torch.float64, device=wav.device), BF)
    g = dfb.double().abs().reshape(B * T, d)
    ref["proj_w"], r_dyP = vjp(f_r, [Jw, yPa], dfb.reshape(f_r.shape))
    bound["proj_w"] = TAU * (g.t() @ yP.double().abs())
    dyP, dz, _ = ln_bwd_of(log, zs[-1])
    got["dyP"] = dyP.reshape(B, T, C)
    chk["dyP"] = (r_dyP, TAU * (g @ Jw.abs()).reshape(B, T, C), BF)
    r_dz, ref["post_w"], ref["post_b"] = vjp(yP_r, [zl, Pw, Pb], dyP.reshape(B, T, C))
    ex, bound["post_w"], bound["post_b"] = ln_stage(zs[-1], dyP, _f32(params[3 * n]), _f32(params[3 * n + 1]), eps, False)
    r_dz, e_dz = r_dz.transpose(1, 2), to_ct(ex, B)
    for i in reversed(range(n)):
        kk, st = spec[i][1], spec[i][2]
        dzi, dy, _ = ln_bwd_of(log, ys[i])
        got[f"dz{i}"], got[f"dy{i}"] = to_ct(dzi, B), to_ct(dy, B)
        chk[f"dz{i}"] = (r_dz, e_dz, BF)
        r_dy, ref[f"lnw{i}"], ref[f"lnb{i}"] = vjp(zr[i], [y_r[i], Lw[i], Lb[i]], to_ct(dzi, B))
        ex, bound[f"lnw{i}"], bound[f"lnb{i}"] = ln_stage(ys[i], dzi, _f32(params[n + i]), _f32(params[2 * n + i]), eps,
                                                          True)
        chk[f"dy{i}"] = (r_dy, to_ct(ex, B), BF)
        g = to_ct(dy, B).double().abs()
        if i == 0:                                   # the GEMM reads bf16(wav), the reference wav
            (ref["conv0"],) = vjp(y_r[0], [Ws[0]], to_ct(dy, B))
            bound["conv0"] = (TAU * conv1d_weight(a1.abs()[:, None], Ws[0].shape, g, stride=st)
                              + conv1d_weight((wav64 - a1).abs()[:, None], Ws[0].shape, g, stride=st))
        else:
            xin = to_ct(zs[i - 1], B).double()
            ref[f"conv{i}"], r_dz = vjp(y_r[i], [Ws[i], z_in[i]], to_ct(dy, B))
            bound[f"conv{i}"] = TAU * conv1d_weight(xin.abs(), Ws[i].shape, g, stride=st)
            e_dz = (TAU * (1 + R8) + R8 + kk * U32) * conv1d_input(xin.shape, Ws[i].abs(), g, stride=st)
    names = ([f"conv{i}" for i in range(n)] + [f"lnw{i}" for i in range(n)] + [f"lnb{i}" for i in range(n)]
             + ["post_w", "post_b", "proj_w", "proj_b"])
    for nm, p in zip(names, params):
        chk[nm] = (ref[nm], bound[nm].reshape(ref[nm].shape), p.dtype)
    return chk, got


# ----------------------------------------------------------------------------------------------------------------------
# comparison
# ----------------------------------------------------------------------------------------------------------------------
def share(got, ref, bound, out_dtype):
    """largest |got - ref| / (bound + u_out |ref|) over the elements (kernel_ref.assert_within's ratio; 0 / 0 = 0, and a
    nonzero error against a zero bound, a NaN or an Inf is infinite)"""
    g, r = got.detach().double().reshape(ref.shape), ref.double()
    tol = bound + (R8 if out_dtype == BF else 0.0) * r.abs()
    err = (g - r).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / tol)
    ratio = torch.nan_to_num(ratio, nan=float("inf"), posinf=float("inf"))
    return ratio.max().item() if ratio.numel() else 0.0


def shares(got, checks):
    """{name: share} for got[name] against checks[name] = (ref, bound, out dtype)"""
    return {k: share(got[k], *checks[k]) for k in checks}
