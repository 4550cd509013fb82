"""Training path of the classification head (models/one_peace/one_peace_base.py:132-235, OnePeaceClassifyHead with attention
pooling) and of the classification and grounding criteria (criterions/classify_loss.py, criterions/hinge_loss.py,
criterions/refcoco_loss.py), as
``torch.autograd.Function`` nodes whose forward and backward are sm_90a kernels:

    per-token features [B, S, d] (after the modality's final LayerNorm; CLS row dropped)
      -> k | v = one GEMM against [Wk; Wv] with bias [0; bv]        -> opb_attn_pool_fwd (csrc/classify.cu)
      -> out_proj (GEMM)  -> classify_head.norm (LayerNorm)          -> pooler tanh(Linear) when use_pooler
      -> [pass 1 | pass 2] when use_two_images
      -> Linear -> LayerNorm + GELU (one kernel) -> Linear           -> logits [B, num_classes]

The classifier's output rows are zero-padded to a multiple of 8 (the GEMM wants N % 8 == 0); the logits are a view of the
first num_classes columns.  The two passes of use_two_images run as one batch of 2B rows through pooling, out_proj, norm and
pooler, so their parameter gradients are summed inside the dW GEMMs.  torch is used for allocation, dtype / layout copies
and the pooler's tanh and its derivative on the [B, d] fp32 tensor.
"""
import torch

from . import kernels as K
from .autograd import _dw, _dx, _pad8
from .components import bf16, f32


def head_params(head):
    """The head's parameters in the order ClassifyHeadFn takes them (pooler entries are None without use_pooler)."""
    ap = head.attn_pooling_func
    pool = head.pooler[1] if head.pooler is not None else None
    c = head.classifier
    return [head.norm.weight, head.norm.bias, ap.q, ap.k_proj.weight, ap.v_proj.weight, ap.v_proj.bias, ap.out_proj.weight,
            ap.out_proj.bias, pool.weight if pool is not None else None, pool.bias if pool is not None else None,
            c[0].weight, c[0].bias, c[1].weight, c[1].bias, c[3].weight, c[3].bias]


def head_pack(head, cache):
    """bf16 / fp32 kernel operands of the head, rebuilt after each optimizer step."""
    ps = head_params(head)

    def build():
        nw, nb, q, wk, wv, bv, wo, bo, wp, bp, w0, b0, g1, be1, w3, b3 = ps
        d = wk.shape[0]
        n_cls = w3.shape[0]
        n_pad = _pad8(n_cls)
        w3p = torch.zeros(n_pad, w3.shape[1], dtype=torch.bfloat16, device=w3.device)
        w3p[:n_cls].copy_(w3.detach())
        b3p = torch.zeros(n_pad, dtype=torch.float32, device=w3.device)
        b3p[:n_cls].copy_(b3.detach())
        return dict(norm_w=f32(nw), norm_b=f32(nb), q=f32(q).view(-1, 64), wkv=torch.cat([bf16(wk), bf16(wv)], 0).contiguous(),
                    bkv=torch.cat([torch.zeros(d, device=wk.device), f32(bv)]).contiguous(), wo=bf16(wo), bo=f32(bo),
                    wp=bf16(wp) if wp is not None else None, bp=f32(bp) if bp is not None else None, w0=bf16(w0), b0=f32(b0),
                    g1=f32(g1), be1=f32(be1), w3=w3p, b3=b3p, n_cls=n_cls)
    return cache.get([p for p in ps if p is not None], build)


class ClassifyHeadFn(torch.autograd.Function):
    """(feats_1, feats_2 or None) -> logits [B, num_classes] fp32.  meta = (pack, key_pad uint8 [B, S] or None, norm eps,
    classifier LayerNorm eps); then the 16 head_params (None for an absent pooler)."""

    @staticmethod
    def forward(ctx, meta, f1, f2, *params):
        pk, key_pad, eps_n, eps_c = meta
        feats = [f1] if f2 is None else [f1, f2]
        P = len(feats)
        B, S, d = f1.shape
        T = S - 1
        if T < 1:
            raise ValueError("attention pooling needs at least one token after CLS")
        dev = f1.device

        def e(r, n, dt=torch.bfloat16):
            return torch.empty(r, n, dtype=dt, device=dev)
        # classify_head.forward_features (one_peace_base.py:216-226): features[:, 1:], padding_masks[:, 1:]
        xb = e(P * B * T, d)
        for p, f in enumerate(feats):
            xb[p * B * T:(p + 1) * B * T].view(B, T, d).copy_(f[:, 1:])
        kp = None
        if key_pad is not None:
            kp = key_pad[:, 1:].to(torch.uint8)
            kp = (kp if P == 1 else torch.cat([kp] * P)).contiguous()         # the second pass reuses the first's mask
        kv = K.gemm(xb, pk["wkv"], K.EPI_STORE_BF16, e(P * B * T, 2 * d), bias=pk["bkv"])
        o, lse = K.attn_pool_fwd(kv, pk["q"], kp, P * B, T)
        y = K.gemm(o, pk["wo"], K.EPI_STORE_F32, e(P * B, d, torch.float32), bias=pk["bo"])
        zn = K.layernorm(y, pk["norm_w"], pk["norm_b"], e(P * B, d), eps=eps_n)
        t = None
        if pk["wp"] is not None:
            t = torch.tanh(K.gemm(zn, pk["wp"], K.EPI_STORE_F32, e(P * B, d, torch.float32), bias=pk["bp"]))
            pooled = t.to(torch.bfloat16)
        else:
            pooled = zn
        cin = pooled if P == 1 else torch.cat([pooled[:B], pooled[B:]], 1).contiguous()
        inner = pk["w0"].shape[0]
        h = K.gemm(cin, pk["w0"], K.EPI_STORE_F32, e(B, inner, torch.float32), bias=pk["b0"])
        g = K.layernorm(h, pk["g1"], pk["be1"], e(B, inner), eps=eps_c, gelu=True)
        logits = K.gemm(g, pk["w3"], K.EPI_STORE_F32, e(B, pk["w3"].shape[0], torch.float32), bias=pk["b3"])
        ctx.meta = (pk, eps_n, eps_c, P, B, T, d)
        ctx.saved = dict(xb=xb, kv=kv, kp=kp, o=o, lse=lse, y=y, zn=zn, t=t, cin=cin, h=h, g=g)
        ctx.dtypes = [p.dtype if p is not None else None for p in params]
        ctx.shapes = [p.shape if p is not None else None for p in params]
        return logits[:, :pk["n_cls"]]

    @staticmethod
    def backward(ctx, dlogits):
        pk, eps_n, eps_c, P, B, T, d = ctx.meta
        s = ctx.saved
        dev = dlogits.device
        n_cls = pk["n_cls"]
        inner = pk["w0"].shape[0]

        def e(r, n, dt=torch.bfloat16):
            return torch.empty(r, n, dtype=dt, device=dev)

        def g32(n):
            return torch.empty(n, dtype=torch.float32, device=dev)
        dl = torch.zeros(B, pk["w3"].shape[0], dtype=torch.bfloat16, device=dev)
        dl[:, :n_cls].copy_(dlogits)
        db3 = K.colsum(dl, g32(dl.shape[1]))[:n_cls]
        dW3 = _dw(dl, s["g"], torch.float32)[:n_cls]
        dg = _dx(dl, pk["w3"], inner)
        dg1, dbe1 = g32(inner), g32(inner)
        dh = K.layernorm_bwd(s["h"], dg, pk["g1"], pk["be1"], e(B, inner), eps=eps_c, gelu=True, dgamma=dg1, dbeta=dbe1)
        db0 = K.colsum(dh, g32(inner))
        dW0 = _dw(dh, s["cin"], torch.float32)
        dcin = _dx(dh, pk["w0"], P * d)
        dpool = dcin if P == 1 else torch.cat([dcin[:, :d], dcin[:, d:]], 0).contiguous()
        dWp = dbp = None
        if s["t"] is not None:
            t = s["t"]
            dt = (dpool.float() * (1.0 - t * t)).to(torch.bfloat16)          # tanh' on the [P*B, d] fp32 tensor
            dbp = K.colsum(dt, g32(d))
            dWp = _dw(dt, s["zn"], torch.float32)
            dzn = _dx(dt, pk["wp"], d)
        else:
            dzn = dpool
        dnw, dnb = g32(d), g32(d)
        dy = K.layernorm_bwd(s["y"], dzn, pk["norm_w"], pk["norm_b"], e(P * B, d), eps=eps_n, dgamma=dnw, dbeta=dnb)
        dbo = K.colsum(dy, g32(d))
        dWo = _dw(dy, s["o"], torch.float32)
        do = _dx(dy, pk["wo"], d)
        dkv, dq = K.attn_pool_bwd(s["kv"], pk["q"], s["kp"], s["lse"], do, P * B, T)
        dbv = K.colsum(dkv[:, d:], g32(d))
        dWkv = _dw(dkv, s["xb"], torch.float32)
        dfeats = [None, None]
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dxb = _dx(dkv, pk["wkv"], d)
            for p in range(P):
                if ctx.needs_input_grad[1 + p]:
                    df = torch.zeros(B, T + 1, d, dtype=torch.float32, device=dev)       # CLS row: no gradient
                    df[:, 1:].copy_(dxb[p * B * T:(p + 1) * B * T].view(B, T, d))
                    dfeats[p] = df
        grads = [dnw, dnb, dq, dWkv[:d], dWkv[d:], dbv, dWo, dbo, dWp, dbp, dW0, db0, dg1, dbe1, dW3, db3]
        out = [None if gr is None else gr.reshape(shp).to(dt) for gr, shp, dt in zip(grads, ctx.shapes, ctx.dtypes)]
        ctx.saved = None
        return (None, dfeats[0], dfeats[1], *out)


class ClassifyLossFn(torch.autograd.Function):
    """logits [rows, C] (any row pitch) -> (loss sum, n_correct sum, per-row n_correct); the gradient of the loss is computed
    in the same launch (opb_classify_loss) and scaled by the upstream gradient in the backward."""

    @staticmethod
    def forward(ctx, logits, mode, labels, targets, eps, num_choices):
        x = logits.detach()
        if x.dtype != torch.float32 or x.stride(1) != 1:
            x = x.float().contiguous()
        _, dl, row_correct, out2 = K.classify_loss(x, logits.shape[1], mode, labels=labels, targets=targets, eps=eps,
                                                    num_choices=num_choices)
        ctx.dl = dl[:, :logits.shape[1]]
        ctx.dtype = logits.dtype
        loss, n_correct = out2[0], out2[1]
        ctx.mark_non_differentiable(n_correct, row_correct)
        return loss, n_correct, row_correct

    @staticmethod
    def backward(ctx, g_loss, _g1, _g2):
        return (ctx.dl * g_loss.to(torch.float32)).to(ctx.dtype), None, None, None, None, None


class RefcocoLossFn(torch.autograd.Function):
    """logits [B, 4] (any row pitch), targets [B, 4], nsentences -> (loss, L1 part, n_valid) of refcoco_criterion
    (criterions/refcoco_loss.py:36-46); the gradient is computed in the same launch (opb_refcoco_loss) and scaled by the
    upstream gradient in the backward.  The loss is NaN when no row is valid while the gradient stays the finite L1 part."""

    @staticmethod
    def forward(ctx, logits, targets, nsentences):
        x = logits.detach()
        if x.dtype != torch.float32 or x.stride(1) != 1:
            x = x.float().contiguous()
        out, _, _, dl = K.refcoco_loss(x, targets.detach(), nsentences)
        ctx.dl = dl[:, :logits.shape[1]]
        ctx.dtype = logits.dtype
        l1, n_valid = out[1], out[2]
        ctx.mark_non_differentiable(l1, n_valid)
        return out[0], l1, n_valid

    @staticmethod
    def backward(ctx, g_loss, _g1, _g2):
        return (ctx.dl * g_loss.to(torch.float32)).to(ctx.dtype), None, None


class VitHeadFn(torch.autograd.Function):
    """Head of OnePeaceViT (one_peace_vision/classification/models_vit.py:431-434): the last layer's residual stream x fp32
    [B, S, d] -> logits fp32 [B, num_classes].

      global_pool : mean over the S - 1 patch rows -> fc_norm       (opb_token_mean_ln_fwd / _bwd, csrc/vit_head.cu)
      otherwise   : encoder.layer_norm on the CLS row                (opb_layernorm / opb_layernorm_bwd at a row pitch of S * d)
      then head (GEMM, output rows zero-padded to a multiple of 8).

    meta = (pack, global_pool, norm eps); then norm weight, norm bias, head weight, head bias.  The gradient of x is written
    whole by the kernels: the pooled form's backward writes every row, the CLS form's its rows into a zeroed buffer."""

    @staticmethod
    def forward(ctx, meta, x, nw, nb, w, b):
        pk, pool, eps = meta
        B, S, d = x.shape
        dev = x.device
        x = x.contiguous()
        if pool:
            a, m, mean, rstd = K.token_mean_ln_fwd(x, pk["norm_w"], pk["norm_b"], eps)
            ctx.saved = (m, mean, rstd)
        else:
            a = K.layernorm(x, pk["norm_w"], pk["norm_b"], torch.empty(B, d, dtype=torch.bfloat16, device=dev), rows=B, dim=d,
                            ld_in=S * d, ld_out=d, eps=eps)
            ctx.saved = (x,)
        logits = K.gemm(a, pk["w"], K.EPI_STORE_F32, torch.empty(B, pk["w"].shape[0], dtype=torch.float32, device=dev),
                        bias=pk["b"])
        ctx.meta = (pk, pool, eps, B, S, d)
        ctx.a = a
        ctx.dtypes = (nw.dtype, nb.dtype, w.dtype, b.dtype)
        return logits[:, :pk["n_cls"]]

    @staticmethod
    def backward(ctx, dlogits):
        pk, pool, eps, B, S, d = ctx.meta
        dev = dlogits.device
        n_cls, n_pad = pk["n_cls"], pk["w"].shape[0]
        dl = torch.zeros(B, n_pad, dtype=torch.bfloat16, device=dev)
        dl[:, :n_cls].copy_(dlogits)
        db = K.colsum(dl, torch.empty(n_pad, dtype=torch.float32, device=dev))[:n_cls]
        dW = _dw(dl, ctx.a, torch.float32)[:n_cls]
        da = _dx(dl, pk["w"], d, out=torch.empty(B, d, dtype=torch.float32, device=dev))
        if pool:
            m, mean, rstd = ctx.saved
            dx = torch.empty(B, S, d, dtype=torch.float32, device=dev)
            dnw, dnb = K.token_mean_ln_bwd(da, m, mean, rstd, pk["norm_w"], dx)
        else:
            (x,) = ctx.saved
            dx = torch.zeros(B, S, d, dtype=torch.float32, device=dev)
            dnw = torch.empty(d, dtype=torch.float32, device=dev)
            dnb = torch.empty(d, dtype=torch.float32, device=dev)
            K.layernorm_bwd(x, da, pk["norm_w"], pk["norm_b"], dx, eps=eps, dgamma=dnw, dbeta=dnb, rows=B, dim=d, ldx=S * d,
                            ld_dx=S * d)
        ctx.saved = ctx.a = None
        grads = [g.to(dt) for g, dt in zip((dnw, dnb, dW, db), ctx.dtypes)]
        return (None, dx, *grads)
