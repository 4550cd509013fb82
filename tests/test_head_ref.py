"""CPU: the bounds of tests/head_ref.py against the training Functions of one_peace_b200/autograd_classify.py and
one_peace_b200/autograd_general.py run on the fp64 emulation of their kernels (``test_stem_ref.Emu``).

The Functions run unchanged, packs, pads, views and concatenations included, from fresh copies of their modules
(``test_stem_ref.functions``).  Their results must stay within the bounds in every form the model uses, and each planted
mistake (a one-line change of a module's source, or of one emulated kernel) must exceed them at least 100-fold somewhere.

Each case builder runs one Function and returns a ``Res``: the share of its bound each output used, the outputs that may
come out exact (copies), the column reductions, the device outputs (for a bit-for-bit repeat on the GPU) and the outputs
that fp32 atomics make order-dependent.  tests/test_gpu_head_contract.py runs the same builders on the kernels."""
from collections import namedtuple
from types import SimpleNamespace as NS

import pytest
import torch

import head_ref as HR
import stem_ref as SR
from one_peace_b200 import autograd_classify as AC
from one_peace_b200 import autograd_general as AGN
from one_peace_b200.adapter.text import canvas_index, flat_ids
from test_classify_host_logic import HARD, HINGE, MULTI, SOFT
from test_stem_ref import MISS, Emu, functions

BF, F32 = torch.bfloat16, torch.float32
Res = namedtuple("Res", "shares exact reductions outputs atomic checks")


def _result(got, chk, exact=(), reductions=(), atomic=()):
    return Res(SR.shares(got, chk), set(exact), set(reductions), got, set(atomic), chk)


def _gen(seed):
    g = torch.Generator().manual_seed(seed)

    def rn(*s, sc=1.0, off=0.0, dt=F32, dev="cpu", grad=True):
        t = (off + sc * torch.randn(*s, generator=g)).to(dev, dt)
        return t.requires_grad_() if grad else t
    return g, rn


# ----------------------------------------------------------------------------------------------------------------------
# autograd_classify
# ----------------------------------------------------------------------------------------------------------------------
def classify_case(fns, B=3, S=6, d=128, ratio=2, n_cls=7, pooler=True, two=False, pads=((1, 4), (2, 2)), p_dtype=F32,
                  seed=0, dev="cpu"):
    """ClassifyHeadFn; pads: (sample, first padded token) per padded sample, None: no key_pad"""
    g, rn = _gen(seed)
    H, inner, c_in = d // 64, d * ratio, 2 * d if two else d
    feats = [rn(B, S, d, off=0.2, dev=dev) for _ in range(2 if two else 1)]
    kp = None
    if pads is not None:
        kp = torch.zeros(B, S, dtype=torch.uint8)
        for b, t in pads:
            kp[b, t:] = 1
        kp = kp.to(dev)
    p = lambda *s, **k: rn(*s, dt=p_dtype, dev=dev, **k)
    w = lambda n, k, sc=1.0: p(n, k, sc=sc * k ** -0.5)
    params = [p(d, sc=0.2, off=1.0), p(d, sc=0.1), p(1, 1, H, 64, sc=0.3), w(d, d), w(d, d), p(d, sc=0.1), w(d, d),
              p(d, sc=0.1)]
    params += [w(d, d, 1.5), p(d, sc=0.3)] if pooler else [None, None]        # pre-activations up to ~5: saturated units
    params += [w(inner, c_in), p(inner, sc=0.1), p(inner, sc=0.2, off=1.0), p(inner, sc=0.1), w(n_cls, inner),
               p(n_cls, sc=0.1)]
    nw, nb, q, wk, wv, bv, wo, bo, wp, bp, w0, b0, g1, be1, w3, b3 = params
    head = NS(norm=NS(weight=nw, bias=nb), attn_pooling_func=NS(q=q, k_proj=NS(weight=wk), v_proj=NS(weight=wv, bias=bv),
                                                                 out_proj=NS(weight=wo, bias=bo)),
              pooler=[None, NS(weight=wp, bias=bp)] if pooler else None,
              classifier=[NS(weight=w0, bias=b0), NS(weight=g1, bias=be1), None, NS(weight=w3, bias=b3)])
    pk = fns.head_pack(head, NS(get=lambda ps, build: build()))
    logits = fns.ClassifyHeadFn.apply((pk, kp, 1e-5, 1e-5), feats[0], feats[1] if two else None, *params)
    saved = logits.grad_fn.saved
    dl = torch.randn(B, n_cls, generator=g).to(dev)
    fns.K.log.clear()
    names = [f"f{i + 1}" for i in range(len(feats))] + [k for k, t in zip(HR.CLASSIFY_GRADS, params) if t is not None]
    got = dict(zip(names, torch.autograd.grad(logits, feats + [t for t in params if t is not None], dl)))
    chk, inter = HR.classify_head_ref(feats, kp, 1e-5, 1e-5, params, saved, dl, fns.K.log)
    got.update(inter, logits=logits)
    return _result(got, chk, exact=("xb", "cin", "dl") + (() if pooler else ("dzn",)),
                   reductions=("b3", "b0", "bp", "bo", "bv", "g1", "be1", "nw", "nb", "q", "lse"))


def vit_case(fns, B=3, S=7, d=64, n_cls=9, pool=True, p_dtype=F32, seed=1, dev="cpu"):
    """VitHeadFn, pooled (global_pool) or CLS form"""
    g, rn = _gen(seed)
    x = (rn(B, S, d, dev=dev, grad=False) + rn(1, 1, d, sc=0.5, dev=dev, grad=False)).requires_grad_()
    nw, nb = rn(d, sc=0.2, off=1.0, dt=p_dtype, dev=dev), rn(d, sc=0.1, dt=p_dtype, dev=dev)
    w, b = rn(n_cls, d, sc=d ** -0.5, dt=p_dtype, dev=dev), rn(n_cls, sc=0.1, dt=p_dtype, dev=dev)
    n_pad = (n_cls + 7) // 8 * 8
    wpk = torch.zeros(n_pad, d, dtype=BF, device=dev)
    wpk[:n_cls] = w.detach().to(BF)
    bpk = torch.zeros(n_pad, device=dev)
    bpk[:n_cls] = b.detach().float()
    pk = dict(norm_w=nw.detach().float(), norm_b=nb.detach().float(), w=wpk, b=bpk, n_cls=n_cls)
    logits = fns.VitHeadFn.apply((pk, pool, 1e-6), x, nw, nb, w, b)
    saved, a = logits.grad_fn.saved, logits.grad_fn.a
    dl = torch.randn(B, n_cls, generator=g).to(dev)
    fns.K.log.clear()
    got = dict(zip(HR.VIT_GRADS, torch.autograd.grad(logits, [x, nw, nb, w, b], dl)))
    chk, inter = HR.vit_head_ref(x, nw, nb, w, b, pool, 1e-6, saved, a, dl, fns.K.log)
    got.update(inter, logits=logits)
    return _result(got, chk, exact=("dl",), reductions=("nw", "nb", "b", "m", "mean", "rstd"))


def _distinct_logits(g, rows, C):
    """well-separated values per row (0.5 apart): arg-max and hinge activity are the same in fp32, bf16 and fp64"""
    z = torch.stack([torch.randperm(C, generator=g) for _ in range(rows)]).double() * 0.5 - C / 4
    return z + 0.05 * torch.rand(rows, C, generator=g)


def loss_case(fns, mode=HARD, rows=6, C=9, ld=16, dtype=F32, eps=0.1, g_loss=0.37, num_choices=1, seed=2, dev="cpu"):
    """ClassifyLossFn on logits [rows, C] read out of a [rows, ld] buffer (a row pitch of ld), upstream gradient g_loss"""
    g, _ = _gen(seed)
    buf = torch.randn(rows, ld, generator=g).double()
    buf[:, :C] = _distinct_logits(g, rows, C)
    buf = buf.to(dev, dtype).requires_grad_()
    logits = buf[:, :C]
    labels = targets = None
    if mode == HARD:
        labels = torch.randint(0, C, (rows,), generator=g).to(dev)
    elif mode == SOFT:
        targets = torch.softmax(torch.randn(rows, C, generator=g), 1).to(dev)
    elif mode == MULTI:
        targets = (torch.rand(rows, C, generator=g) < 0.3).float().to(dev)
    else:
        labels = torch.randint(0, num_choices, (rows // num_choices,), generator=g).to(dev)
    loss, n_correct, row_correct = fns.ClassifyLossFn.apply(logits, mode, labels, targets, eps, num_choices)
    gl = torch.tensor(g_loss, device=dev)
    (dz,) = torch.autograd.grad(loss, [logits], gl)
    chk = HR.classify_loss_ref(logits, mode, labels, targets, eps, num_choices, gl)
    got = dict(loss=loss.reshape(1), n_correct=n_correct.reshape(1), row_correct=row_correct, dlogits=dz)
    # hinge: dlogits are counts of active margins times g_loss, which fp32 may hold exactly
    return _result(got, chk, exact=("n_correct", "row_correct") + (("dlogits",) if mode == HINGE else ()),
                   reductions=("loss",))


def refcoco_case(fns, B=7, ld=8, dtype=F32, ns=5, g_loss=0.37, seed=3, dev="cpu"):
    """RefcocoLossFn on box logits [B, 4] read out of a [B, ld] buffer; row 1's box is inverted (not valid)"""
    g, _ = _gen(seed)
    lo = 0.1 + 0.3 * torch.rand(B, 2, generator=g, dtype=torch.float64)
    p = torch.cat([lo, lo + 0.1 + 0.4 * torch.rand(B, 2, generator=g, dtype=torch.float64)], 1)
    p[1] = p[1, [2, 3, 0, 1]]
    lo = 0.1 + 0.3 * torch.rand(B, 2, generator=g, dtype=torch.float64)
    t = torch.cat([lo, lo + 0.1 + 0.4 * torch.rand(B, 2, generator=g, dtype=torch.float64)], 1).float().to(dev)
    buf = torch.randn(B, ld, generator=g, dtype=torch.float64)
    buf[:, :4] = torch.logit(p)
    buf = buf.to(dev, dtype).requires_grad_()
    logits = buf[:, :4]
    loss, l1, nv = fns.RefcocoLossFn.apply(logits, t, ns)
    gl = torch.tensor(g_loss, device=dev)
    (dz,) = torch.autograd.grad(loss, [logits], gl)
    chk = HR.refcoco_loss_ref(logits, t, ns, gl)
    got = dict(loss=loss.reshape(1), l1=l1.reshape(1), n_valid=nv.reshape(1), dlogits=dz)
    return _result(got, chk, exact=("n_valid",), reductions=("loss", "l1"))


# ----------------------------------------------------------------------------------------------------------------------
# autograd_general
# ----------------------------------------------------------------------------------------------------------------------
def dcl_case(fns, B=2, S=10, d=32, pad_from=(None, 6), s_dtype=F32, scale=2.5, eps=0.1, g_loss=0.37, seed=4, dev="cpu"):
    """DclLossFn with the row selections of compute_dcl_loss (``dcl_indices``): about half the tokens masked, sample b's
    tokens padded from pad_from[b]"""
    g, rn = _gen(seed)
    student = rn(B * S, d, dt=s_dtype, dev=dev)
    teacher = rn(B * S, d, dev=dev, grad=False)
    mask = torch.rand(B, S, generator=g) < 0.5
    pad = torch.zeros(B, S - 1, dtype=torch.bool)
    for b, f in enumerate(pad_from):
        if f is not None:
            pad[b, f:] = True
    stu_idx, tea_idx = fns.dcl_indices(mask.to(dev), pad.to(dev))
    assert stu_idx.numel() % 8 and tea_idx.numel() % 8, "row counts that are multiples of 8 would not exercise the padding"
    fns.K.log.clear()
    loss = fns.DclLossFn.apply(student, teacher, stu_idx, tea_idx, scale, eps)
    fwd_log = list(fns.K.log)
    fns.K.log.clear()
    gl = torch.tensor(g_loss, device=dev)
    (ds,) = torch.autograd.grad(loss, [student], gl)
    chk, got = HR.dcl_ref(student, teacher, stu_idx, tea_idx, scale, eps, gl, fwd_log, fns.K.log)
    got["student"] = ds
    # the student's gradient: each selected row receives one fp32 addition onto zero, exact
    return _result(got, chk, exact=("s_rows", "t_rows", "a3", "b3", "student"), reductions=("loss", "lse"))


def _preserve_ids(g, B, K, S, n_pad):
    """(B, K) kept positions (CLS first, the rest sorted), the last n_pad[b] slots of sample b padded with -1"""
    ids = torch.stack([torch.cat([torch.zeros(1, dtype=torch.long), 1 + torch.randperm(S - 1, generator=g)[:K - 1].sort()[0]])
                       for _ in range(B)])
    for b, n in enumerate(n_pad):
        if n:
            ids[b, K - n:] = -1
    return ids


def gather_case(fns, form="canvas", B=2, S=9, K=5, d=16, seed=5, dev="cpu"):
    """RowGatherFn as the adapters call it: the decoder's mask-token canvas with positions ('canvas', text.py:120), the
    encoder's preserve-ids gather ('preserve', text.py:137) and the audio frame gather with a repeated index ('repeat',
    audio.py:286-291)"""
    g, rn = _gen(seed)
    ids = _preserve_ids(g, B, K, S, (0, 2))
    fill = add = None
    if form == "canvas":
        src = rn(B * K, d, dev=dev)
        idx = canvas_index(ids, S)
        fill, add = rn(1, d, dev=dev), rn(S, d, sc=0.5, dev=dev)
    elif form == "preserve":
        src = rn(B * S, d, dev=dev)
        idx = flat_ids(ids, S)
    else:
        T = S - 1
        src = rn(B * T, d, dev=dev)
        pid = ids.masked_fill(ids.eq(-1), K - 1)[:, 1:] - 1
        idx = (pid + torch.arange(B)[:, None] * T).reshape(-1).contiguous()
        assert idx.unique().numel() < idx.numel()
    idx = idx.to(dev)
    out = fns.RowGatherFn.apply(src, idx, fill, add)
    dout = torch.randn(out.shape, generator=g).to(dev)
    ins = [t for t in (src, fill, add) if t is not None]
    names = [n for n, t in (("src", src), ("fill", fill), ("add", add)) if t is not None]
    got = dict(zip(names, torch.autograd.grad(out, ins, dout)), out=out)
    chk = HR.row_gather_fn_ref(src, idx, fill, add, dout)
    return _result(got, chk, exact=("out", "src") if add is None else ("src",), reductions=("src", "fill", "add"),
                   atomic=("src",) if form == "repeat" else ())


def zero_pad_case(fns, B=3, S=6, d=16, seed=6, dev="cpu"):
    g, rn = _gen(seed)
    x = rn(B * S, d, dev=dev)
    pad = (torch.rand(B * S, generator=g) < 0.3).to(torch.uint8).to(dev)
    out = fns.ZeroPadFn.apply(x, pad)
    dout = torch.randn(out.shape, generator=g).to(dev)
    (dx,) = torch.autograd.grad(out, [x], dout)
    return _result(dict(out=out, x=dx), HR.zero_pad_ref(x, pad, dout), exact=("out", "x"))


def _bucket(g, L, nb):
    return torch.randint(0, nb - 3, (L, L), generator=g)                # the last three rows of the table stay unused


def block_bias_case(fns, H=4, n_t=5, n_i=6, Bb=3, L=10, mixed=True, t_dtype=F32, seed=7, dev="cpu"):
    """BlockBiasFn on a 'vl' canvas: the text block shared by every sample (ids None) at 0..n_t-1, and, when mixed, the
    image block gathered per sample by preserve ids (with padded slots) at n_t..; otherwise the shared block alone"""
    g, rn = _gen(seed)
    tables = [rn(20, H, dt=t_dtype, dev=dev)]
    blocks = [(_bucket(g, n_t, 20).to(dev), None, n_t, 0)]
    S = n_t
    if mixed:
        tables.append(rn(30, H, dt=t_dtype, dev=dev))
        ids = torch.stack([torch.randperm(L, generator=g)[:n_i] for _ in range(Bb)])
        ids[1, -2:] = -1
        blocks.append((_bucket(g, L, 30).to(dev), ids.to(dev), n_i, n_t))
        S += n_i
    bias = fns.BlockBiasFn.apply((H, S, blocks), *tables)
    db = torch.randn(bias.shape, generator=g).to(dev)
    names = [f"t{i}" for i in range(len(tables))]
    got = dict(zip(names, torch.autograd.grad(bias, tables, db)), bias=bias)
    return _result(got, HR.block_bias_ref(H, S, blocks, tables, db), exact=("bias",), reductions=names, atomic=names)


def linear_case(fns, rows=10, n_in=24, n_out=40, bias=True, x_dtype=F32, p_dtype=F32, seed=8, dev="cpu"):
    g, rn = _gen(seed)
    x = rn(rows, n_in, dt=x_dtype, dev=dev)
    w = rn(n_out, n_in, sc=n_in ** -0.5, dt=p_dtype, dev=dev)
    b = rn(n_out, sc=0.1, dt=p_dtype, dev=dev) if bias else None
    y = fns.LinearFn.apply(x, w, b)
    saved = y.grad_fn.saved_tensors
    dy = torch.randn(y.shape, generator=g).to(dev)
    fns.K.log.clear()
    ins = [x, w] + ([b] if bias else [])
    got = dict(zip(("x", "w", "b"), torch.autograd.grad(y, ins, dy)), y=y)
    chk, inter = HR.linear_fn_ref(x, w, b, saved, dy, fns.K.log)
    got.update(inter)
    return _result(got, chk, exact=("xb", "dyb"), reductions=("b",))


def final_norm_case(fns, rows=12, d=48, seed=9, dev="cpu"):
    g, rn = _gen(seed)
    x = (rn(rows, d, dev=dev, grad=False) + rn(rows, 1, dev=dev, grad=False)).requires_grad_()
    w, b = rn(d, sc=0.2, off=1.0, dev=dev), rn(d, sc=0.1, dev=dev)
    out = fns.FinalNormFn.apply(x, w, b, 1e-6)
    dy = torch.randn(out.shape, generator=g).to(dev)
    got = dict(zip(("x", "w", "b"), torch.autograd.grad(out, [x, w, b], dy)), out=out)
    return _result(got, HR.final_norm_ref(x, w, b, 1e-6, dy), reductions=("w", "b"))


CASE_FNS = dict(classify=(classify_case, AC), vit=(vit_case, AC), loss=(loss_case, AC), refcoco=(refcoco_case, AC),
                dcl=(dcl_case, AGN), gather=(gather_case, AGN), zero_pad=(zero_pad_case, AGN),
                block_bias=(block_bias_case, AGN), linear=(linear_case, AGN), final_norm=(final_norm_case, AGN))

# name -> (case, arguments)
CASES = {
    "classify_pooler_keypad_7cls": ("classify", {}),
    "classify_no_pooler_no_keypad_9cls": ("classify", dict(pooler=False, pads=None, n_cls=9, seed=10)),
    "classify_two_images_pooler_keypad": ("classify", dict(two=True, n_cls=2, seed=11)),
    "classify_two_images_no_pooler": ("classify", dict(two=True, pooler=False, pads=None, n_cls=9, seed=12)),
    "classify_t1_1cls": ("classify", dict(S=2, n_cls=1, pads=(), seed=13)),
    "classify_bf16_params_two_heads": ("classify", dict(d=128, p_dtype=BF, pads=((0, 3),), seed=14)),
    "vit_pooled_9cls": ("vit", {}),
    "vit_cls_7cls": ("vit", dict(pool=False, n_cls=7, seed=15)),
    "vit_pooled_1cls_bf16": ("vit", dict(n_cls=1, p_dtype=BF, seed=16)),
    "vit_cls_s2": ("vit", dict(pool=False, S=2, B=2, seed=17)),
    "loss_hard_strided": ("loss", {}),
    "loss_hard_bf16": ("loss", dict(dtype=BF, ld=9, g_loss=-1.5, seed=18)),
    "loss_soft_strided": ("loss", dict(mode=SOFT, eps=0.0, seed=19)),
    "loss_multi_bf16_strided": ("loss", dict(mode=MULTI, dtype=BF, eps=0.0, seed=20)),
    "loss_hinge": ("loss", dict(mode=HINGE, rows=8, C=1, ld=1, num_choices=4, eps=0.0, seed=21)),
    "refcoco_strided": ("refcoco", {}),
    "refcoco_bf16": ("refcoco", dict(dtype=BF, ld=4, g_loss=2.0, seed=22)),
    "dcl": ("dcl", {}),
    "dcl_bf16_student": ("dcl", dict(s_dtype=BF, pad_from=(5, None), eps=0.0, seed=4)),
    "gather_canvas": ("gather", {}),
    "gather_preserve": ("gather", dict(form="preserve", seed=24)),
    "gather_repeat": ("gather", dict(form="repeat", seed=25)),
    "zero_pad": ("zero_pad", {}),
    "block_bias_shared": ("block_bias", dict(mixed=False)),
    "block_bias_mixed": ("block_bias", dict(seed=26)),
    "block_bias_mixed_bf16": ("block_bias", dict(t_dtype=BF, seed=27)),
    "linear": ("linear", {}),
    "linear_bf16_no_bias": ("linear", dict(bias=False, x_dtype=BF, p_dtype=BF, seed=28)),
    "final_norm": ("final_norm", {}),
}


def run(case, args, kernels, edit=None, dev="cpu"):
    build, module = CASE_FNS[case]
    return build(functions(kernels, edit, module), **args, dev=dev)


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulation_within_bounds(name):
    case, args = CASES[name]
    sh = run(case, args, Emu()).shares
    bad = {k: v for k, v in sh.items() if not v <= 1.0}
    assert not bad, f"{name}: outside the bound: {bad}"


# name -> (case, case arguments, source edit, emulated-kernel flags)
E = lambda old, new: dict(edit=(old, new))
MISTAKES = {
    # ClassifyHeadFn
    "dbv from the k half of dkv": ("classify", {}, E("K.colsum(dkv[:, d:]", "K.colsum(dkv[:, :d]")),
    "two passes swapped in cin": ("classify", dict(two=True, n_cls=2, seed=11),
                                  E("torch.cat([pooled[:B], pooled[B:]], 1)", "torch.cat([pooled[B:], pooled[:B]], 1)")),
    "dcin halves swapped": ("classify", dict(two=True, n_cls=2, seed=11),
                            E("torch.cat([dcin[:, :d], dcin[:, d:]], 0)", "torch.cat([dcin[:, d:], dcin[:, :d]], 0)")),
    "second pass without the first's mask": ("classify", dict(two=True, n_cls=2, seed=11),
                                             E("torch.cat([kp] * P)", "torch.cat([kp, torch.zeros_like(kp)])")),
    "tanh' floored on saturated units": ("classify", {}, E("(1.0 - t * t)", "(1.0 - t * t).clamp_min(1e-2)")),
    "key_pad shifted the wrong way": ("classify", {}, E("key_pad[:, 1:]", "key_pad[:, :-1]")),
    "CLS row takes a gradient": ("classify", {}, E("df[:, 1:].copy_(", "df[:, :-1].copy_(")),
    "dW3 from the padded rows": ("classify", dict(n_cls=9, pads=None, seed=10),
                                 E('s["g"], torch.float32)[:n_cls]', 's["g"], torch.float32)[-n_cls:]')),
    # ClassifyLossFn, RefcocoLossFn
    "classify loss ignores the upstream gradient": ("loss", {}, E(
        "(ctx.dl * g_loss.to(torch.float32)).to(ctx.dtype), None, None, None, None, None",
        "ctx.dl.to(ctx.dtype), None, None, None, None, None")),
    "refcoco gradient read at the logits' width": ("refcoco", {}, E(
        "ctx.dl = dl[:, :logits.shape[1]]\n        ctx.dtype = logits.dtype\n        l1",
        "ctx.dl = dl.view(-1)[:logits.numel()].view(logits.shape)\n        ctx.dtype = logits.dtype\n        l1")),
    # VitHeadFn
    "ViT CLS dx at the row pitch d": ("vit", dict(pool=False, n_cls=7, seed=15), E("ld_dx=S * d)", "ld_dx=d)")),
    "ViT fc_norm dgamma and dbeta swapped": ("vit", {}, E("dnw, dnb = K.token_mean_ln_bwd", "dnb, dnw = K.token_mean_ln_bwd")),
    # DclLossFn
    "DCL without 1 / n_m": ("dcl", {}, E("coef=1.0 / n_m", "coef=1.0")),
    "DCL ignores the upstream gradient": ("dcl", {}, E("K.row_scatter_add(dx32 * g_loss.to(torch.float32), stu_idx, ds)",
                                                       "K.row_scatter_add(dx32, stu_idx, ds)")),
    # RowGatherFn
    "dfill summed over the gathered rows": ("gather", {}, E("torch.nonzero(idx < 0,", "torch.nonzero(idx >= 0,")),
    "scatter-add keeps one of repeated rows": ("gather", dict(form="repeat", seed=25), dict(flags=dict(scatter_overwrite=True))),
    "dadd over one period": ("gather", {}, E("dout.shape[0] // period, period * dim", "1, period * dim")),
    # BlockBiasFn
    "shared block written into sample 0 only": ("block_bias", dict(seed=26), E(
        "for bb in range(Bb):\n                    K.relpos_bias_block(f32(t)",
        "for bb in range(1):\n                    K.relpos_bias_block(f32(t)")),
    "shared block's gradient from sample 0 only": ("block_bias", dict(seed=26), E(
        "for bb in range(Bb):\n                    K.relpos_bias_block_bwd(",
        "for bb in range(1):\n                    K.relpos_bias_block_bwd(")),
    # ZeroPadFn, LinearFn, FinalNormFn
    "padded rows keep their gradient": ("zero_pad", {}, E("K.zero_padded_rows(dx, pad_rows)", "pass")),
    "dW against rows shifted by one": ("linear", {}, E("dW = _dw(dyb, xb, w.dtype)", "dW = _dw(dyb, xb.roll(1, 0), w.dtype)")),
    "final norm dgamma and dbeta swapped": ("final_norm", {}, E("dgamma=dg, dbeta=db", "dgamma=db, dbeta=dg")),
}


@pytest.mark.parametrize("name", sorted(MISTAKES))
def test_planted_mistake_exceeds_bound(name):
    case, args, how = MISTAKES[name]
    sh = run(case, args, Emu(**how.get("flags", {})), how.get("edit")).shares
    worst = max(sh, key=sh.get)
    assert sh[worst] >= MISS, f"{name}: largest share of a bound only {sh[worst]:.3g} ({worst})"


# (case, arguments, output, index) of outputs whose reference is exactly zero: the bound there is zero, so the value must be
EXACT_ZEROS = [
    ("classify", {}, "f1", (slice(None), 0)),                                     # the CLS rows
    ("classify", {}, "dkv", ([8, 9, 11, 12, 13, 14], slice(None))),               # keys padded in samples 1 and 2 (T = 5)
    ("classify", {}, "dl", (slice(None), slice(7, None))),                        # the classifier's padded columns
    ("vit", dict(pool=False, n_cls=7, seed=15), "x", (slice(None), slice(1, None))),
    ("block_bias", dict(seed=26), "t0", (slice(17, None),)),                      # table rows no bucket uses
    ("block_bias", dict(seed=26), "t1", (slice(27, None),)),
]


@pytest.mark.parametrize("case,args,name,at", EXACT_ZEROS)
def test_exact_zeros(case, args, name, at):
    r = run(case, args, Emu())
    ref, bound, _ = r.checks[name]
    assert (bound[at] == 0).all() and (ref[at] == 0).all()
    assert (r.outputs[name].detach().double().reshape(ref.shape)[at] == 0).all()
    t = r.outputs[name].detach().clone().reshape(ref.shape)
    t[at] = 1e-30                                  # any nonzero value there is infinitely far outside its bound
    assert SR.share(t, ref, bound, torch.float32) == float("inf")


def test_exact_zeros_of_masked_rows():
    """ZeroPadFn's padded rows and DclLossFn's student rows outside stu_idx"""
    r = run("zero_pad", {}, Emu())
    rows = r.checks["x"][0].abs().sum(1) == 0
    assert 0 < int(rows.sum()) < rows.numel() and (r.outputs["x"][rows] == 0).all() and (r.outputs["out"][rows] == 0).all()
    r = run("dcl", {}, Emu())
    ref, bound, _ = r.checks["student"]
    rows = bound.sum(1) == 0
    assert 0 < int(rows.sum()) < rows.numel() and (ref[rows] == 0).all() and (r.outputs["student"][rows] == 0).all()
