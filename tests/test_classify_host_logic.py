"""CPU: host logic of one_peace_classify and the fp64 references of its three kernels (csrc/classify.cu).

Error contract.  u = 2^-24 (fp32 unit roundoff), ub = 2^-8 (bf16).  Inputs are what the kernels read (bf16 kv / dout, fp32 q /
logits), so the references start from the same values and only the kernels' own arithmetic is bounded:
  * a 64-term fp32 dot product errs by at most (64 + 8) u sum_i |a_i b_i|; a score error e_s moves p_j by <= p_j (2 e_s + 8u);
  * a fixed-order fp32 sum of n terms errs by at most (n + 8) u sum |terms|; expf / logf by <= 4u relative;
  * every bf16 output carries one rounding, ub |value|.
Pooling forward, per (b, h) with E = max_j e_s(j) + 8u and the key count n:  |d out_e| <= ub |out_e| + (2E + (n + 16) u) sum_j
p_j |v_je|;  |d lse| <= E + (n + 16) u + u |lse|.
Pooling backward: |d dp_j| <= (72 u) sum_i |dout_i v_ji|; |d delta| <= sum_j (|dp_j| |d p_j| + p_j |d dp_j|) + (n + 16) u sum_j p_j |dp_j|;
|d ds_j| <= |d p_j| |dp_j - delta| + p_j (|d dp_j| + |d delta|) + 2u |ds_j|; dk = ds q and dv = p dout then add ub |value|; dq sums
over B n terms: |d dq| <= sum |d ds_j| |k_j| + (B n + 16) u sum |ds_j k_j|.
Loss (C = n_valid classes): lse errs by L = (C + 16) u (1 + |lse|); every row value is bounded by the propagated L plus
(C + 16) u times the sum of the magnitudes of its terms; the totals add (rows + 16) u sum |row values|.
"""
import math

import pytest
import torch

import synth
import synth_classify as sc

u = 2.0 ** -24
ub = 2.0 ** -8


# ------------------------------------------------------------------------------------------------------------------------------
# fp64 references with bounds
# ------------------------------------------------------------------------------------------------------------------------------
def _split(kv, B, T):
    kv = kv.double().view(B, T, 2, -1)
    return kv[:, :, 0], kv[:, :, 1]


def pool_fwd_ref(kv, q, key_pad, B, T):
    """kv [B*T, 2d], q [H, 64], key_pad [B, T] uint8 or None -> (out [B, d], lse [B, H], bound_out, bound_lse), fp64."""
    H = q.shape[0]
    k, v = _split(kv, B, T)
    k, v = k.view(B, T, H, 64), v.view(B, T, H, 64)
    qd = q.double()
    s = torch.einsum("bthe,he->bht", k, qd)
    es = 72 * u * torch.einsum("bthe,he->bht", k.abs(), qd.abs())
    valid = torch.ones(B, T, dtype=torch.bool, device=kv.device) if key_pad is None else key_pad == 0
    s = s.masked_fill(~valid[:, None, :], -math.inf)
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    out = torch.einsum("bht,bthe->bhe", p, v)
    n = valid.sum(1).double()[:, None]
    E = es.masked_fill(~valid[:, None, :], 0).amax(-1) + 8 * u
    pv = torch.einsum("bht,bthe->bhe", p, v.abs())
    b_out = ub * out.abs() + (2 * E + (n + 16) * u)[..., None] * pv
    b_lse = E + (n + 16) * u + u * lse.abs()
    return out.reshape(B, -1), lse, b_out.reshape(B, -1), b_lse


def pool_bwd_ref(kv, q, key_pad, dout, B, T):
    """-> (dkv [B*T, 2d], dq [H, 64], bound_dkv, bound_dq), fp64."""
    H = q.shape[0]
    k, v = _split(kv, B, T)
    k, v = k.view(B, T, H, 64), v.view(B, T, H, 64)
    qd, do = q.double(), dout.double().view(B, H, 64)
    valid = torch.ones(B, T, dtype=torch.bool, device=kv.device) if key_pad is None else key_pad == 0
    s = torch.einsum("bthe,he->bht", k, qd).masked_fill(~valid[:, None, :], -math.inf)
    es = 72 * u * torch.einsum("bthe,he->bht", k.abs(), qd.abs())
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    n = valid.sum(1).double()[:, None, None]
    E = es.masked_fill(~valid[:, None, :], 0).amax(-1, keepdim=True) + 8 * u
    dp = torch.einsum("bthe,bhe->bht", v, do)
    edp = 72 * u * torch.einsum("bthe,bhe->bht", v.abs(), do.abs())
    delta = (p * dp).sum(-1, keepdim=True)
    dpj = p * (2 * E + (n + 16) * u)
    edelta = (dp.abs() * dpj + p * edp).sum(-1, keepdim=True) + (n + 16) * u * (p * dp.abs()).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    eds = dpj * (dp - delta).abs() + p * (edp + edelta) + 2 * u * ds.abs()
    dk = torch.einsum("bht,he->bthe", ds, qd)
    dv = torch.einsum("bht,bhe->bthe", p, do)
    bdk = torch.einsum("bht,he->bthe", eds, qd.abs()) + ub * dk.abs()
    bdv = torch.einsum("bht,bhe->bthe", dpj, do.abs()) + ub * dv.abs() + u * dv.abs()
    dq = torch.einsum("bht,bthe->he", ds, k)
    bdq = torch.einsum("bht,bthe->he", eds, k.abs()) + (B * T + 16) * u * torch.einsum("bht,bthe->he", ds.abs(), k.abs())
    dkv = torch.stack([dk.reshape(B, T, -1), dv.reshape(B, T, -1)], 2).reshape(B * T, -1)
    bkv = torch.stack([bdk.reshape(B, T, -1), bdv.reshape(B, T, -1)], 2).reshape(B * T, -1)
    return dkv, dq, bkv, bdq


HARD, SOFT, MULTI, HINGE = 0, 1, 2, 3


def loss_ref(logits, n_valid, mode, labels=None, targets=None, eps=0.0, num_choices=1):
    """logits [rows, >= n_valid] -> dict(row_loss, dlogits [rows, n_valid], row_correct, loss, n_correct) and the bounds
    b_row_loss, b_dlogits, b_row_correct, b_loss, b_n_correct (fp64)."""
    z = logits[:, :n_valid].double()
    C = n_valid
    if mode == HINGE:
        zg = z[:, 0].view(-1, num_choices)
        G = zg.shape[0]
        t = labels.long()
        pos = zg.gather(1, t[:, None])
        h = 1 + zg - pos
        act = (h > 0).double()
        row = (h.clamp_min(0)).sum(1)
        dz = act.clone()
        dz.scatter_add_(1, t[:, None], -act.sum(1, keepdim=True))
        corr = (zg.argmax(1) == t).double()
        brow = (num_choices + 16) * u * (1 + zg.abs() + pos.abs()).sum(1)
        bdz = torch.zeros_like(dz)
        dl = dz.view(-1, 1)
        bdl = bdz.view(-1, 1)
    else:
        mx = z.max(1, keepdim=True).values
        lse = torch.logsumexp(z, 1, keepdim=True)
        p = torch.softmax(z, 1)
        L = (C + 16) * u * (1 + lse.abs())
        bp = p * (2 * L + (z - mx).abs() * 2 * u + 8 * u)
        if mode == MULTI:
            t = targets[:, :C].double()
            row = (z.clamp_min(0) - z * t + torch.log1p(torch.exp(-z.abs()))).sum(1)
            dl = torch.sigmoid(z) - t
            corr = t.gather(1, z.argmax(1, keepdim=True))[:, 0]
            brow = (C + 16) * u * (z.abs() * (1 + t.abs()) + 1).sum(1)
            bdl = 8 * u * (torch.sigmoid(z) + t.abs())
            bcorr = torch.zeros_like(corr)
        elif mode == SOFT:
            t = targets[:, :C].double()
            row = (t * (lse - z)).sum(1)
            ts = t.sum(1, keepdim=True)
            dl = ts * p - t
            corr = (p * t).sum(1)
            brow = (C + 16) * u * (t.abs() * (lse.abs() + z.abs())).sum(1) + L[:, 0] * t.abs().sum(1)
            bdl = bp * ts.abs() + (C + 16) * u * t.abs().sum(1, keepdim=True) * p + 2 * u * dl.abs()
            bcorr = (bp * t.abs()).sum(1) + (C + 16) * u * (p * t.abs()).sum(1)
        else:
            t = labels.long()
            valid = (t >= 0) & (t < C)
            tc = t.clamp(0, C - 1)
            zt = z.gather(1, tc[:, None])[:, 0]
            row = ((1 - eps) * (lse[:, 0] - zt) + eps * (lse[:, 0] - z.mean(1))) * valid
            dl = (p - (1 - eps) * torch.nn.functional.one_hot(tc, C) - eps / C) * valid[:, None]
            corr = ((z.argmax(1) == t) & valid).double()
            brow = (L[:, 0] + (C + 16) * u * (z.abs().sum(1) / C * eps + lse.abs()[:, 0] + zt.abs())) * valid
            bdl = (bp + 2 * u * dl.abs() + 4 * u * eps / C) * valid[:, None]          # eps / C: fp32 eps, a division
            bcorr = torch.zeros_like(corr)
        if mode != SOFT:
            bcorr = torch.zeros_like(corr)
        bdz = None
    if mode == HINGE:
        bcorr = torch.zeros_like(corr)
    nr = row.numel()
    return dict(row_loss=row, dlogits=dl, row_correct=corr, loss=row.sum(), n_correct=corr.sum(),
                b_row_loss=brow, b_dlogits=bdl, b_row_correct=bcorr,
                b_loss=brow.sum() + (nr + 16) * u * row.abs().sum(),
                b_n_correct=bcorr.sum() + (nr + 16) * u * corr.abs().sum())


def excess(got, want, bound):
    """max over elements of |got - want| / bound (> 1 is a violation; exact agreement where the bound is 0)."""
    err = (got.double() - want.double()).abs()
    b = bound.double()
    r = torch.where(b > 0, err / b.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return r.max().item()


# ------------------------------------------------------------------------------------------------------------------------------
# fp32 emulation of the kernels, with the mistakes the bounds must catch
# ------------------------------------------------------------------------------------------------------------------------------
def pool_fwd_emul(kv, q, key_pad, B, T, mistake=None):
    H = q.shape[0]
    kvf = kv.float().view(B, T, 2, H, 64)
    k, v = kvf[:, :, 0], kvf[:, :, 1]
    qf = q.float()
    if mistake == "q_scaled":
        qf = qf / 8
    if mistake == "neighbour_head":
        qf = qf.roll(1, 0)
    if mistake == "k_bias":
        k = k + 0.1
    s = torch.einsum("bthe,he->bht", k, qf)
    valid = torch.ones(B, T, dtype=torch.bool, device=kv.device) if key_pad is None else key_pad == 0
    if mistake != "padded_key":
        s = s.masked_fill(~valid[:, None, :], -math.inf)
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    out = (torch.einsum("bht,bthe->bhe", e, v) / l).bfloat16()
    return out.reshape(B, -1), (m + torch.log(l))[..., 0]


def pool_bwd_emul(kv, q, key_pad, dout, B, T, mistake=None):
    H = q.shape[0]
    kvf = kv.float().view(B, T, 2, H, 64)
    k, v = kvf[:, :, 0], kvf[:, :, 1]
    qf, do = q.float(), dout.float().view(B, H, 64)
    valid = torch.ones(B, T, dtype=torch.bool, device=kv.device) if key_pad is None else key_pad == 0
    s = torch.einsum("bthe,he->bht", k, qf).masked_fill(~valid[:, None, :], -math.inf)
    p = torch.softmax(s, -1)
    dp = torch.einsum("bthe,bhe->bht", v, do)
    delta = (p * dp).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    dk = torch.einsum("bht,he->bthe", ds, qf).bfloat16()
    dv = torch.einsum("bht,bhe->bthe", p, do).bfloat16()
    part = torch.einsum("bht,bthe->bhe", ds, k)
    if mistake == "dq_drop_sample":
        part = part[1:]
    dq = part.sum(0)
    dkv = torch.stack([dk.reshape(B, T, -1), dv.reshape(B, T, -1)], 2).reshape(B * T, -1)
    return dkv, dq


def loss_emul(logits, n_valid, mode, labels=None, targets=None, eps=0.0, num_choices=1, mistake=None):
    z = logits[:, :n_valid].float()
    if mode == HINGE:
        zg = z[:, 0].view(-1, num_choices)
        pos = zg.gather(1, labels.long()[:, None])
        h = zg - pos if mistake == "hinge_no_constant" else 1 + zg - pos
        return h.clamp_min(0).sum(1)
    lse = torch.logsumexp(z, 1, keepdim=True)
    t = targets[:, :n_valid].float()
    row = (t * (lse - z)).sum(1)
    if mistake == "eps_on_soft":
        row = (1 - eps) * row + eps * (lse[:, 0] - z.mean(1)) * t.sum(1)
    return row


def _pool_case(B=3, T=12, H=2, pad=True, q_std=0.5, seed=0):
    g = torch.Generator().manual_seed(seed)
    d = 64 * H
    kv = torch.randn(B * T, 2 * d, generator=g).bfloat16()
    q = q_std * torch.randn(H, 64, generator=g)
    kp = None
    if pad:
        kp = torch.zeros(B, T, dtype=torch.uint8)
        for b in range(B):
            kp[b, T - b:] = 1 if b else 0
    dout = torch.randn(B, d, generator=g).bfloat16()
    return kv, q, kp, dout


def test_pool_emulation_within_bounds():
    kv, q, kp, dout = _pool_case()
    out, lse, bo, bl = pool_fwd_ref(kv, q, kp, 3, 12)
    eo, el = pool_fwd_emul(kv, q, kp, 3, 12)
    assert excess(eo, out, bo) <= 1 and excess(el, lse, bl) <= 1
    dkv, dq, bkv, bdq = pool_bwd_ref(kv, q, kp, dout, 3, 12)
    ekv, edq = pool_bwd_emul(kv, q, kp, dout, 3, 12)
    assert excess(ekv, dkv, bkv) <= 1 and excess(edq, dq, bdq) <= 1


@pytest.mark.parametrize("mistake", ["padded_key", "q_scaled", "neighbour_head", "k_bias"])
def test_pool_forward_mistakes_exceed_bounds(mistake):
    kv, q, kp, _ = _pool_case()
    out, lse, bo, bl = pool_fwd_ref(kv, q, kp, 3, 12)
    eo, el = pool_fwd_emul(kv, q, kp, 3, 12, mistake=mistake)
    assert max(excess(eo, out, bo), excess(el, lse, bl)) > 1


def test_pool_cls_row_pooled_exceeds_bounds():
    """Pooling the CLS row: the features' row 0 joins the keys."""
    B, T = 3, 12
    kv, q, kp, _ = _pool_case(B=B, T=T + 1)
    kp = kp[:, 1:].contiguous()
    rest = kv.view(B, T + 1, -1)[:, 1:].reshape(B * T, -1)
    out, _, bo, _ = pool_fwd_ref(rest, q, kp, B, T)
    eo, _ = pool_fwd_emul(kv, q, torch.cat([torch.zeros(B, 1, dtype=torch.uint8), kp], 1), B, T + 1)
    assert excess(eo, out, bo) > 1


def test_pool_dq_dropped_sample_exceeds_bound():
    kv, q, kp, dout = _pool_case()
    _, dq, _, bdq = pool_bwd_ref(kv, q, kp, dout, 3, 12)
    _, edq = pool_bwd_emul(kv, q, kp, dout, 3, 12, mistake="dq_drop_sample")
    assert excess(edq, dq, bdq) > 1


def test_loss_emulation_and_mistakes():
    g = torch.Generator().manual_seed(4)
    z = 3 * torch.randn(6, 16, generator=g)
    t = torch.softmax(torch.randn(6, 11, generator=g), 1)
    r = loss_ref(z, 11, SOFT, targets=t)
    assert excess(loss_emul(z, 11, SOFT, targets=t), r["row_loss"], r["b_row_loss"]) <= 1
    assert excess(loss_emul(z, 11, SOFT, targets=t, eps=0.1, mistake="eps_on_soft"), r["row_loss"], r["b_row_loss"]) > 1
    zh = torch.randn(8, 8, generator=g)
    lab = torch.tensor([1, 3])
    r = loss_ref(zh, 1, HINGE, labels=lab, num_choices=4)
    assert excess(loss_emul(zh, 1, HINGE, labels=lab, num_choices=4), r["row_loss"], r["b_row_loss"]) <= 1
    assert excess(loss_emul(zh, 1, HINGE, labels=lab, num_choices=4, mistake="hinge_no_constant"), r["row_loss"],
                  r["b_row_loss"]) > 1


def test_loss_ref_matches_torch_criteria():
    g = torch.Generator().manual_seed(5)
    z = 2 * torch.randn(5, 9, generator=g)
    lab = torch.randint(0, 9, (5,), generator=g)
    r = loss_ref(z, 9, HARD, labels=lab, eps=0.1)
    assert torch.allclose(r["loss"], torch.nn.functional.cross_entropy(z.double(), lab, label_smoothing=0.1, reduction="sum"))
    tm = (torch.rand(5, 9, generator=g) < 0.4).double()
    r = loss_ref(z, 9, MULTI, targets=tm)
    assert torch.allclose(r["loss"], torch.nn.functional.binary_cross_entropy_with_logits(z.double(), tm, reduction="sum"))


# ------------------------------------------------------------------------------------------------------------------------------
# model host logic against the committed fixture
# ------------------------------------------------------------------------------------------------------------------------------
def _golden(golden_dir):
    import os
    return torch.load(os.path.join(golden_dir, "classify.pt"), weights_only=False)


def _model(case, **over):
    from one_peace_b200.one_peace.one_peace_classify import OnePeaceClassifyConfig, OnePeaceClassifyModel
    from one_peace_b200.one_peace.hub_interface import _Dictionary
    from one_peace_b200.unify_model_config import one_peace_4b_encoder_config
    c = sc.CLASSIFY_TINY
    cfg = OnePeaceClassifyConfig(attn_pooling=True, use_pooler=case["use_pooler"], use_image_features=case["use_image_features"])
    for k, v in over.items():
        setattr(cfg, k, v)
    cfg.encoder = one_peace_4b_encoder_config(c["layers"], c["embed_dim"], c["ffn"], c["heads"], 224)
    return OnePeaceClassifyModel(cfg, _Dictionary(), case.get("head_type"), case["num_classes"], case["use_two_images"])


def test_parameter_names_and_order_match_reference(golden_dir):
    gold = _golden(golden_dir)
    for name, rec in gold["cases"].items():
        m = _model(rec["case"])
        assert [n for n, _ in m.named_parameters()] == rec["param_order"], name


def test_pruning_per_head_type_matches_reference(golden_dir):
    gold = _golden(golden_dir)
    full = synth.make_state_dict(**sc.CLASSIFY_TINY, seed=0)
    for name, rec in gold["cases"].items():
        m = _model(rec["case"])
        sd = dict(full)
        m.upgrade_state_dict_named(sd, "")
        assert sorted(sd) == rec["upgraded_keys"], (name, sorted(set(sd) ^ set(rec["upgraded_keys"])))


@pytest.mark.parametrize("over,head", [(dict(attn_pooling=False), "audio"), (dict(pooler_dropout=0.1), "audio"), ({}, "val")])
def test_refusals(over, head):
    case = dict(use_pooler=False, use_image_features=False, num_classes=3, use_two_images=False, head_type=head)
    with pytest.raises(NotImplementedError):
        _model(case, **over)


def test_new_entry_points_reject_bad_arguments_without_a_gpu():
    import ctypes
    from one_peace_b200 import _lib
    lib = _lib.load()
    assert lib.opb_attn_pool_fwd(None, None, None, None, None, 1, 1, 256, None) == 1
    assert lib.opb_attn_pool_bwd(None, None, None, None, None, None, None, None, 1, 1, 256, None) == 1
    assert lib.opb_classify_loss(None, 8, 1, 1, 0, None, None, 0, ctypes.c_float(0.0), 1, None, None, None, None, None,
                                 None) == 1
    p = ctypes.c_void_p(16)                       # never dereferenced: the shape checks come first
    assert lib.opb_attn_pool_fwd(p, p, None, p, p, 1, 1, 100, None) == 1          # d % 64 != 0
    assert lib.opb_attn_pool_fwd(p, p, None, p, p, 1, 0, 256, None) == 1          # T < 1
    assert lib.opb_classify_loss(p, 8, 6, 2, 3, p, None, 0, ctypes.c_float(0.0), 4, p, p, p, p, p, None) == 1   # hinge, n_valid 2
