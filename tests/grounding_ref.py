"""fp64 reference of the visual-grounding kernels (csrc/grounding.cu) with per-element first-order error bounds for their fp32
results, and an fp32 emulation of the kernel arithmetic into which the host tests plant mistakes.

refcoco(z, t, ns) restates criterions/refcoco_loss.py:36-46 in closed form (p = sigmoid(z), L1 / nsentences, GIoU over the
valid rows, NaN when none is valid) together with its gradient d loss / d z in the form torch's autograd produces (tests
check both against torchvision's generalized_box_iou and torch.autograd).  Every rounding step of the fp32 evaluation is
tracked: a subtraction or addition contributes u (|a| + |b|), a product or quotient u |result|, the sigmoid 4 u p, and the
bound of an output is the sum over steps of |d output / d step| times that, taken by autograd through the fp64 graph, plus
the flip terms of sign(p - t) near a tie.  Rows whose validity could flip under the fp32 error of p are reported so that the
tests can leave them out.
"""
import torch

U32 = 2.0 ** -24


class _Tape:
    def __init__(self):
        self.vals, self.mags = [], []

    def rec(self, v, mag):
        self.vals.append(v)
        self.mags.append(mag.detach())
        return v

    def sub(self, a, b):
        return self.rec(a - b, a.abs() + b.abs())

    def add(self, a, b):
        return self.rec(a + b, a.abs() + b.abs())

    def mul(self, a, b):
        v = a * b
        return self.rec(v, v.abs())

    def div(self, a, b):
        v = a / b
        return self.rec(v, v.abs())


def _dmax(a, b):
    return torch.where(a > b, 1.0, torch.where(a == b, 0.5, 0.0)).to(a.dtype)


def _dmin(a, b):
    return torch.where(a < b, 1.0, torch.where(a == b, 0.5, 0.0)).to(a.dtype)


def _giou_parts(tp, p, t):
    """(giou [N], d giou / d p [N, 4]) of every row, recorded on the tape (the kernel's operation structure)."""
    P = [p[:, j] for j in range(4)]
    T = [t[:, j] for j in range(4)]
    a1 = tp.mul(tp.sub(P[2], P[0]), tp.sub(P[3], P[1]))
    a2 = tp.mul(tp.sub(T[2], T[0]), tp.sub(T[3], T[1]))
    wr = tp.sub(torch.minimum(P[2], T[2]), torch.maximum(P[0], T[0]))
    hr = tp.sub(torch.minimum(P[3], T[3]), torch.maximum(P[1], T[1]))
    w, h = wr.clamp(min=0), hr.clamp(min=0)
    inter = tp.mul(w, h)
    uni = tp.sub(tp.add(a1, a2), inter)
    wcr = tp.sub(torch.maximum(P[2], T[2]), torch.minimum(P[0], T[0]))
    hcr = tp.sub(torch.maximum(P[3], T[3]), torch.minimum(P[1], T[1]))
    wc, hc = wcr.clamp(min=0), hcr.clamp(min=0)
    c = tp.mul(wc, hc)
    giou = tp.sub(tp.div(inter, uni), tp.div(tp.sub(c, uni), c))
    d_uni = tp.add(-tp.div(inter, tp.mul(uni, uni)), tp.div(torch.ones_like(c), c))
    d_inter = tp.sub(tp.div(torch.ones_like(uni), uni), d_uni)
    d_c = -tp.div(uni, tp.mul(c, c))
    ph, pw = tp.sub(P[3], P[1]), tp.sub(P[2], P[0])
    g = [-tp.mul(d_uni, ph), -tp.mul(d_uni, pw), tp.mul(d_uni, ph), tp.mul(d_uni, pw)]
    dw = torch.where(wr >= 0, tp.mul(d_inter, h), torch.zeros_like(wr))
    dh = torch.where(hr >= 0, tp.mul(d_inter, w), torch.zeros_like(hr))
    dwc = torch.where(wcr >= 0, tp.mul(d_c, hc), torch.zeros_like(wcr))
    dhc = torch.where(hcr >= 0, tp.mul(d_c, wc), torch.zeros_like(hcr))
    g[2] = tp.add(tp.add(g[2], tp.mul(dw, _dmin(P[2], T[2]))), tp.mul(dwc, _dmax(P[2], T[2])))
    g[0] = tp.sub(tp.sub(g[0], tp.mul(dw, _dmax(P[0], T[0]))), tp.mul(dwc, _dmin(P[0], T[0])))
    g[3] = tp.add(tp.add(g[3], tp.mul(dh, _dmin(P[3], T[3]))), tp.mul(dhc, _dmax(P[3], T[3])))
    g[1] = tp.sub(tp.sub(g[1], tp.mul(dh, _dmax(P[1], T[1]))), tp.mul(dhc, _dmin(P[1], T[1])))
    return giou, torch.stack(g, 1)


def refcoco(z, t, ns):
    """z [B, 4] (the logits as the kernel sees them, fp32 values), t [B, 4], ns -> dict of fp64 values and bounds:
    p, valid (bool), giou, loss, l1, n_valid, dlogits, and b_p, b_giou, b_loss, b_l1, b_dlogits, unsure (rows whose validity
    could flip)."""
    z = z.detach().double()
    t = t.detach().double().clone().requires_grad_(True)       # so that every step of the target's area is on the tape
    B = z.shape[0]
    tp = _Tape()
    zl = z.clone().requires_grad_(True)
    p = torch.sigmoid(zl)
    tp.rec(p, 4.0 * p.abs())
    valid = ((p[:, 0] < p[:, 2]) & (p[:, 1] < p[:, 3])).detach()
    giou, g = _giou_parts(tp, p, t)
    nv = int(valid.sum())
    absd = [tp.rec((p[:, j] - t[:, j]).abs(), (p[:, j].abs() + t[:, j].abs())) for j in range(4)]
    l1row = tp.add(tp.add(tp.add(absd[0], absd[1]), absd[2]), absd[3])
    l1sum = l1row.sum()
    # summation of B terms in any order: gamma_B sum |term|
    l1 = tp.div(l1sum, torch.tensor(float(ns), dtype=torch.float64))
    one_minus = tp.sub(torch.ones_like(giou), giou)
    gsum = torch.where(valid, one_minus, 0.0).sum()
    gpart = tp.div(gsum, torch.tensor(float(max(nv, 1)), dtype=torch.float64))
    loss = tp.add(l1, gpart) if nv > 0 else l1 + float("nan")
    sign = torch.sign((p - t).detach())
    t = t.detach()
    s = 1.0 / ns
    q = (p * (1.0 - p)).detach()
    gterm = torch.where(valid[:, None], tp.div(-g, torch.tensor(float(max(nv, 1)), dtype=torch.float64)), 0.0)
    dp = tp.add(sign * s, gterm)
    dz = tp.mul(tp.mul(dp, tp.sub(torch.ones_like(p), p)), p)
    out = dict(p=p.detach(), valid=valid, giou=giou.detach(), loss=loss.detach(), l1=l1.detach(), n_valid=nv,
               dlogits=dz.detach())

    def bound(y):
        """first-order bound of a scalar-per-row quantity y [B] (rows independent) or a scalar."""
        gs = torch.autograd.grad(y.sum(), tp.vals, retain_graph=True, allow_unused=True)
        b = torch.zeros_like(y.detach())
        for gk, mk in zip(gs, tp.mags):
            if gk is None:
                continue
            c = torch.nan_to_num(gk.abs() * mk, nan=0.0, posinf=0.0)    # 0 * inf of a row whose value is not finite
            if b.dim() == 0:
                c = c.sum()
            elif c.dim() == 2:
                c = c.sum(1)
            b = b + c
        return U32 * b

    b_p = 4.0 * U32 * p.detach()
    out["b_p"] = b_p
    out["b_giou"] = 2.0 * bound(giou) + 1e-30
    gam = (B * 4 + 4) * U32
    out["b_l1"] = 2.0 * bound(l1) + gam * l1.detach().abs()
    if nv > 0:
        out["b_loss"] = 2.0 * bound(loss) + gam * l1.detach().abs() + (nv + 2) * U32 * gpart.detach().abs()
    else:
        out["b_loss"] = torch.tensor(float("nan"), dtype=torch.float64)
    bd = []
    for j in range(4):
        bd.append(bound(dz[:, j]))
    b_dz = torch.stack(bd, 1) * 2.0 + 1e-30
    # sign(p - t) may differ in fp32 when |p - t| is within the error of p
    near = (p.detach() - t).abs() <= 2 * b_p
    b_dz = b_dz + near.double() * 2.0 * s * q
    out["b_dlogits"] = b_dz
    gap = torch.minimum(p[:, 2] - p[:, 0], p[:, 3] - p[:, 1]).detach().abs()
    out["unsure"] = (gap <= 4 * b_p.max(1).values) & (gap != 0)
    return out


def refcoco_autograd(z, t, ns):
    """The reference's own expression in fp64 through torchvision and torch.autograd -> (loss, dlogits, per-row giou, valid)."""
    from torchvision.ops import generalized_box_iou
    zl = z.detach().double().clone().requires_grad_(True)
    t = t.detach().double()
    p = zl.sigmoid()
    loss = torch.nn.functional.l1_loss(p, t, reduction="sum") / ns
    valid = (p[:, :2] < p[:, 2:]).all(1)
    ious = torch.diag(generalized_box_iou(p[valid], t[valid]))
    loss = loss + (1 - ious).mean()
    loss.backward()
    with torch.no_grad():
        giou_all = torch.diag(generalized_box_iou(p, t))
    return loss.detach(), zl.grad, giou_all, valid


def emulate(z, t, ns, mistake=None):
    """The kernel's arithmetic in fp32 torch ops -> (p, valid, giou, loss, dlogits).  mistake plants one error:
    'nvalid_as_B', 'valid_le', 'no_sigmoid_grad', 'unclamped_enclosing', 'l1_sign', 'invalid_giou_grad'."""
    z = z.float()
    t = t.float()
    B = z.shape[0]
    p = 1.0 / (1.0 + torch.exp(-z))
    if mistake == "valid_le":
        valid = (p[:, 0] <= p[:, 2]) & (p[:, 1] <= p[:, 3])
    else:
        valid = (p[:, 0] < p[:, 2]) & (p[:, 1] < p[:, 3])
    P = [p[:, j] for j in range(4)]
    T = [t[:, j] for j in range(4)]
    a1 = (P[2] - P[0]) * (P[3] - P[1])
    a2 = (T[2] - T[0]) * (T[3] - T[1])
    wr = torch.minimum(P[2], T[2]) - torch.maximum(P[0], T[0])
    hr = torch.minimum(P[3], T[3]) - torch.maximum(P[1], T[1])
    w, h = wr.clamp(min=0), hr.clamp(min=0)
    inter = w * h
    uni = a1 + a2 - inter
    wcr = torch.maximum(P[2], T[2]) - torch.minimum(P[0], T[0])
    hcr = torch.maximum(P[3], T[3]) - torch.minimum(P[1], T[1])
    if mistake == "unclamped_enclosing":
        wc, hc = wcr, hcr
    else:
        wc, hc = wcr.clamp(min=0), hcr.clamp(min=0)
    c = wc * hc
    giou = inter / uni - (c - uni) / c
    nv = int(valid.sum())
    l1 = (p - t).abs().sum() / ns
    loss = l1 + ((1 - giou)[valid].sum() / nv if nv > 0 else float("nan"))
    d_uni = -inter / (uni * uni) + 1.0 / c
    d_inter = 1.0 / uni - d_uni
    d_c = -uni / (c * c)
    g = torch.stack([-d_uni * (P[3] - P[1]), -d_uni * (P[2] - P[0]), d_uni * (P[3] - P[1]), d_uni * (P[2] - P[0])], 1)
    dw = torch.where(wr >= 0, d_inter * h, 0.0)
    dh = torch.where(hr >= 0, d_inter * w, 0.0)
    dwc = torch.where(wcr >= 0, d_c * hc, 0.0)
    dhc = torch.where(hcr >= 0, d_c * wc, 0.0)
    g[:, 2] += dw * _dmin(P[2], T[2]).float() + dwc * _dmax(P[2], T[2]).float()
    g[:, 0] -= dw * _dmax(P[0], T[0]).float() + dwc * _dmin(P[0], T[0]).float()
    g[:, 3] += dh * _dmin(P[3], T[3]).float() + dhc * _dmax(P[3], T[3]).float()
    g[:, 1] -= dh * _dmax(P[1], T[1]).float() + dhc * _dmin(P[1], T[1]).float()
    sign = torch.sign(p - t)
    if mistake == "l1_sign":
        sign = -sign
    denom = B if mistake == "nvalid_as_B" else max(nv, 1)
    gate = torch.ones_like(valid) if mistake == "invalid_giou_grad" else valid
    dp = sign / ns + torch.where(gate[:, None], -g / denom, 0.0)
    dz = dp if mistake == "no_sigmoid_grad" else dp * (1.0 - p) * p
    return p, valid, giou, torch.as_tensor(loss, dtype=torch.float32), dz


def iou_hits(hyps, refs):
    """metrics/iou_acc.py:20-32 on fp32 tensors with torch's own elementwise ops (each rounded on its own) -> bool [n]."""
    i0 = torch.where(hyps[:, 0] < refs[:, 0], refs[:, 0], hyps[:, 0])
    i1 = torch.where(hyps[:, 1] < refs[:, 1], refs[:, 1], hyps[:, 1])
    i2 = torch.where(hyps[:, 2] < refs[:, 2], hyps[:, 2], refs[:, 2])
    i3 = torch.where(hyps[:, 3] < refs[:, 3], hyps[:, 3], refs[:, 3])
    ap = (hyps[:, 2] - hyps[:, 0]) * (hyps[:, 3] - hyps[:, 1])
    at = (refs[:, 2] - refs[:, 0]) * (refs[:, 3] - refs[:, 1])
    iw, ih = i2 - i0, i3 - i1
    ai = iw * ih
    iou = ai / (ap + at - ai)
    return (iou >= 0.5) & (iw > 0) & (ih > 0)


def excess(got, want, bound):
    """max over elements of |got - want| / bound; a finiteness mismatch counts as infinite, matching non-finite values as 0."""
    got, want, bound = got.double(), want.double(), bound.double().expand_as(want)
    fin = torch.isfinite(want) & torch.isfinite(got)
    mism = torch.isfinite(want) != torch.isfinite(got)
    if mism.any():
        return float("inf")
    if not fin.any():
        return 0.0
    return ((got - want).abs()[fin] / bound[fin]).max().item()
