"""fp64 reference of one fused Adan step (``opb_adan_multi_step``, csrc/adam.cu) on the operands the kernel reads, with a
first-order error bound for every output element, in the style of kernel_ref.py "Optimizer" (which this module reuses for
``f32_rel``, ``assert_within`` and ``bf16_param_check``).

Plain PyTorch on whatever device the inputs live on; nothing here calls the extension.

The kernel, per element in fp32, every operation correctly rounded on its own (``__fadd_rn`` ...; sqrtf is IEEE):
    x = g s;  d = first ? 0 : x - pre;  u = x + b2 d
    m' = b1 m + (1 - b1) x;  n' = b2 n + (1 - b2) d;  v' = b3 v + ((1 - b3) u) u
    den = sqrt(v') / sb3 + eps,  sb3 = sqrt(1 - b3^t)
    upd = (m' / bc1 + (b2 n') / bc2) / den,  bc1 = 1 - b1^t, bc2 = 1 - b2^t
    lw = lr wd;  no_prox: p' = p (1 - lw) + (-lr) upd;  proximal: p' = (p + (-lr) upd) / (1 + lw);  pre' = x
The reference evaluates this in fp64 with the hyperparameters as the user's Python doubles, so the bound pays for their
fp32 rounding: e_h = |fp32(h) - h| / |h| for h = b1, b2, b3, eps, lr, wd, bc1, bc2, sb3 and the grad scale s (computed, not
assumed), and for the kernel's 1 - b_i, formed from the already-rounded b_i (exact by Sterbenz for 0.5 <= b < 1):
e_ci = |(1 - fp32(b_i)) - (1 - b_i)| / (1 - b_i).  Bounds are absolute, first order, u = 2^-24:
``x``     dx = |g| |s| (e_s + u) + |g| ds   (ds: the error of a grad scale that was itself computed)
``d``     first: 0.  Else dx + u |d| (pre is read exactly as stored)
``u``     dx + b2 dd + |b2 d| (e_b2 + u) + u |u|
``m'``    |b1 m| (e_b1 + u) + (1 - b1) (|x| (e_c1 + u) + dx) + u |m'|
``n'``    |b2 n| (e_b2 + u) + (1 - b2) (|d| (e_c2 + u) + dd) + u |n'|
``v'``    |b3 v| (e_b3 + u) + (1 - b3) (u^2 (e_c3 + 2u) + 2 |u| du) + u v'
``sqrt``  sqrt(v') - sqrt(max(v' - dv, 0)) + u sqrt(v')   (the exact fall: finite where sqrt(v') ~ 0, |g| ~ eps)
``den``   dsqrt / sb3 + |sqrt(v') / sb3| (e_sb3 + u) + eps e_eps + u den
``q``     a = m' / bc1: dm / bc1 + |a| (e_bc1 + u);  b = b2 n' / bc2: b2 dn / bc2 + |b| (e_b2 + e_bc2 + 2u);  dq = da + db + u |q|
``upd``   dq / den + |upd| dden / den + u |upd|
``lr upd``  lr dupd + |lr upd| (e_lr + u)
``decay`` 1 -+ lw: lw (e_lr + e_wd + u) + u |decay|  (0 when wd = 0: the kernel's 1 -+ 0 is exact)
``p'``    no_prox: |p| ddecay + u |p decay| + dL + u |p'|;  proximal: (dL + u |p - L|) / decay + |p'| (ddecay / decay + u)
``pre'``  dx
bf16 parameters: with a master copy p16 must equal bf16_rn(master') bit for bit; without one, ``bf16_param_check``.
"""
import math
from types import SimpleNamespace

import numpy as np
import torch

from kernel_ref import U32, assert_within, bf16_param_check, f32_rel  # noqa: F401  (re-exported for the tests)

BETAS = (0.98, 0.92, 0.99)
EPS = 1e-8


def group_coefs(t, betas):
    """(bc1, bc2, sqrt(bc3)) in Python doubles for the group step t, as optim/adan.py passes them to the kernel"""
    b1, b2, b3 = betas
    return 1 - b1 ** t, 1 - b2 ** t, math.sqrt(1 - b3 ** t)


def _e_c(b):
    c = 1 - b
    return abs((1 - float(np.float32(b))) - c) / c


def adan_ref(p, g, m, n, v, pre, *, first, t, lr, wd, no_prox, betas=BETAS, eps=EPS, grad_scale=None, grad_scale_err=0.0):
    """fp64 Adan step on the operands the kernel reads (p: fp32 master or the parameter up-cast; g as stored; m, n, v, pre
    fp32; ``first``: bool tensor or Python bool, diff = 0 there); t the group step after this step; grad_scale a Python
    float (None = 1) with the absolute error ``grad_scale_err`` of its computed value.  Returns a namespace with m, n, v,
    pre, p (the fp32 p' of the master copy or an fp32 parameter), upd and ``<name>_err`` for each."""
    b1, b2, b3 = betas
    for b in betas:
        assert 0.5 <= b < 1, "1 - fp32(b) is exact only for 0.5 <= b < 1"
    u = U32
    P, G, M0, N0, V0, PRE = (x.double() for x in (p, g, m, n, v, pre))
    first = torch.as_tensor(first, device=P.device).expand_as(P)
    s = 1.0 if grad_scale is None else float(grad_scale)
    c1, c2, c3 = 1 - b1, 1 - b2, 1 - b3
    X = G * s
    dX = G.abs() * (abs(s) * (f32_rel(s) + u) + grad_scale_err)
    D = torch.where(first, torch.zeros_like(X), X - torch.where(first, torch.zeros_like(PRE), PRE))
    dD = torch.where(first, torch.zeros_like(X), dX + u * D.abs())
    Uu = X + b2 * D
    dU = dX + b2 * dD + (b2 * D).abs() * (f32_rel(b2) + u) + u * Uu.abs()
    Mn = b1 * M0 + c1 * X
    dM = (b1 * M0).abs() * (f32_rel(b1) + u) + c1 * (X.abs() * (_e_c(b1) + u) + dX) + u * Mn.abs()
    Nn = b2 * N0 + c2 * D
    dN = (b2 * N0).abs() * (f32_rel(b2) + u) + c2 * (D.abs() * (_e_c(b2) + u) + dD) + u * Nn.abs()
    Vn = b3 * V0 + c3 * Uu * Uu
    dV = (b3 * V0).abs() * (f32_rel(b3) + u) + c3 * (Uu * Uu * (_e_c(b3) + 2 * u) + 2 * Uu.abs() * dU) + u * Vn.abs()
    R = Vn.sqrt()
    dR = R - (Vn - dV).clamp_min(0.0).sqrt() + u * R
    bc1, bc2, sb3 = group_coefs(t, betas)
    S = R / sb3
    dS = dR / sb3 + S.abs() * (f32_rel(sb3) + u)
    Den = S + eps
    dDen = dS + eps * f32_rel(eps) + u * Den
    A = Mn / bc1
    dA = dM / bc1 + A.abs() * (f32_rel(bc1) + u)
    B = b2 * Nn / bc2
    dB = b2 * dN / bc2 + B.abs() * (f32_rel(b2) + f32_rel(bc2) + 2 * u)
    Q = A + B
    dQ = dA + dB + u * Q.abs()
    Upd = Q / Den
    dUpd = dQ / Den + Upd.abs() * dDen / Den + u * Upd.abs()
    L = lr * Upd
    dL = lr * dUpd + L.abs() * (f32_rel(lr) + u)
    lw = lr * wd
    lw32 = float(np.float32(lr)) * float(np.float32(wd))
    if no_prox:
        decay = 1 - lw
        d_decay = abs(lw) * (f32_rel(lr) + f32_rel(wd) + u) + (u * abs(decay) if lw32 != 0 else 0.0)
        P1 = P * decay
        Pn = P1 - L
        dPn = P.abs() * d_decay + u * P1.abs() + dL + u * Pn.abs()
    else:
        decay = 1 + lw
        d_decay = abs(lw) * (f32_rel(lr) + f32_rel(wd) + u) + (u * abs(decay) if lw32 != 0 else 0.0)
        P1 = P - L
        Pn = P1 / decay
        dPn = (dL + u * P1.abs()) / decay + Pn.abs() * (d_decay / decay + u)
    return SimpleNamespace(m=Mn, m_err=dM, n=Nn, n_err=dN, v=Vn, v_err=dV, pre=X, pre_err=dX, p=Pn, p_err=dPn, upd=Upd,
                           upd_err=dUpd)


def sample_operands(count, t, seed, betas=BETAS, device="cpu"):
    """fp32 operands of one step at group step t: N(0, 0.3) gradients with every 4th in a band 1e-9 <= |g| <= 1e-6
    (sqrt(v) / sqrt(bc3) comparable to eps), every 16th gradient and state zero; m, n, v preset as t - 1 steps leave them;
    pre a previous gradient of the same law.  -> dict p, g, m, n, v, pre"""
    gen = torch.Generator(device=device).manual_seed(seed)
    e = torch.arange(count, device=device)
    band, zero = e % 4 == 1, e % 16 == 3
    b1, b2, b3 = betas

    def grad():
        x = torch.randn(count, device=device, generator=gen) * 0.3
        small = 10.0 ** (-9 + 3 * torch.rand(count, device=device, generator=gen))
        return torch.where(band, torch.sign(x) * small, x)
    g, pre = grad(), grad()
    sc = torch.where(band, 1e-7, 0.3)
    h = [torch.randn(count, device=device, generator=gen) * sc for _ in range(3)]
    td = float(t - 1)
    m = ((1 - b1 ** td) * h[0]).float()
    n = ((1 - b2 ** td) * h[1] * 0.3).float()
    v = ((1 - b3 ** td) * h[2] * h[2]).float()
    g, m, n, v, pre = (torch.where(zero, 0.0, x) for x in (g, m, n, v, pre))
    p = torch.randn(count, device=device, generator=gen)
    return dict(p=p, g=g, m=m, n=n, v=v, pre=pre)
