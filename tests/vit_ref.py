"""fp64 reference of the pooled OnePeaceViT head kernels (csrc/vit_head.cu) with per-element error bounds, an fp32 emulation of
their arithmetic, and the planted mistakes the bounds must catch.  The bounds are derived in DESIGN.md, "Vision
classification"; u = 2^-24 (fp32 unit roundoff), gamma(k) = k u / (1 - k u), and every sum is bounded for any summation order.

    forward   m = x[:, 1:].mean(1), y = bf16(LayerNorm(m) * gamma + beta), mean / rstd = LayerNorm statistics of m
    backward  dgamma / dbeta summed over the samples; dx[b, s] = LayerNorm adjoint of row b / (S - 1) for s >= 1, 0 for s = 0
The backward reference takes the kernel's own m, mean and rstd as exact inputs, as the kernel does."""
import torch

U = 2.0 ** -24
U_BF16 = 2.0 ** -8
MISTAKES_FWD = ("cls_included", "divide_by_S", "ln_batch_axis")
MISTAKES_BWD = ("dgamma_missing_term", "cls_grad_nonzero", "divide_by_S")


def gam(k):
    return k * U / (1.0 - k * U)


def head_fwd(x, gamma, beta, eps):
    """x [B, S, d] -> dict of fp64 values m, mean, rstd, y and their bounds b_m, b_mean, b_rstd, b_y."""
    x, g, be = x.double(), gamma.double(), beta.double()
    B, S, d = x.shape
    n = S - 1
    xp = x[:, 1:]
    m = xp.sum(1) / n
    A = xp.abs().sum(1)
    b_m = gam(n + 1) * A / n
    mu = m.mean(1)
    b_mu = (b_m.sum(1) + gam(d + 1) * m.abs().sum(1)) / d
    t = m - mu[:, None]
    var = (t * t).mean(1)
    dt = b_m + b_mu[:, None] + U * t.abs()
    b_var = ((2 * t.abs() * dt + dt * dt).sum(1) + gam(d + 2) * (t * t).sum(1)) / d
    rstd = 1.0 / torch.sqrt(var + eps)
    b_rstd = rstd * (0.5 * (b_var + U * (var + eps)) / (var + eps) + 4 * U)
    xh = t * rstd[:, None]
    y = xh * g + be
    pre = rstd[:, None] * g.abs() * dt + t.abs() * g.abs() * b_rstd[:, None] + 4 * U * (xh.abs() * g.abs() + be.abs())
    b_y = pre + U_BF16 * (y.abs() + pre)
    return dict(m=m, mean=mu, rstd=rstd, y=y, b_m=b_m, b_mean=b_mu + U * mu.abs(), b_rstd=b_rstd, b_y=b_y)


def head_bwd(dy, m, mean, rstd, gamma, S):
    """dy fp32 [B, d] and the forward's fp32 m / mean / rstd -> dict of fp64 dx [B, S, d], dgamma, dbeta and bounds."""
    dy, m, mu, rs, g = dy.double(), m.double(), mean.double(), rstd.double(), gamma.double()
    B, d = dy.shape
    n = S - 1
    xh = (m - mu[:, None]) * rs[:, None]
    gx = dy * g
    mean_g = gx.mean(1, keepdim=True)
    mean_gx = (gx * xh).mean(1, keepdim=True)
    dm = rs[:, None] * (gx - mean_g - xh * mean_gx)
    b_mg = gam(d + 3) * gx.abs().sum(1, keepdim=True) / d
    b_mgx = gam(d + 5) * (gx * xh).abs().sum(1, keepdim=True) / d
    b_dm = rs[:, None] * (b_mg + xh.abs() * b_mgx + 6 * U * (gx.abs() + mean_g.abs() + (xh * mean_gx).abs()))
    g_row = dm / n
    b_row = (b_dm + 2 * U * dm.abs()) / n
    dx = torch.zeros(B, S, d, dtype=torch.float64, device=dy.device)
    dx[:, 1:] = g_row[:, None, :]
    b_dx = torch.zeros(B, S, d, dtype=torch.float64, device=dy.device)
    b_dx[:, 1:] = b_row[:, None, :]
    dgamma = (dy * xh).sum(0)
    dbeta = dy.sum(0)
    return dict(dx=dx, dgamma=dgamma, dbeta=dbeta, b_dx=b_dx, b_dgamma=gam(B + 4) * (dy * xh).abs().sum(0),
                b_dbeta=gam(B) * dy.abs().sum(0))


def excess(got, want, bound):
    """max |got - want| / bound over the elements (an exact match where the bound is 0 counts as 0)."""
    err = (got.double() - want.double()).abs()
    b = bound.double()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / b.clamp_min(1e-300))
    return ratio.max().item()


def emulate_fwd(x, gamma, beta, eps, mistake=None):
    """fp32 evaluation of the forward kernels' arithmetic -> (y bf16, m, mean, rstd); `mistake` plants one error."""
    x = x.float()
    B, S, d = x.shape
    if mistake == "cls_included":
        m = x.sum(1) / S
    elif mistake == "divide_by_S":
        m = x[:, 1:].sum(1) / S
    else:
        m = x[:, 1:].sum(1) / (S - 1)
    axis = 0 if mistake == "ln_batch_axis" else 1
    mu = m.mean(axis, keepdim=True)
    var = ((m - mu) ** 2).mean(axis, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    y = ((m - mu) * rstd * gamma.float() + beta.float()).to(torch.bfloat16)
    if axis == 0:
        mu, rstd = m.mean(1, keepdim=True), torch.rsqrt(((m - m.mean(1, keepdim=True)) ** 2).mean(1, keepdim=True) + eps)
    return y, m, mu.view(B), rstd.view(B)


def emulate_bwd(dy, m, mean, rstd, gamma, S, mistake=None):
    """fp32 evaluation of the backward kernels' arithmetic -> (dx [B, S, d], dgamma, dbeta)."""
    dy, m, g = dy.float(), m.float(), gamma.float()
    B, d = dy.shape
    xh = (m - mean[:, None]) * rstd[:, None]
    gx = dy * g
    dm = rstd[:, None] * (gx - gx.mean(1, keepdim=True) - xh * (gx * xh).mean(1, keepdim=True))
    dx = torch.zeros(B, S, d, device=dy.device)
    dx[:, 1:] = (dm / (S if mistake == "divide_by_S" else S - 1))[:, None, :]
    if mistake == "cls_grad_nonzero":
        dx[:, 0] = dx[:, 1]
    terms = dy * xh
    dgamma = terms[1:].sum(0) if mistake == "dgamma_missing_term" else terms.sum(0)
    return dx, dgamma, dy.sum(0)
