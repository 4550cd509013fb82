"""fp64 references of the segmentation kernels (csrc/seg.cu), written as direct sums, and the per-element bounds of the
kernels' fp32 / bf16 arithmetic.

  dwconv_gelu_ref : per-level depthwise 3x3 conv with zero padding + bias + exact GELU over token rows
  out_map_ref     : scale * (extra + c_l + bilinear(x, align_corners=False)) + shift, fp32 NCHW
"""
import math

import torch

U32 = 2.0 ** -24        # fp32 unit round-off
U16 = 2.0 ** -8         # bf16 unit round-off (8 significant bits, round to nearest)


def _levels(rows, shapes, B):
    """token rows [B * T, C] -> list of [B, C, H, W] level grids."""
    T = sum(h * w for h, w in shapes)
    x = rows.view(B, T, -1)
    out, s = [], 0
    for h, w in shapes:
        out.append(x[:, s:s + h * w].transpose(1, 2).reshape(B, -1, h, w))
        s += h * w
    return out


def _rows(grids):
    return torch.cat([g.flatten(2).transpose(1, 2) for g in grids], 1).reshape(-1, grids[0].shape[1])


def dwconv_terms(x, w, shapes, B):
    """-> per level the nine shifted products [9, B, C, H, W] (zero outside the level) of x rows and w [C, 1, 3, 3]."""
    out = []
    for g in _levels(x.double(), shapes, B):
        _, C, H, W = g.shape
        p = torch.zeros(g.shape[0], C, H + 2, W + 2, dtype=torch.float64)
        p[:, :, 1:-1, 1:-1] = g
        out.append(torch.stack([p[:, :, ky:ky + H, kx:kx + W] * w[:, 0, ky, kx].double().view(1, C, 1, 1)
                                for ky in range(3) for kx in range(3)]))
    return out


def dwconv_gelu_ref(x, w, b, shapes, B):
    """-> (y fp64 [B * T, C], pre-activation fp64, A = sum of |products| + |bias|, both [B * T, C])."""
    pre, absum = [], []
    for t in dwconv_terms(x, w, shapes, B):
        bb = b.double().view(1, -1, 1, 1)
        pre.append(t.sum(0) + bb)
        absum.append(t.abs().sum(0) + bb.abs())
    z, a = _rows(pre), _rows(absum)
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0))), z, a


def dwconv_gelu_bound(y, z, a):
    """|kernel - ref| bound: ten fp32 roundings of the sum (|z| error <= 10 u32 A), gelu' <= 1.13, the erf approximation
    (1.5e-7 absolute on erf, times |z| / 2), the fp32 GELU arithmetic (4 u32 |y|), then one bf16 rounding."""
    g = 1.13 * 10 * U32 * a + 0.5 * z.abs() * 1.5e-7 + 4 * U32 * y.abs()
    return U16 * (y.abs() + g) + g + 1e-30


def bilinear_ref(x, H, W):
    """x [B, C, h, w] -> [B, C, H, W], align_corners=False, by direct weights (torch's source index clamped at 0)."""
    def axis(n_in, n_out):
        s = ((torch.arange(n_out, dtype=torch.float64) + 0.5) * (n_in / n_out) - 0.5).clamp_min(0.0)
        i0 = s.floor().long().clamp_max(n_in - 1)
        i1 = (i0 + 1).clamp_max(n_in - 1)
        return i0, i1, s - i0
    y0, y1, fy = axis(x.shape[2], H)
    x0, x1, fx = axis(x.shape[3], W)
    xd = x.double()
    top = xd[:, :, y0][:, :, :, x0] * (1 - fx) + xd[:, :, y0][:, :, :, x1] * fx
    bot = xd[:, :, y1][:, :, :, x0] * (1 - fx) + xd[:, :, y1][:, :, :, x1] * fx
    fy = fy.view(-1, 1)
    return top * (1 - fy) + bot * fy, (xd.abs().amax(dim=(2, 3), keepdim=True)).expand(-1, -1, H, W)


def convt_ref(x, w, b):
    """ConvTranspose2d(k=2, s=2) by its pixel-shuffle sum: x [B, Ci, h, w], w [Ci, Co, 2, 2] -> [B, Co, 2h, 2w]."""
    B, _, h, wd = x.shape
    y = torch.einsum("bihw,iokl->bohkwl", x.double(), w.double()).reshape(B, w.shape[1], 2 * h, 2 * wd)
    return y + b.double().view(1, -1, 1, 1)


def out_map_ref(c, x, scale, shift, extra=None):
    """c [B, C, H, W], x [B, C, g, g], extra [B, C, H, W] or None (all fp64-exact inputs) -> (f fp64, bound)."""
    H, W = c.shape[2:]
    up, xmax = bilinear_ref(x, H, W)
    v = c.double() + up
    mag = c.double().abs() + 2 * xmax
    if extra is not None:
        v = v + extra.double()
        mag = mag + extra.double().abs()
    s, t = scale.double().view(1, -1, 1, 1), shift.double().view(1, -1, 1, 1)
    f = v * s + t
    return f, 12 * U32 * (mag * s.abs() + t.abs()) + 1e-30
