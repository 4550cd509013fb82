"""fp64 references and error bounds of the detection backbone's two kernels (DESIGN.md, "Object detection backbone").

opb_relpos_decomp_proj: each term is a sum of 64 fp32 products of q_c = 8 * bf16 (exact) and R_c (fp32), accumulated by
FMA in channel order, so |got - ref| <= g(65) * 8 * sum_c |q_c R_c| with g(n) = n u / (1 - n u), u = 2^-24.

opb_attention_decomp_fwd: the logit is ((q.k + b) + rel_h) + rel_w in fp32.  Its error is the LUT kernel's e_ij (TAU times
sum |q||k|, plus the exponent / lse terms kernel_ref.attention_ref adds) plus the two terms' errors (the bound above) and
u times the magnitude of each of the two extra fp32 sums.  The lse / out / ln_stats formulas of kernel_ref.attention_ref
then apply unchanged with the larger e_ij.
"""
from types import SimpleNamespace

import torch

from kernel_ref import C_EXP, LSE_REL, TAU, U32, heads_to_rows, split_qkv

Q_UNSCALE = 8.0
G65 = 65 * U32 / (1 - 65 * U32)


def proj_ref(qkv, rel_pos_h, rel_pos_w, pos_y, pos_x, B, S, H, kh, kw):
    """-> (rel_h, err_h, rel_w, err_w) fp64, [B, H, S, k]"""
    q, _, _ = split_qkv(qkv, B, S, H)
    q = Q_UNSCALE * q
    out = []
    for table, pos, k in ((rel_pos_h, pos_y, kh), (rel_pos_w, pos_x, kw)):
        idx = pos.long()[:, None] - torch.arange(k, device=pos.device)[None, :] + k - 1       # [S, k]
        R = table.double()[idx]                                                               # [S, k, 64]
        out.append(torch.einsum("bhsc,skc->bhsk", q, R))
        out.append(G65 * torch.einsum("bhsc,skc->bhsk", q.abs(), R.abs()))
    return out


def decomp_attention_ref(qkv, bias, rel_h, err_h, rel_w, err_w, key_y, key_x, B, S, H):
    """kernel_ref.attention_ref for the decomposed logits.  bias fp32 [H, S, S] (the LUT values); rel_* [B, H, S, k] and
    their bounds from proj_ref (or exact values with zero bounds)."""
    q, k, v = split_qkv(qkv, B, S, H)
    ky, kx = key_y.long(), key_x.long()
    th, tw = rel_h.double()[..., ky], rel_w.double()[..., kx]            # [B, H, S, S]
    s0 = q @ k.transpose(-1, -2) + bias.double()[None]
    s = s0 + th + tw
    e = TAU * (q.abs() @ k.abs().transpose(-1, -2)) + err_h.double()[..., ky] + err_w.double()[..., kx]
    e = e + U32 * ((s0 + th).abs() + s.abs())
    lse = torch.logsumexp(s, -1)
    p = (s - lse[..., None]).exp()
    e = e + C_EXP * (1 + s.abs() + lse.abs()[..., None])
    pe = p * e
    dlse = pe.sum(-1) + LSE_REL * (1 + lse.abs())
    o = p @ v
    pv = p @ v.abs()
    w = pe + p * dlse[..., None]
    oerr = (2.0 ** -8 + TAU) * pv + w @ v.abs() + w.sum(-1, keepdim=True) * o.abs()
    st = torch.stack([o.sum(-1), (o * o).sum(-1)], -1)
    st_err = torch.stack([oerr.sum(-1) + TAU * o.abs().sum(-1),
                          (2 * o.abs() * oerr + oerr * oerr).sum(-1) + TAU * (o * o).sum(-1)], -1)
    to_rec = lambda t: t.permute(1, 0, 2, 3).reshape(H, B * S, 2)
    return SimpleNamespace(out=heads_to_rows(o, B, S, H), out_err=heads_to_rows(oerr, B, S, H), lse=lse, dlse=dlse,
                           stats=to_rec(st), stats_err=to_rec(st_err))


def proj_emulate_fp32(q_bf16, table, pos, k):
    """fp32 emulation of the projection kernel: products of the (exact) unscaled q and the table, FMA-accumulated over the
    64 channels in order (each step rounded to fp32).  q_bf16 [N, 64] -> [N, k]."""
    q = q_bf16.float() * Q_UNSCALE
    idx = pos.long()[:, None] - torch.arange(k)[None, :] + k - 1
    R = table.float()[idx]                          # [N, k, 64]
    acc = torch.zeros(q.shape[0], k, dtype=torch.float32)
    for c in range(64):
        acc = (acc.double() + q[:, None, c].double() * R[:, :, c].double()).float()      # fma: one rounding per step
    return acc
