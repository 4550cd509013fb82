"""fp64 references of the GEMM epilogues (csrc/gemm_wgmma.cu), of the contrastive-head reductions (csrc/infonce.cu) and of
the attention forward and backward (csrc/attention.cu, csrc/attention_bwd.cu), with an error bound for every output
element, and NaN-canary output buffers.

Plain PyTorch on whatever device the inputs live on; nothing here calls the extension.

Error contract
--------------
A kernel output ``got`` passes ``assert_within`` when, element by element,

    |got - ref| <= tau * mag + extra + u_out * |ref|

``ref``   the operation in fp64 on exactly the operands the kernel was given (bf16 A and B, fp32 vectors and records).
``mag``   |A| @ |B|^T carried through the epilogue, each step adding the magnitudes of its terms (see ``gemm_ref``).  A bf16
          product is exact in fp32, so the only roundings in the accumulation are its additions, and every partial sum is
          bounded by ``mag``.  An fp32 evaluation of the epilogue rounds a value bounded by ``mag`` a fixed handful of times.
``tau``   2^-16 (``TAU``).  The worst case of K ordered fp32 additions is K * 2^-24 * mag; it is not reached with data
          of either sign, where the rounding errors of the partial sums (each <= 2^-24 |s_k|, |s_k| ~ sqrt(k)) add like a
          random walk to about 2^-24 * mag whatever K is.  Additions that truncate instead of rounding (errors all of one
          sign) reach about 2^-23 * sqrt(K / 16) * mag for 16-deep tensor-core steps, 2^-18.2 at K = 12608.  The largest
          error measured on an H100 is 2^-19.7 * mag (dW, K = 12608), so 2^-16 leaves room for any fp32 accumulation order
          (tiled, split-K, persistent) and is still 2^10 below the error of a wrong fragment row, a column slice shifted
          by 8 or a dropped k-block (tests/test_kernel_ref.py shows each of them failing).
``extra`` absolute allowances that do not scale with ``mag``: the fp32 evaluation of LayerNorm statistics from partial
          records (``ln_stats_ref``) and, for the contrastive head, the errors of the bf16x3 logits.
``u_out`` 2^-8 for a bf16 output, 0 for fp32.  Round-to-nearest to 8 significant bits moves the kernel's fp32 value v by
          less than 2^-8 |v|, and |v| exceeds |ref| by at most the fp32 error (itself far inside tau * mag).

Attention (``attention_ref``, ``attention_bwd_ref``)
-----------------------------------------------------
The reference is the operation in fp64 on the operands the kernel receives: bf16 ``qkv`` with q already scaled, the fp32
bias values the kernel adds (for the LUT forms, the dense table they encode), padded keys at -inf.  The backward also
takes the forward's bf16 ``out``, ``d_out`` and fp32 ``lse``, and defines delta_i = sum_d dO_id out_id on the given bf16
``out`` (as the kernel and flash-attention do), so delta is part of the operation and not a source of error.  Bounds are
absolute (``assert_within(got, ref, bound, 1.0, dtype)``; a bf16 output adds u_out |ref| there) and first order.

``e_ij``   logit error, tau (|q_i| . |k_j|) + c_exp_ij + eps_b |b_ij|.  tau covers the fp32 accumulation of q.k (as for the
           GEMM).  c_exp = 2^-19 (1 + |s_ij| + |lse_i|): __expf(x) = ex2.approx(x log2 e) is off by 2^-22 relative plus the
           rounding of x log2 e, and x = s - m is itself rounded twice (s + b, then - m; |m| <= |lse| + log S), which is a
           few ulps of |s| and |lse| and stays under 32 ulps of (1 + |s| + |lse|).  eps_b = 0 for the fp32 bias forms.
           The transposed half2 tables of the backward hold fp16(b log2 e): eps_b = 2^-11 + 2^-22 (round-to-nearest to 11
           bits, then the fp32 products), plus an absolute 2^-24 for fp16 subnormals (``EPS_B_HALF``).
``lse``    sum_j P_ij e_ij + 2^-16 (1 + |lse_i|).  The second term is the fp32 sum of up to 750 positive exponentials (round
           to nearest: a random walk far below 2^-16 relative), at most a dozen rescales by exp(m_old - m_new) of 2^-22
           each, and the log.
``out``    2^-8 (P @ |V|) + sum_j P_ij (e_ij + dlse_i) (|v_j| + |o_i|) + tau (P @ |V|), then u_out |ref|.  P.V runs on bf16 P
           (2^-9 relative under round-to-nearest, doubled for margin, whatever the key blocking) while the denominator is
           summed from the unrounded fp32 values, so the rounding does not cancel.  A relative error d_j of P_ij moves
           o_i = sum_j P_ij v_j / sum_j P_ij by sum_j P_ij d_j (v_j - o_i); |v_j - o_i| <= |v_j| + |o_i|.
``ln_stats`` per (head, row) sum and sum of squares of the 64 fp32 outputs before rounding: the ``out`` bound (without
           u_out) carried through both sums, plus tau of the fp32 sums of |o| and o^2.
``dV``     sum_i P_ij (2^-8 + e'_ij) |dO_i| + tau P^T |dO|, where e'_ij = e_ij + |lse_given_i - lse_i| is the error of the
           recomputed P (the backward recomputes P from the given lse, so its actual error enters).
``dS``     dS_ij = P_ij (dP_ij - delta_i), dP = dO V^T.  err(dS_ij) = P_ij (|dP_ij - delta_i| e'_ij + tau (|dO_i| . |v_j| +
           sum_d |dO_id| |out_id|)): the error of P scales dP - delta, tau covers the fp32 dot products of dP and delta.
``dbias``  sum_b dS_b over the batch for a shared table (fp32 atomics onto the initial values: + (B + 1) 2^-24 (|init| +
           sum_b |dS_b|)); dS_b alone for per-sample tables.  Centring a row, c_ij = d_ij - mean_j d_ij, is exact in fp64;
           the bound becomes err_ij + mean_j err_ij + S 2^-24 sum_j |d_ij| (the fp32 row sum).
``dQ, dK`` dQ = q_scale bf16(dS) @ K and dK = bf16(dS)^T @ Q: (2^-8 |dS| + err(dS)) @ |K or Q| + tau |dS| @ |K or Q| (times
           q_scale for dQ), then u_out |ref|.
"""
from types import SimpleNamespace

import numpy as np
import torch

TAU = 2.0 ** -16
U32 = 2.0 ** -24              # fp32 unit round-off
GELU_SLOPE = 1.13             # max |gelu'(x)| = Phi(sqrt 2) + sqrt 2 phi(sqrt 2) = 1.1289

EPI_STORE_BF16, EPI_GEGLU_BF16, EPI_RESID_F32, EPI_STORE_F32, EPI_GELU_BF16 = 0, 1, 2, 3, 4


def _gelu(x):
    return torch.nn.functional.gelu(x)


def ln_stats_ref(records, parts, M, dim, eps):
    """(mu, rstd) of M rows from [parts, M, 2] (sum, sum of squares) records, in fp64, and the allowances of the kernel's
    fp32 evaluation: ``dmu`` (absolute error of mu) and ``rel`` (relative error of rstd).

    The kernel adds the P = parts records in fp32 (in any order), divides by n = dim, and takes
    var = E[x^2] - mu^2, rstd = rsqrt(max(var, 0) + eps).  With u = 2^-24 and a1 = sum_p |s1_p| / n:
      |d mu|   <= P u a1 + u |mu|                            (mixed-sign sum, then the division)
      |d E2|   <= P u E[x^2]                                 (sum of non-negative records, then the division)
      |d mu^2| <= 2 |mu| |d mu| + u mu^2
      |d var|  <= (P + 2) u (E[x^2] + 2 |mu| a1)             (mu^2 <= E[x^2], var <= E[x^2])
    so rstd is off by at most |d var| / (2 (var + eps)) relative, plus 2^-22 for rsqrtf (2 ulp).  The E[x^2] / var factor is
    the cancellation of E[x^2] - mu^2 for rows whose mean is large against their spread."""
    r = records.reshape(parts, M, 2).double()
    s1, s2 = r[..., 0].sum(0), r[..., 1].sum(0)
    mu, ex2 = s1 / dim, s2 / dim
    var = (ex2 - mu * mu).clamp_min(0.0)
    rstd = (var + eps).rsqrt()
    a1 = r[..., 0].abs().sum(0) / dim
    dmu = parts * U32 * a1 + U32 * mu.abs()
    rel = (parts + 2) * U32 * (ex2 + 2 * mu.abs() * a1) / (2 * (var + eps)) + 2.0 ** -22
    return mu, rstd, dmu, rel


def gemm_ref(a, w, epi, *, bias=None, colscale=None, gamma=None, resid=None, ln_mu=None, ln_rstd=None, ln_colsum=None,
             ln_partial=None, out_group=0, out_group_stride=0, out_row_offset=0, out_group_valid=0, resid_period=0,
             resid_row_offset=0, stats=False):
    """fp64 result of ``epilogue(a[M,K] @ w[N,K]^T)`` as the kernel defines it (csrc/gemm.h), for the logical rows m < M.

    Returns a namespace with
      y, mag, extra   [M, N_out] (N_out = N / 2 for GeGLU): the result and its bound terms (module docstring);
      rows, valid     [M]: the output row each logical row is stored to, and whether it is stored (out_group_valid);
      stats, stats_mag, stats_extra   when ``stats``: the (sum, sum of squares) records the epilogue writes,
                      [N / 256, M, 2] (residual) or [N / 128, M, 2] with every second record zero (GeGLU).

    How ``mag`` is carried (first order; products of two allowances are below 2^-32 relative and left out):
      acc     : |A| @ |B|^T
      LN      : x = rstd (acc - mu colsum):  rstd (mag_acc + |mu colsum|), extra rstd (rel (mag_acc + |mu colsum|) + dmu |colsum|)
      bias    : + |bias|
      colscale: * |colscale|;   gelu: * 1.13 (the largest slope of gelu)
      GeGLU   : u = gelu(g) l:  1.13 mag_g |l| + |gelu(g)| mag_l   (same for extra)
      residual: y = resid + gamma x:  |resid| + |gamma| mag_x
    The statistics records sum 128 or 256 stored values v in fp32 (<= 70 additions deep, under 2^-16 of sum |v|):
      sum     : tau * sum (mag_v + |v|) + sum extra_v
      sum sq  : tau * sum (2 |v| mag_v + v^2) + sum 2 |v| extra_v"""
    A, B = a.double(), w.double()
    M, N = A.shape[0], B.shape[0]
    x = A @ B.t()
    xm = A.abs() @ B.abs().t()
    xe = torch.zeros_like(x)
    if ln_colsum is not None:
        cs = ln_colsum.double()[None, :]
        if ln_partial is not None:
            rec, parts, dim, eps = ln_partial
            mu, rstd, dmu, rel = ln_stats_ref(rec, parts, M, dim, eps)
        else:
            mu, rstd = ln_mu.double(), ln_rstd.double()
            dmu, rel = torch.zeros_like(mu), torch.zeros_like(mu)
        mu, rstd, dmu, rel = mu[:, None], rstd[:, None], dmu[:, None], rel[:, None]
        tm = xm + (mu * cs).abs()
        x = rstd * (x - mu * cs)
        xm = rstd * tm
        xe = rstd * (rel * tm + dmu * cs.abs())
    if bias is not None:
        x = x + bias.double()
        xm = xm + bias.double().abs()
    m = torch.arange(M, device=A.device)
    rows, valid = m, torch.ones(M, dtype=torch.bool, device=A.device)
    if out_group > 0:
        rows = (m // out_group) * out_group_stride + (m % out_group) + out_row_offset
        if out_group_valid > 0:
            valid = (m % out_group) < out_group_valid
    st = None
    if epi in (EPI_STORE_BF16, EPI_GELU_BF16, EPI_STORE_F32):
        if colscale is not None and epi != EPI_STORE_F32:
            c = colscale.double()
            x, xm, xe = x * c, xm * c.abs(), xe * c.abs()
        if epi == EPI_GELU_BF16:
            x, xm, xe = _gelu(x), GELU_SLOPE * xm, GELU_SLOPE * xe
        y, ym, ye = x, xm, xe
    elif epi == EPI_RESID_F32:
        gm = gamma.double() if gamma is not None else torch.ones(N, dtype=torch.float64, device=A.device)
        y, ym, ye = gm * x, gm.abs() * xm, gm.abs() * xe
        if resid is not None:
            res_rows = (m % resid_period) + resid_row_offset if resid_period > 0 else rows
            r = resid.double()[res_rows]
            y, ym = y + r, ym + r.abs()
        width = 256
    elif epi == EPI_GEGLU_BF16:
        assert N % 256 == 0
        def halves(t):
            t = t.view(M, N // 256, 2, 128)
            return t[:, :, 0].reshape(M, N // 2), t[:, :, 1].reshape(M, N // 2)
        (g, l), (gmag, lmag), (gex, lex) = halves(x), halves(xm), halves(xe)
        gg = _gelu(g)
        y = gg * l
        ym = GELU_SLOPE * gmag * l.abs() + gg.abs() * lmag
        ye = GELU_SLOPE * gex * l.abs() + gg.abs() * lex
        width = 128
    else:
        raise ValueError(f"no reference for epilogue {epi}")
    if stats:
        assert epi in (EPI_RESID_F32, EPI_GEGLU_BF16)
        nt = (y.shape[1] + width - 1) // width
        pad = nt * width - y.shape[1]
        def tiles(t):
            return torch.nn.functional.pad(t, (0, pad)).view(M, nt, width)
        v, vm, ve = tiles(y), tiles(ym), tiles(ye)
        s = torch.stack([v.sum(2), (v * v).sum(2)], 2)
        sm = torch.stack([(vm + v.abs()).sum(2), (2 * v.abs() * vm + v * v).sum(2)], 2)
        se = torch.stack([ve.sum(2), (2 * v.abs() * ve).sum(2)], 2)
        s, sm, se = (t.transpose(0, 1) for t in (s, sm, se))
        if epi == EPI_GEGLU_BF16:          # a zero record after every tile's
            s, sm, se = (torch.stack([t, torch.zeros_like(t)], 1).reshape(2 * nt, M, 2) for t in (s, sm, se))
        st = (s.contiguous(), sm.contiguous(), se.contiguous())
    ns = SimpleNamespace(y=y, mag=ym, extra=ye, rows=rows, valid=valid, stats=None, stats_mag=None, stats_extra=None)
    if st is not None:
        ns.stats, ns.stats_mag, ns.stats_extra = st
    return ns


def assert_within(got, ref, mag, tau, out_dtype, extra=None, what="output"):
    """|got - ref| <= tau * mag + extra + u_out * |ref| element by element (u_out = 2^-8 for a bf16 output, 0 for fp32).
    On failure names the worst element (index, got, ref, ratio) and how many elements fail.  Returns the largest ratio
    |got - ref| / bound, the fraction of the bound used."""
    g = got.double()
    ref = ref.double()
    u_out = 2.0 ** -8 if out_dtype == torch.bfloat16 else 0.0
    tol = tau * mag + u_out * ref.abs()
    if extra is not None:
        tol = tol + extra
    err = (g - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / tol)
    ratio = torch.nan_to_num(ratio, nan=float("inf"))          # a NaN or Inf output fails
    worst = ratio.max().item() if ratio.numel() else 0.0
    if not worst <= 1.0:
        flat = int(ratio.argmax().item())
        idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
        n_bad = int((ratio > 1.0).sum().item())
        raise AssertionError(
            f"{what}: {n_bad} of {ratio.numel()} elements outside the bound; worst at {idx}: got {g[idx].item()!r}, "
            f"ref {ref[idx].item()!r}, |err| {err[idx].item():.3e} = {worst:.3g} x bound {tol[idx].item():.3e} "
            f"(tau {tau:.3g} x mag {mag[idx].item():.3e})")
    return worst


def _nan_bits(dtype, device):
    it = torch.int16 if dtype == torch.bfloat16 else torch.int32
    return torch.full((1,), float("nan"), dtype=dtype, device=device).view(it), it


def canary_out(shape, ldo_extra=0, rows_before=0, rows_after=0, dtype=torch.float32, device="cuda"):
    """An output view of ``shape`` (rows, cols) inside a larger NaN-filled buffer: ``rows_before`` / ``rows_after`` spare
    rows around it and a row pitch of cols + ``ldo_extra``.  Returns (view, buffer)."""
    rows, cols = shape
    buf = torch.full((rows_before + rows + rows_after, cols + ldo_extra), float("nan"), dtype=dtype, device=device)
    return buf[rows_before:rows_before + rows, :cols], buf


def assert_canary(buf, out, written=None, what="output"):
    """Every element of ``buf`` outside the written part of ``out`` (a view into it) is still the bit pattern it was filled
    with, and every written element is finite.  ``written``: bool mask over ``out`` (default: all of it)."""
    ld = buf.stride(0)
    off = out.storage_offset() - buf.storage_offset()
    r0, c0 = off // ld, off % ld
    mask = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    region = mask[r0:r0 + out.shape[0], c0:c0 + out.shape[1]]
    region.copy_(written if written is not None else torch.ones(out.shape, dtype=torch.bool, device=buf.device))
    nan_bits, it = _nan_bits(buf.dtype, buf.device)
    outside = buf.view(it)[~mask]
    touched = int((outside != nan_bits).sum().item())
    assert touched == 0, f"{what}: {touched} elements outside the logical output were written"
    inside = buf[mask]
    bad = int((~torch.isfinite(inside)).sum().item())
    assert bad == 0, f"{what}: {bad} of {inside.numel()} elements of the logical output are not finite (never written?)"


# ----------------------------------------------------------------------------------------------------------------------
# contrastive head
# ----------------------------------------------------------------------------------------------------------------------
# Logit error of the bf16x3 split GEMM: z = s * (hi.hi' + hi.lo' + lo.hi') with hi = bf16(x), lo = bf16(x - hi), so
# |x - hi - lo| <= 2^-18 |x|, the dropped lo.lo' term is <= 2^-18 |x y|, and x y - (the three kept terms) <= 3 * 2^-18 |x y|;
# the fp32 accumulation adds tau over (1 + 2^-8) sum |x y|, the scale product 2^-24.
Z_TAU = TAU * (1 + 2.0 ** -8) + 3 * 2.0 ** -18 + U32


def infonce_ref(xa, xb_all, scale, target_offset, eps, n_valid=0):
    """One direction of the InfoNCE head from the fp32 features, in fp64: local rows xa [b, d], gathered rows xb_all [n, d]
    (rows >= n_valid are padding when n_valid > 0), s = scale (python float), target of row i = i + target_offset.

      z = s xa xb^T (classes j < n_cls),  lse_i = logsumexp_j z_ij,  eps_i = eps / (n_cls - 1)
      loss_i = (1 - eps - eps_i)(lse_i - z_it) + eps_i (n_cls lse_i - sum_j z_ij)
      G_ij = softmax(z)_ij - (1 - eps - eps_i)[j == t_i] - eps_i,  gz_i = sum_j G_ij z_ij

    Bounds (first order in the logit error dz_ij <= Z_TAU * s * (|xa| |xb|^T)_ij):
      lse : sum_j p_ij dz_ij, plus 2^-16 (1 + |lse|) for the fp32 sum of exponentials (<= 300 additions deep) and log;
      loss: (1 - eps - eps_i)(d lse + dz_it) + eps_i (n d lse + sum_j dz_ij), plus 2^-16 times the magnitudes of its terms;
      gz  : sum_j (|dG_ij| |z_ij| + |G_ij| dz_ij) + 2^-16 sum_j |G_ij z_ij|, with |dG_ij| <= p_ij (dz_ij + d lse + 2^-20)."""
    b = xa.shape[0]
    n_cls = n_valid if n_valid > 0 else xb_all.shape[0]
    xa64, xb64 = xa.double(), xb_all[:n_cls].double()
    z = scale * (xa64 @ xb64.t())
    dz = Z_TAU * scale * (xa64.abs() @ xb64.abs().t())
    lse = torch.logsumexp(z, 1)
    p = (z - lse[:, None]).exp()
    dlse = (p * dz).sum(1) + 2.0 ** -16 * (1 + lse.abs())
    eps_i = eps / (n_cls - 1) if eps != 0 else 0.0
    hit = 1.0 - eps - eps_i
    rows = torch.arange(b, device=xa.device)
    tgt = rows + target_offset
    zt, dzt = z[rows, tgt], dz[rows, tgt]
    zsum, dzsum, azsum = z.sum(1), dz.sum(1), z.abs().sum(1)
    loss = hit * (lse - zt) + eps_i * (n_cls * lse - zsum)
    dloss = hit * (dlse + dzt) + eps_i * (n_cls * dlse + dzsum)
    dloss = dloss + 2.0 ** -16 * (lse.abs() + zt.abs() + eps_i * (n_cls * lse.abs() + azsum))
    G = p - eps_i
    G[rows, tgt] -= hit
    dG = p * (dz + dlse[:, None] + 2.0 ** -20)
    gz = (G * z).sum(1)
    dgz = (dG * z.abs() + G.abs() * dz).sum(1) + 2.0 ** -16 * (G * z).abs().sum(1)
    return SimpleNamespace(z=z, dz=dz, lse=lse, dlse=dlse, loss=loss, dloss=dloss, p=p, G=G, dG=dG, gz=gz, dgz=dgz,
                           eps_i=eps_i, n_cls=n_cls, tgt=tgt)


def infonce_grad_ref(r, xb_hi, scale, coef):
    """grad = s coef G @ B_hi (the kernel contracts its bf16-rounded G with the bf16 "hi" part of the gathered rows),
    and its absolute bound: the bf16 rounding of each s coef G_ij (2^-8 |.| with the fp32 error of the value rounded), the
    error of G (r.dG), and tau of the fp32 accumulation over sum_j |s coef G_ij| |B_hi,jk|."""
    Bh = xb_hi[:r.n_cls].double()
    f = scale * coef
    grad = f * (r.G @ Bh)
    tol = f * ((2.0 ** -8 * r.G.abs() + r.dG) @ Bh.abs()) + TAU * f * (r.G.abs() @ Bh.abs())
    return grad, tol


def argmax_ok(z, dz, got):
    """Rows whose arg-max ``got`` is a maximum of z within the logit error: z[got] >= max z - dz[got] - dz[argmax]."""
    ref = z.argmax(1)
    rows = torch.arange(z.shape[0], device=z.device)
    g = got.long()
    zg = z[rows, g]
    return zg >= z[rows, ref] - dz[rows, g] - dz[rows, ref]


# ----------------------------------------------------------------------------------------------------------------------
# attention (module docstring, "Attention")
# ----------------------------------------------------------------------------------------------------------------------
HD = 64                                 # head dim of every attention kernel
C_EXP = 2.0 ** -19
LSE_REL = 2.0 ** -16
EPS_B_HALF = (2.0 ** -11 + 2.0 ** -22, 2.0 ** -24)       # (relative, absolute) logit error of the fp16 transposed tables


def split_qkv(qkv, B, S, H):
    """bf16 [B*S, 3*H*64] -> fp64 q, k, v of shape [B, H, S, 64]"""
    t = qkv.double().view(B, S, 3, H, HD).permute(2, 0, 3, 1, 4)
    return t[0], t[1], t[2]


def heads_to_rows(t, B, S, H):
    """[B, H, S, 64] -> [B*S, H*64] (the row layout of the attention output and of each third of dqkv)"""
    return t.permute(0, 2, 1, 3).reshape(B * S, H * HD)


def _logits(qkv, bias, key_pad, B, S, H, eps_b):
    """scores s = q k^T + b with padded keys at -inf, and the parts of the logit error e (without c_exp, which needs lse)"""
    q, k, v = split_qkv(qkv, B, S, H)
    s = q @ k.transpose(-1, -2)
    e = TAU * (q.abs() @ k.abs().transpose(-1, -2))
    if bias is not None:
        b = bias.double()
        b = b if b.dim() == 4 else b[None]
        s = s + b
        if eps_b:
            e = e + eps_b[0] * b.abs() + eps_b[1]
    dead = torch.zeros(B, 1, 1, S, dtype=torch.bool, device=qkv.device)
    if key_pad is not None:
        dead = key_pad.bool().view(B, 1, 1, S)
    s = s.masked_fill(dead, float("-inf"))
    return q, k, v, s, e, dead


def attention_ref(qkv, bias, key_pad, B, S, H, eps_b=None):
    """fp64 attention forward and its bounds (module docstring).  bias: the values the kernel adds, fp32 (H,S,S) shared or
    (B,H,S,S) per sample (logical columns only), or None; key_pad uint8 (B,S) or None; eps_b: EPS_B_HALF for the fp16
    tables.  Every row needs a live key.

    Returns a namespace with out / out_err [B*S, H*64], lse / dlse [B, H, S], stats / stats_err [H, B*S, 2] (the
    ln_stats records), and p, e (P and the logit error, [B, H, S, S]) for ``attention_bwd_ref``."""
    q, k, v, s, e, dead = _logits(qkv, bias, key_pad, B, S, H, eps_b)
    lse = torch.logsumexp(s, -1)
    p = (s - lse[..., None]).exp()
    sf = torch.where(dead, torch.zeros_like(s), s)
    e = (e + C_EXP * (1 + sf.abs() + lse.abs()[..., None])).masked_fill(dead, 0.0)
    pe = p * e
    dlse = pe.sum(-1) + LSE_REL * (1 + lse.abs())
    o = p @ v
    pv = p @ v.abs()
    w = pe + p * dlse[..., None]                        # sum_j P_ij (e_ij + dlse_i) (|v_j| + |o_i|)
    oerr = (2.0 ** -8 + TAU) * pv + w @ v.abs() + w.sum(-1, keepdim=True) * o.abs()
    st = torch.stack([o.sum(-1), (o * o).sum(-1)], -1)                                        # [B, H, S, 2]
    st_err = torch.stack([oerr.sum(-1) + TAU * o.abs().sum(-1),
                          (2 * o.abs() * oerr + oerr * oerr).sum(-1) + TAU * (o * o).sum(-1)], -1)
    to_rec = lambda t: t.permute(1, 0, 2, 3).reshape(H, B * S, 2)
    return SimpleNamespace(out=heads_to_rows(o, B, S, H), out_err=heads_to_rows(oerr, B, S, H), lse=lse, dlse=dlse,
                           stats=to_rec(st), stats_err=to_rec(st_err), p=p, e=e)


def attention_bwd_ref(qkv, out, d_out, lse, bias, key_pad, B, S, H, q_scale, eps_b=None):
    """fp64 attention backward on the operands of the backward call and its bounds (module docstring).  out, d_out bf16
    [B*S, H*64]; lse fp32 [B*H*S] as given to the kernel; bias and key_pad as for ``attention_ref``.

    Returns a namespace with dqkv / dqkv_err [B*S, 3*H*64] and dS, dS_err [B, H, S, S] for ``dbias_ref``."""
    f = attention_ref(qkv, bias, key_pad, B, S, H, eps_b)
    q, k, v = split_qkv(qkv, B, S, H)
    do = d_out.double().view(B, S, H, HD).permute(0, 2, 1, 3)
    o = out.double().view(B, S, H, HD).permute(0, 2, 1, 3)
    p = f.p
    ep = f.e + (lse.double().view(B, H, S) - f.lse).abs()[..., None]
    dp = do @ v.transpose(-1, -2)
    delta = (do * o).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    ds_err = p * ((dp - delta).abs() * ep + TAU * (do.abs() @ v.abs().transpose(-1, -2) + (do.abs() * o.abs()).sum(-1, keepdim=True)))
    dv = p.transpose(-1, -2) @ do
    dv_err = ((2.0 ** -8 + TAU) * p + p * ep).transpose(-1, -2) @ do.abs()
    a = 2.0 ** -8 * ds.abs() + ds_err + TAU * ds.abs()
    dq = q_scale * (ds @ k)
    dq_err = abs(q_scale) * (a @ k.abs())
    dk = ds.transpose(-1, -2) @ q
    dk_err = a.transpose(-1, -2) @ q.abs()
    rows = lambda *ts: torch.cat([heads_to_rows(t, B, S, H) for t in ts], 1)
    return SimpleNamespace(dqkv=rows(dq, dk, dv), dqkv_err=rows(dq_err, dk_err, dv_err), dS=ds, dS_err=ds_err, fwd=f)


def dbias_ref(r, init, launches=1, per_sample=False):
    """the bias gradient the backward accumulates onto ``init`` (fp32, logical columns): sum_b dS_b for a shared table
    ((H,S,S); ``launches`` backward calls on the same operands add into it), dS_b for per-sample tables ((B,H,S,S)).
    Returns (value, bound); the fp32 additions add (adds + 1) 2^-24 (|init| + sum |terms|)."""
    i = init.double()
    if per_sample:
        d, err, mag, adds = r.dS, r.dS_err, r.dS.abs(), 1
    else:
        d, err, mag, adds = launches * r.dS.sum(0), launches * r.dS_err.sum(0), launches * r.dS.abs().sum(0), launches * r.dS.shape[0]
    return i + d, err + (adds + 1) * U32 * (i.abs() + mag)


def center_ref(d, err):
    """row-centred bias gradient c_ij = d_ij - mean_j d_ij over the S logical columns, and its bound"""
    S = d.shape[-1]
    return d - d.mean(-1, keepdim=True), err + err.mean(-1, keepdim=True) + S * U32 * d.abs().sum(-1, keepdim=True)
