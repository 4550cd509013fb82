"""fp64 references of the GEMM epilogues (csrc/gemm_wgmma.cu) and of the convolutions lowered onto that GEMM, of the
contrastive-head reductions (csrc/infonce.cu), of the attention forward and backward (csrc/attention.cu,
csrc/attention_bwd.cu) and of the row kernels (csrc/layernorm.cu, csrc/backward.cu, csrc/pack.cu, csrc/gather.cu), with an
error bound for every output element, and NaN-canary output buffers; of the fused Adam step and the gradient norm
(csrc/adam.cu); and of the embedding, gather, transpose and ranking kernels (csrc/adapters.cu, csrc/gather.cu,
csrc/infonce.cu, csrc/recall.cu), most of them exact.

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
          records (``ln_stats_ref``), the fp32 colsum and bias of a LayerNorm fold when the reference takes their exact
          values (``ln_colsum_err``, ``bias_err``: the ``ln_fold_ref`` bounds) and, for the contrastive head, the errors of
          the bf16x3 logits.
``u_out`` 2^-8 for a bf16 output, 0 for fp32.  Round-to-nearest to 8 significant bits moves the kernel's fp32 value v by
          less than 2^-8 |v|, and |v| exceeds |ref| by at most the fp32 error (itself far inside tau * mag).

Convolutions (``window_matrix``, ``grouped_window_ref``)
---------------------------------------------------------
The adapters lower convolutions onto the same GEMM, and each form is the GEMM of a window matrix, so its reference is
``gemm_ref`` on that matrix with the same bound (no new constant).  The grouped sliding window (``grouped_conv1d``) of
group g is A_g[r, j * c_pad + c] = X[r + j, g, c] against the weight rows W[g * n : (g + 1) * n], its output the columns
g * n ... (g + 1) * n - 1 with bias[g * n : (g + 1) * n]; every c < c_pad counts, padding channels included.  The
reference builds one group's fp64 window at a time on the inputs' device (about 30 MB at the audio positional conv).
Overlapping strided rows (``gemm(..., K=kw*C, lda=2*C)``, the feature-extractor convolutions) are the plain reference
on ``flat.as_strided((M, K), (lda, 1))``; narrow K (K < 64: one zero-filled k-block) is the plain reference as is.

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
``lse``    sum_j P_ij e_ij + 2^-16 (1 + |lse_i|).  The second term is the fp32 sum of up to S = 1025 positive exponentials,
           the longest sequence the suite runs (the 512^2 ViT): each lane adds about S / 4 of them before a 4-lane
           reduction, and round-to-nearest errors add like a random walk to about sqrt(S / 4) 2^-24 = 2^-20 relative; one
           rescale by exp(m_old - m_new) per further 64-key block, at most 16 of 2^-22 each (2^-18); and the log.  The
           total stays under 2^-17.5, so 2^-16 still holds at S = 1025.
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

Row kernels (``layernorm_ref``, ``layernorm_bwd_ref`` and the functions after them)
----------------------------------------------------------------------------------
Bounds are absolute (``assert_within(got, ref, bound, 1.0, dtype)``), first order, u = 2^-24.  Every fp32 reduction in these
kernels is at most 256 additions deep (a row: <= 24 per thread, 5 shuffle levels, <= 8 warps; a column: <= 48 rows per CTA
at 12608 rows, <= 10 + 32 steps in ``partial_reduce_kernel``), so tau = 2^-16 >= 256 u bounds its worst case, in any order.

``fast_erf``  Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7) evaluated in fp32 with rcp.approx (1 ulp) and ex2.approx (2^-22
           relative).  Near x = 0, 1 - p e cancels: eight roundings of values near 1 add <= 5e-7, rcp moves p e by
           |t p'(t)| e 2^-23 <= 3e-7, ex2 by 2^-22 p e <= 2.4e-7: ERF_ABS = 2^-19 (1.9e-6) covers the sum, 1.2e-6.
           gelu_erf(y) = 0.5 y (1 + erf(y / sqrt 2)) is then off by |y| GELU_REL, GELU_REL = ERF_ABS / 2 + 4 u.
           gelu_grad(z) = Phi(z) + z phi(z) with phi from __expf (2 + 1.173 |x| ulps): GELU_GRAD_ABS = ERF_ABS / 2 + 2^-21
           (the z phi(z) (2 + 0.59 z^2) 2^-23 <= 2^-23 term and the roundings).  tests/test_kernel_ref.py evaluates an fp32
           port with every approximation perturbed by its limit and checks all three constants.  An error dz of the
           argument moves gelu by <= 1.13 dz and gelu' by <= 0.8 dz (max |gelu''| = 2 phi(0)).
``layernorm`` (two-pass statistics, one warp per row)  With a1 = mean |x|:  dmu = (tau + u) a1;  the centred sum of squares
           about the rounded mean is var + dmu^2 exactly, so dvar = (tau + 3u) var + dmu^2;  rel(rstd) = dvar / (2 (var +
           eps)) + 2^-22 (rsqrtf; every rel here uses the form of ``ln_stats_ref`` that stays exact for large dvar);
           xhat: rstd (dmu + u |x - mu|) + |xhat| (rel + u);  affine: |g| dxhat + 2u (|xhat g| + |b|);  gelu: 1.13 dy +
           |y| GELU_REL;  fp32 ``accumulate``: + u (|prev| + |y|);  then u_out |ref|.  ``raw`` writes bf16(x) (bit-exact)
           and mu / rstd with the bounds dmu and rel.
``layernorm_bwd``  dx = rstd (dy g - m1 - xhat m2), m1 = mean(dy g), m2 = mean(dy g xhat).  The plain path reduces in one
           pass about K = x[row][0]: ms = mean(x - K), var = mean((x - K)^2) - ms^2.  With A = mean |x - K| and
           Q = mean (x - K)^2 = var + ms^2:  dms = (tau + u) A;  dvar = (tau + 2u) Q + 2 A dms + dms^2 (the Q / var factor
           is the cancellation, small while K is near the mean, large for an outlier in column 0 or |mean| / std ~ 10^3);
           m2 = rstd mean(dy g (x - K - ms)) is off by rstd ((tau + 2u) mean |dy g| |x - K| + |ms| dm1 + |m1| dms +
           2u |ms m1|) + |m2| (rel + u).  The gelu path runs two-pass statistics as the forward and first multiplies dy by
           gelu'(z), z = xhat g + b (dz = |g| dxhat + u |z|, d gelu' = 0.8 dz + GELU_GRAD_ABS).  Both paths then give
           dx: rstd (d(dy g) + dm1 + |xhat| dm2 + |m2| dxhat + 2u (|dy g| + |m1| + |xhat m2|)) + |dx| (rel + u).
           dgamma = sum_rows dy' xhat and dbeta = sum_rows dy' (dy' = dy, or dy gelu'(z)): sum of the terms' errors plus
           (tau + u) sum |terms|.
``geglu``  u = gelu(g) l: |l| |g| GELU_REL + 2u |u|.  Backward: dg = du l gelu'(g): |du l| GELU_GRAD_ABS + 3u |dg|;
           dl = du gelu(g): |du g| GELU_REL + u |dl|.  bf16 outputs add u_out |ref|.
``scale_resid``  forward out = x + rs gamma o: 2u (|rs gamma o| + |out|).  Backward d = rs gamma dx (2u |d|), d_o = bf16(d);
           dgamma = sum_rows rs dx o and dbias = sum_rows d, both with (tau + 2u) sum |terms|.  dbias sums the fp32 values d,
           not the rounded d_o (the fp32 value is the better estimate of the true gradient; ``colsum`` serves the passes
           that only have d_o and sums exactly those bf16 values).
``colsum``  sum of the given bf16 values: tau sum |y|.
``ln_fold``  Wg = bf16(fp32(W g)) is bit-exact; colsum = sum_k Wg (the rounded values): tau sum |Wg|; bias' = W beta + b:
           (tau + u) sum |W| |beta| + u (|bias'| + |b|).
``l2_normalize_bwd``  dx = dy / |x| - x (x . dy) / |x|^3.  The fp32 norm is off by rel_n = (tau + 2u) / 2 + u relative
           (``L2_NORM_REL``: tau for the sum of squares, then the sqrt's rounding),
           1 / |x| by rel_n + u; k = (x . dy) / |x|^3 by (tau + u) sum |x dy| / |x|^3 + |k| (3 rel_n + 4u); dx: |dy| / |x|
           (rel_n + 2u) + |x| dk + u (|x k| + |dx|).
scatter-adds  (fp32 atomics, ``batch_sum``): onto init, count contributions in any order: (count + 1) u (|init| + sum |g|)
           per destination element.  ``window_scatter`` sums <= kw bf16 terms in a fixed order: kw u sum |terms|, then
           u_out |ref|.

Embedding, gather, transpose and ranking kernels (``text_embed_ref`` and the functions after it)
-------------------------------------------------------------------------------------------------
``text_embed``, ``cls_row_init``, ``zero_padded_rows``, ``relpos_bias_build``, ``relpos_lut_build``, ``row_gather``,
``relpos_bias_block``, ``transpose_bf16``, ``topk10_rows`` and ``recall_hits`` are exact: each output element is a gather,
a copy, or one fp32 addition followed by at most one round-to-nearest to bf16.  The reference is the same fp32 operation in
torch and the comparison is bit for bit.  One exception: ``text_embed`` zeroes pad rows, which the reference writes as
(emb + pos) * (1 - mask); that can be -0.0, so pad rows are compared by value.
``l2_normalize_rows``  y = x / max(|x|, 1e-12) in fp64.  The kernel's fp32 norm is off by ``L2_NORM_REL`` relative (as for
           ``l2_normalize_bwd``: the sum of squares of a row is <= 16 + 5 + 8 additions deep per 256-thread CTA at D = 4096,
           far under tau); max(., fp32(1e-12)) adds the rounding of 1e-12 to fp32 for a clamped row; the reciprocal and the
           product add u each: |y| (L2_NORM_REL + rel(fp32(1e-12)) + 2u).  The bf16 copy is rounded from the same register,
           so it equals bf16(y_fp32) bit for bit.
``topk10_rows``  ranks each row by a total order (``order_key``): fp32 values in IEEE order with -0.0 equal to +0.0, every
           NaN above +inf, -inf like any other value, and equal keys by the smaller column.  That is a stable descending
           sort of the row, with NaN first as ``torch.topk`` ranks it.  Slots past C hold column -1 and value -inf.
``topk_within``  for the retrieval similarity (bf16x3 GEMM logits, error dz = Z_TAU (|a| @ |b|^T)): the returned list is a
           top-10 of some matrix within dz of the fp64 similarity.  Consecutive returned entries are ordered within their
           two errors, and no column left out beats the 10th returned one by more than their two errors.  Recall@k can then
           differ from the fp64 count only in rows whose k-th and (k+1)-th fp64 values lie within twice the row's largest
           error (``recall_ref``).

Optimizer (``adam_ref``, ``bf16_param_check``, ``grad_norm_ref``, ``clip_scale_ref``)
-----------------------------------------------------------------------------------
csrc/adam.cu, per element in fp32 (``adam_math``):  x = g s;  m' = b1 m + (1 - b1) x;  v' = b2 v + ((1 - b2) x) x;
d = sqrt(v') + eps;  p1 = p + p (-lr wd) (skipped when lr wd = 0);  p' = p1 + (-lr bc) (m' / d), bc = sqrt(1 - b2^t) /
(1 - b1^t).  The reference evaluates this in fp64 on the operands the kernel reads (p: the fp32 master, or the bf16
parameter up-cast; g as stored; m, v; the grad scale s) with the hyperparameters as the user's Python doubles, so the bound
pays for their fp32 rounding: e_h = |fp32(h) - h| / |h| for h = b1, b2, eps, lr, wd, bc (computed, not assumed), and for
the kernel's ``1.f - b2``, formed from the already-rounded b2 (exact by Sterbenz for 0.5 <= b < 1):
e_c2 = |(1 - fp32(b2)) - (1 - b2)| / (1 - b2), 9.5e-7 at b2 = 0.98 and 1.3e-5 at 0.999 (e_c1 likewise).  Bounds are
absolute, first order, u = 2^-24, every fp32 operation correctly rounded (no fast-math; ``__fdiv_rn``):
``x``      dx = |g| (u |s| + ds)  (ds: the error of a grad scale that was itself computed, ``clip_scale_ref``)
``m'``     |b1 m| (e_b1 + u) + (1 - b1) (|x| (e_c1 + u) + dx) + u |m'|
``v'``     |b2 v| (e_b2 + u) + (1 - b2) (x^2 (e_c2 + 2u) + 2 |x| dx) + u v'      (every term >= 0: no cancellation)
``sqrt``   sqrt(v') - sqrt(max(v' - dv, 0)) + u sqrt(v'): sqrt is concave, so that fall is larger than the rise
           sqrt(v' + dv) - sqrt(v'); unlike dv / (2 sqrt v') it stays finite where sqrt(v') ~ 0 (|g| ~ eps)
``d``      d_sqrt + eps e_eps + u d
``q``      q = m' / d: dm / d + |q| dd / d + u |q|
``upd``    lr bc q: lr bc dq + |upd| (e_lr + e_bc + 2u)                (step_size = fp32(lr) fp32(bc) rounded, the product)
``p1``     |p lr wd| (e_lr + e_wd + 2u) + u |p1|
``p'``     dp1 + dupd + u |p'|
bf16 parameters: with a master copy the kernel stores bf16_rn(master') from the same register, so p16 == bf16_rn(master')
bit for bit.  Without one, p16 is bf16_rn of the fp32 p', which lies within dp' of the fp64 p'; rounding is monotone, so
p16 must lie between bf16_rn(p' - dp') and bf16_rn(p' + dp'): equal to bf16_rn(p') except where p' is within dp' of a
rounding midpoint, where either neighbour passes.

Gradient norm: ``grad_sumsq_kernel`` runs grid = min(n_chunks, 1056) CTAs of 256 threads; CTA b owns chunks b, b + grid,
...  Each thread adds its <= 32 elements of each chunk (8 float4 or 4 x 8 bf16 vector loads of a full aligned chunk,
else a 256-strided scalar loop) into one fp32 register, squares rounded once (or fused), then 5 shuffle levels and a
serial sum of the 8 warp partials.  Every term is >= 0, so the fp32 sum of squares is off by at most
depth u S, depth = 1 + 32 ceil(n_chunks / grid) + 5 + 8.  The finalize kernel sums the grid partials in fp64 (1024 threads
strided, 5 shuffle levels, 32 warp partials: <= 40 additions, 2^-53 each), sqrt in fp64, rounds to fp32 (u) and
multiplies by fp32(multiply_factor) (u + e_mf): rel(norm) = depth u / 2 + 41 * 2^-53 + 2u + e_mf.  The clip coefficient
min(1, max_norm / (norm + 1e-6)) is off by r (dnorm / (norm + 1e-6) + |fp32(1e-6) - 1e-6| / (norm + 1e-6) + e_max_norm +
k u), k = 2 fp32 roundings in the kernel (the sum, the division); min(1, .) does not increase it.  grad_scale =
multiply_factor coef: |mf| dcoef + |grad_scale| (e_mf + u).
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
    so rstd is off by at most |d var| / (2 (var + eps)) relative to first order, plus 2^-22 for rsqrtf (2 ulp).  The
    E[x^2] / var factor is the cancellation of E[x^2] - mu^2 for rows whose mean is large against their spread.  Where
    |d var| is not small against var + eps (|mean| / std ~ 10^3 over many records), the first-order form no longer holds:
    the computed variance can fall to 0 and rstd rise to 1 / sqrt(eps).  rsqrt is decreasing and convex, so rstd rises by
    at most rsqrt(max(var - |d var|, 0) + eps) / rstd - 1 (exact) and falls by at most |d var| / (2 (var + eps)) (the
    first-order value bounds the fall); ``rel`` is the larger of the two."""
    r = records.reshape(parts, M, 2).double()
    s1, s2 = r[..., 0].sum(0), r[..., 1].sum(0)
    mu, ex2 = s1 / dim, s2 / dim
    var = (ex2 - mu * mu).clamp_min(0.0)
    rstd = (var + eps).rsqrt()
    a1 = r[..., 0].abs().sum(0) / dim
    dmu = parts * U32 * a1 + U32 * mu.abs()
    dvar = (parts + 2) * U32 * (ex2 + 2 * mu.abs() * a1)
    rel = _rstd(var, dvar, eps)[1]
    return mu, rstd, dmu, rel


def gemm_ref(a, w, epi, *, bias=None, colscale=None, gamma=None, resid=None, ln_mu=None, ln_rstd=None, ln_colsum=None,
             ln_partial=None, out_group=0, out_group_stride=0, out_row_offset=0, out_group_valid=0, resid_period=0,
             resid_row_offset=0, stats=False, ln_colsum_err=None, bias_err=None):
    """fp64 result of ``epilogue(a[M,K] @ w[N,K]^T)`` as the kernel defines it (csrc/gemm.h), for the logical rows m < M.

    ``ln_colsum_err`` / ``bias_err``: bounds of the fp32 colsum and bias the kernel reads when the given ``ln_colsum`` /
    ``bias`` are the exact fp64 values of what ``ln_fold`` computed (``ln_fold_ref``).  The epilogue uses each once, so
    the LN step gains rstd |mu| colsum_err and the bias step bias_err in ``extra``.

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
        if ln_colsum_err is not None:
            xe = xe + rstd * mu.abs() * ln_colsum_err.double()[None, :]
    if bias is not None:
        x = x + bias.double()
        xm = xm + bias.double().abs()
        if bias_err is not None:
            xe = xe + bias_err.double()
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


def window_matrix(X, rows, groups, c_pad, taps, group):
    """fp64 window matrix of ``group`` g in the grouped sliding-window GEMM, A_g [rows, taps * c_pad]:
    A_g[r, j * c_pad + c] = X[r + j, g, c] for r < rows, j < taps, c < c_pad.  X holds >= rows + taps - 1 rows of
    groups * c_pad values (any shape with that row layout)."""
    Xg = X.reshape(-1, groups, c_pad)[:rows + taps - 1, group]
    win = Xg.double().unfold(0, taps, 1)                 # [rows, c_pad, taps]: win[r, c, j] = X[r + j, g, c]
    return win.transpose(1, 2).reshape(rows, taps * c_pad)


def grouped_window_ref(X, W, rows, groups, c_pad, taps, n, epi, bias=None):
    """fp64 result of ``grouped_conv1d``: out[:, g*n:(g+1)*n] = gemm_ref(A_g, W[g*n:(g+1)*n], epi, bias=bias[g*n:(g+1)*n]),
    one group's window at a time.  Returns a namespace with y, mag, extra [rows, groups * n]."""
    ys, mags, extras = [], [], []
    for g in range(groups):
        sl = slice(g * n, (g + 1) * n)
        r = gemm_ref(window_matrix(X, rows, groups, c_pad, taps, g), W[sl], epi, bias=bias[sl] if bias is not None else None)
        ys.append(r.y); mags.append(r.mag); extras.append(r.extra)
    return SimpleNamespace(y=torch.cat(ys, 1), mag=torch.cat(mags, 1), extra=torch.cat(extras, 1))


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


# ----------------------------------------------------------------------------------------------------------------------
# row kernels (module docstring, "Row kernels")
# ----------------------------------------------------------------------------------------------------------------------
ERF_ABS = 2.0 ** -19
GELU_REL = ERF_ABS / 2 + 4 * U32
GELU_GRAD_ABS = ERF_ABS / 2 + 2.0 ** -21
GELU_CURV = 0.8                 # max |gelu''(z)| = 2 phi(0) = 0.798
RSQRT_REL = 2.0 ** -22
L2_NORM_REL = (TAU + 2 * U32) / 2 + U32     # relative error of an fp32 row norm (sum of squares, then sqrt)


def gelu_grad(z):
    """exact d/dz gelu(z) = Phi(z) + z phi(z)"""
    return 0.5 * (1 + torch.special.erf(z / 2 ** 0.5)) + z * torch.exp(-0.5 * z * z) / (2 * np.pi) ** 0.5


def _vec(v, n, fill, like):
    return v.double() if v is not None else torch.full((n,), fill, dtype=torch.float64, device=like.device)


def _rstd(var, dvar, eps):
    """rstd and its relative bound, exact in dvar (``ln_stats_ref``)"""
    rstd = (var + eps).rsqrt()
    rise = (var - dvar).clamp_min(0.0).add(eps).rsqrt() / rstd - 1
    return rstd, torch.maximum(rise, dvar / (2 * (var + eps))) + RSQRT_REL


def layernorm_ref(x, gamma, beta, eps, *, gelu=False, prev=None):
    """fp64 LayerNorm (``opb_layernorm``) of the logical rows x [rows, dim] (fp32 or bf16 as given to the kernel), in input
    row order and column order (``ln_layout`` maps them to the output), and its bound.  prev: the fp32 values an
    ``accumulate`` call adds onto (already in input row order).  Returns a namespace with y, err [rows, dim], mu, rstd,
    dmu, rel [rows] (the ``raw`` statistics and their bounds)."""
    X = x.double()
    n = X.shape[1]
    g, b = _vec(gamma, n, 1.0, X), _vec(beta, n, 0.0, X)
    mu = X.mean(1, keepdim=True)
    xc = X - mu
    var = (xc * xc).mean(1, keepdim=True)
    dmu = (TAU + U32) * X.abs().mean(1, keepdim=True)
    rstd, rel = _rstd(var, (TAU + 3 * U32) * var + dmu * dmu, eps)
    xh = xc * rstd
    dxh = rstd * (dmu + U32 * xc.abs()) + xh.abs() * (rel + U32)
    y = xh * g + b
    err = g.abs() * dxh + 2 * U32 * ((xh * g).abs() + b.abs())
    if gelu:
        err = GELU_SLOPE * err + GELU_REL * y.abs()
        y = _gelu(y)
    if prev is not None:
        p = prev.double()
        err = err + U32 * (p.abs() + (y + p).abs())
        y = y + p
    return SimpleNamespace(y=y, err=err, mu=mu[:, 0], rstd=rstd[:, 0], dmu=dmu[:, 0], rel=rel[:, 0])


def ln_layout(rows, dim, *, merge_grid_w=0, row_period=0, row_valid=0, out_period=0, out_row_shift=0, group_in=0,
              group_out=0):
    """where ``opb_layernorm`` stores input row r, column c: (out_row [rows], col [rows, dim], written [rows])."""
    r = torch.arange(rows)
    c = torch.arange(dim)
    orow, col0, written = r, torch.zeros(rows, dtype=torch.long), torch.ones(rows, dtype=torch.bool)
    if merge_grid_w:
        w = merge_grid_w
        xx, yy, bb = r % w, (r // w) % w, r // (w * w)
        orow = (bb * (w // 2) + yy // 2) * (w // 2) + xx // 2
        col0 = ((yy % 2) * 2 + xx % 2) * dim
    if row_period:
        orow = (r // row_period) * out_period + r % row_period + out_row_shift
        written = (r % row_period) < row_valid
    oc = (c // group_in) * group_out + c % group_in if group_in else c
    return orow, col0[:, None] + oc[None, :], written


def layernorm_bwd_ref(x, dy, gamma, beta, eps, *, gelu=False, old=None):
    """fp64 adjoint of ``layernorm_ref`` (``opb_layernorm_bwd``): x, dy [rows, dim] logical rows as the kernel reads them
    (dy already gathered through the merge map), old: the fp32 dx an ``accumulate`` call adds onto.  Returns a namespace
    with dx, dx_err [rows, dim], dgamma, dgamma_err, dbeta, dbeta_err [dim]."""
    X, G = x.double(), dy.double()
    n = X.shape[1]
    g, b = _vec(gamma, n, 1.0, X), _vec(beta, n, 0.0, X)
    mu = X.mean(1, keepdim=True)
    xc = X - mu
    var = (xc * xc).mean(1, keepdim=True)
    rstd = (var + eps).rsqrt()
    xh = xc * rstd
    mean = lambda t: t.mean(1, keepdim=True)
    if gelu:
        dmu = (TAU + U32) * mean(X.abs())
        _, rel = _rstd(var, (TAU + 3 * U32) * var + dmu * dmu, eps)
        dxh = rstd * (dmu + U32 * xc.abs()) + xh.abs() * (rel + U32)
        z = xh * g + b
        dz = g.abs() * dxh + U32 * z.abs()
        gg = gelu_grad(z)
        Gp = G * gg
        dGp = G.abs() * (GELU_CURV * dz + GELU_GRAD_ABS) + U32 * Gp.abs()
        dyg = Gp * g
        ddyg = g.abs() * dGp + U32 * dyg.abs()
        m1, m2 = mean(dyg), mean(dyg * xh)
        dm1 = TAU * mean(dyg.abs()) + mean(ddyg)
        dm2 = TAU * mean((dyg * xh).abs()) + mean(ddyg * xh.abs() + dyg.abs() * dxh)
    else:
        xs = X - X[:, :1]
        A, Q = mean(xs.abs()), mean(xs * xs)
        ms = mean(xs)
        dms = (TAU + U32) * A
        _, rel = _rstd(var, (TAU + 2 * U32) * Q + 2 * A * dms + dms * dms, eps)
        dxh = rstd * (dms + U32 * (xs.abs() + xc.abs())) + xh.abs() * (rel + U32)
        Gp, dGp = G, torch.zeros_like(G)
        dyg = G * g
        ddyg = U32 * dyg.abs()
        m1, m2 = mean(dyg), mean(dyg * xh)
        dm1 = (TAU + U32) * mean(dyg.abs())
        dm2 = rstd * ((TAU + 2 * U32) * mean(dyg.abs() * xs.abs()) + ms.abs() * dm1 + m1.abs() * dms
                      + 2 * U32 * (ms * m1).abs()) + m2.abs() * (rel + U32)
    dx = rstd * (dyg - m1 - xh * m2)
    dt = ddyg + dm1 + xh.abs() * dm2 + m2.abs() * dxh + 2 * U32 * (dyg.abs() + m1.abs() + (xh * m2).abs())
    err = rstd * dt + dx.abs() * (rel + U32)
    if old is not None:
        o = old.double()
        err = err + U32 * (o.abs() + (dx + o).abs())
        dx = dx + o
    return SimpleNamespace(dx=dx, dx_err=err,
                           dgamma=(Gp * xh).sum(0), dgamma_err=(Gp.abs() * dxh + dGp * xh.abs()).sum(0) + (TAU + U32) * (Gp * xh).abs().sum(0),
                           dbeta=Gp.sum(0), dbeta_err=dGp.sum(0) + (TAU + U32) * Gp.abs().sum(0))


def merge_rows(rows, dim, w):
    """(source row, column offset) of dy row r of ``layernorm_bwd(dy_merge_w=w)``: the forward's pixel-merge map"""
    orow, col, _ = ln_layout(rows, dim, merge_grid_w=w)
    return orow, col[:, 0]


def geglu_ref(gl):
    """u = gelu(g) l of bf16 [rows, 2F] = [g | l] -> (u, bound)"""
    F = gl.shape[1] // 2
    g, l = gl.double()[:, :F], gl.double()[:, F:]
    u = _gelu(g) * l
    return u, l.abs() * g.abs() * GELU_REL + 2 * U32 * u.abs()


def geglu_bwd_ref(gl, du):
    """(d[g | l], bound) of u = gelu(g) l for the bf16 upstream gradient du [rows, F]"""
    F = gl.shape[1] // 2
    g, l, d = gl.double()[:, :F], gl.double()[:, F:], du.double()
    dg, dl = d * l * gelu_grad(g), d * _gelu(g)
    return (torch.cat([dg, dl], 1),
            torch.cat([(d * l).abs() * GELU_GRAD_ABS + 3 * U32 * dg.abs(), (d * g).abs() * GELU_REL + U32 * dl.abs()], 1))


def scale_resid_ref(x, o, gamma, row_scale):
    """out = x + row_scale gamma o -> (out, bound)"""
    n = x.shape[1]
    t = _rs(row_scale, x) * _vec(gamma, n, 1.0, x) * o.double()
    out = x.double() + t
    return out, 2 * U32 * (t.abs() + out.abs())


def _rs(row_scale, like):
    return row_scale.double()[:, None] if row_scale is not None else 1.0


def scale_resid_rows(rows, in_period=0, in_valid=0, in_shift=0):
    """dx row read for output row r of ``scale_resid_bwd`` (the gather behind the CLS slot)"""
    r = torch.arange(rows)
    return (r // in_valid) * in_period + in_shift + r % in_valid if in_valid else r


def scale_resid_bwd_ref(dx_rows, o, gamma, row_scale):
    """dx_rows: the dx rows the kernel reads for each output row (``scale_resid_rows``).  Returns a namespace with d_o, d_o_err
    [rows, n], dgamma, dgamma_err, dbias, dbias_err [n] (dbias sums the fp32 values, module docstring)"""
    n = dx_rows.shape[1]
    rd = _rs(row_scale, dx_rows) * dx_rows.double()
    d = rd * _vec(gamma, n, 1.0, dx_rows)
    tg = rd * o.double() if o is not None else torch.zeros_like(rd)
    return SimpleNamespace(d_o=d, d_o_err=2 * U32 * d.abs(), dgamma=tg.sum(0), dgamma_err=(TAU + 2 * U32) * tg.abs().sum(0),
                           dbias=d.sum(0), dbias_err=(TAU + 2 * U32) * d.abs().sum(0))


def colsum_ref(y):
    Y = y.double()
    return Y.sum(0), TAU * Y.abs().sum(0)


def ln_fold_ref(W, g, beta, bias, interleave=0):
    """``opb_ln_fold`` -> namespace rows (destination row of weight row n), wg (bf16 [N, K], bit-exact), colsum, colsum_err,
    bias, bias_err [N] in weight row order"""
    N, K = W.shape
    gf = g.float() if g is not None else torch.ones(K, dtype=torch.float32, device=W.device)
    wg = (W.float() * gf).bfloat16()
    n = torch.arange(N, device=W.device)
    rows = n if interleave == 0 else (n // 128) * 256 + n % 128 + (128 if interleave == 2 else 0)
    Wd = W.double()
    bt = beta.double() if beta is not None else torch.zeros(K, dtype=torch.float64, device=W.device)
    b0 = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=W.device)
    bs = Wd @ bt + b0
    return SimpleNamespace(rows=rows, wg=wg, colsum=wg.double().sum(1), colsum_err=TAU * wg.double().abs().sum(1), bias=bs,
                           bias_err=(TAU + U32) * (Wd.abs() @ bt.abs()) + U32 * (bs.abs() + b0.abs()))


def l2_normalize_bwd_ref(x, dy):
    """fp64 adjoint of y = x / |x| (``opb_l2_normalize_bwd``) on rows of fp32 x, dy -> (dx, bound)"""
    X, G = x.double(), dy.double()
    nrm = X.norm(dim=1, keepdim=True)
    dot = (X * G).sum(1, keepdim=True)
    k = dot / nrm ** 3
    dx = G / nrm - X * k
    rel_n = L2_NORM_REL
    dk = (TAU + U32) * (X * G).abs().sum(1, keepdim=True) / nrm ** 3 + k.abs() * (3 * rel_n + 4 * U32)
    return dx, G.abs() / nrm * (rel_n + 2 * U32) + X.abs() * dk + U32 * ((X * k).abs() + dx.abs())


def scatter_ref(init, dest, src):
    """fp64 result of fp32-atomic scatter-adds: out = init; out[dest[i]] += src[i] (rows of src [m, ...] onto rows of init
    [n, ...]; dest [m] long, entries < 0 skipped) -> (out, bound), bound (count + 1) u (|init| + sum |src|)"""
    I = init.double()
    keep = dest >= 0
    d, s = dest[keep], src.double()[keep]
    out, mag = I.clone(), I.abs().clone()
    cnt = torch.zeros(I.shape[0], dtype=torch.float64, device=I.device)
    out.index_add_(0, d, s)
    mag.index_add_(0, d, s.abs())
    cnt.index_add_(0, d, torch.ones(d.shape[0], dtype=torch.float64, device=I.device))
    cnt = cnt.view(-1, *([1] * (I.dim() - 1)))
    return out, (cnt + 1) * U32 * mag


def window_scatter_ref(dwin, B, t_in, t_out, stride, kw, pad):
    """fp64 col2im of ``opb_window_scatter``: bf16 [groups, B*t_out, kw*cg] -> ([B*t_in, groups*cg], bound)"""
    groups, _, kc = dwin.shape
    cg = kc // kw
    D = dwin.double().view(groups, B, t_out, kw, cg)
    out = torch.zeros(B, t_in, groups, cg, dtype=torch.float64, device=dwin.device)
    mag = torch.zeros_like(out)
    for t in range(t_out):
        for j in range(kw):
            s = t * stride + j - pad
            if 0 <= s < t_in:
                v = D[:, :, t, j].permute(1, 0, 2)
                out[:, s] += v
                mag[:, s] += v.abs()
    return out.reshape(B * t_in, groups * cg), kw * U32 * mag.reshape(B * t_in, groups * cg)


# ----------------------------------------------------------------------------------------------------------------------
# embedding, gather, transpose and ranking kernels (module docstring, "Embedding, gather, transpose and ranking kernels")
# ----------------------------------------------------------------------------------------------------------------------
def text_embed_ref(tokens, table, pos, cls, pad_idx):
    """``opb_text_embed`` -> (x fp32 [B, T+1, D], pad uint8 [B, T+1]): row 0 = cls + pos[0], row s = fp32(table[tok]) +
    pos[s], then (1 - pad) times that (pad rows may come out as -0.0)"""
    B, T = tokens.shape
    emb = torch.cat([cls.float().expand(B, 1, -1), table.float()[tokens]], 1)
    pad = torch.cat([torch.zeros(B, 1, dtype=torch.bool, device=tokens.device), tokens == pad_idx], 1)
    return (emb + pos[:T + 1].float()[None]) * (~pad)[..., None].float(), pad.to(torch.uint8)


def relpos_bias_ref(table, bucket, S, s_pad):
    """``opb_relpos_bias_build`` -> fp32 [H, S, s_pad]: table[bucket[i, j], h] for i, j < S, zero pad columns"""
    H = table.shape[1]
    out = torch.zeros(H, S, s_pad, dtype=torch.float32, device=table.device)
    out[..., :S] = table[bucket[:S, :S]].permute(2, 0, 1)
    return out


def relpos_lut_ref(table, idx):
    """``opb_relpos_lut_build`` -> fp32 [H, L]: lut[h, l] = table[idx[l], h]"""
    return table[idx.long()].t()


def row_gather_ref(src, idx, out_dtype, fill=None, add=None):
    """``opb_row_gather``: out[r] = (src[idx[r]] if idx[r] >= 0 else fill, or 0) + add[r % period], one fp32 addition,
    then rounded to out_dtype.  src [n, dim] (any row pitch), add fp32 [period, dim]."""
    dim = src.shape[1]
    base = torch.zeros(dim, dtype=torch.float32, device=src.device) if fill is None else fill.float()
    v = torch.where((idx >= 0)[:, None], src.float()[idx.clamp_min(0)], base[None])
    if add is not None:
        a = add.reshape(-1, dim)
        v = v + a[torch.arange(idx.numel(), device=src.device) % a.shape[0]]
    return v.to(out_dtype)


def relpos_bias_block_ref(table, bucket, ids, n, lo, canvas):
    """``opb_relpos_bias_block`` on a copy of ``canvas`` [Bb, H, S, s_pad] -> (canvas, written mask):
    canvas[bb, h, lo+i, lo+j] = table[bucket[p_i, p_j], h], p = ids[bb] (-1 -> n - 1) or arange(n)"""
    Bb = canvas.shape[0]
    p = ids.clone() if ids is not None else torch.arange(n, device=canvas.device).expand(Bb, n)
    p = torch.where(p < 0, torch.full_like(p, n - 1), p)
    out = canvas.clone()
    out[:, :, lo:lo + n, lo:lo + n] = table[bucket[p[:, :, None], p[:, None, :]]].permute(0, 3, 1, 2)
    written = torch.zeros(canvas.shape, dtype=torch.bool, device=canvas.device)
    written[:, :, lo:lo + n, lo:lo + n] = True
    return out, written


def transpose_ref(x):
    """``opb_transpose_bf16``: the [cols, rows] transpose of the logical [rows, cols] view, contiguous"""
    return x.t().contiguous()


def l2_normalize_ref(x):
    """fp64 y = x / max(|x|, 1e-12) per row of fp32 x, and its bound (module docstring)"""
    X = x.double()
    y = X / X.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return y, y.abs() * (L2_NORM_REL + f32_rel(1e-12) + 2 * U32)


def order_key(x):
    """int64 key of the order ``topk10_rows`` ranks fp32 values by, unique per column of x [R, C]: fp32 IEEE order with
    -0.0 == +0.0, every NaN above +inf, and among equal values the smaller column first (the larger key)"""
    b = x.float().contiguous().view(torch.int32).long() & 0xFFFFFFFF
    k = torch.where(b >= 2 ** 31, 0xFFFFFFFF - b, b | 2 ** 31)
    k = torch.where(x == 0, torch.full_like(k, 2 ** 31), k)
    k = torch.where(torch.isnan(x), torch.full_like(k, 0xFFFFFFFF), k)
    col = torch.arange(x.shape[1], device=x.device)
    return (k - 2 ** 31) * 2 ** 32 + (2 ** 31 - 1 - col)


def topk10_ref(x):
    """top-10 of every row of fp32 x [R, C] in the order of ``order_key`` (a stable descending sort, NaN first) ->
    (idx int32 [R, 10], val fp32 [R, 10]); slots past C hold -1 and -inf.  The keys are unique, so torch.topk of them has no
    tie to break."""
    R, C = x.shape
    k = min(10, C)
    top = order_key(x).topk(k, dim=1).indices
    idx = torch.full((R, 10), -1, dtype=torch.int64, device=x.device)
    val = torch.full((R, 10), float("-inf"), dtype=torch.float32, device=x.device)
    idx[:, :k] = top
    val[:, :k] = x.gather(1, top)
    return idx.int(), val


def recall_hits_ref(idx, cand_ids, row_ids):
    """``opb_recall_hits`` -> [hits@1, hits@5, hits@10]: rows whose id is among the ids of their first 1 / 5 / 10 ranked
    candidates (column -1 never hits)"""
    g = idx.long()
    ids = torch.where(g >= 0, cand_ids[g.clamp_min(0)], torch.full_like(g, -2 ** 62))
    eq = ids == row_ids[:, None]
    return [int(eq[:, :k].any(1).sum()) for k in (1, 5, 10)]


def topk_within(z, dz, idx):
    """Rows whose returned list ``idx`` [R, 10] is a top-10 of some matrix within ``dz`` of the fp64 similarity z [R, C]
    (``argmax_ok`` for a ranked list): ten distinct columns in range, each returned entry no smaller than the next one
    minus both their errors, and no column left out above the 10th returned one by more than both their errors."""
    R, C = z.shape
    g = idx.long()
    valid = ((g >= 0) & (g < C)).all(1) & (g.sort(1).values.diff(dim=1) != 0).all(1)
    g = g.clamp(0, C - 1)
    zi, di = z.gather(1, g), dz.gather(1, g)
    ordered = (zi[:, :-1] >= zi[:, 1:] - di[:, :-1] - di[:, 1:]).all(1)
    left_out = torch.ones(R, C, dtype=torch.bool, device=z.device).scatter_(1, g, False)
    beats = left_out & (z > zi[:, -1:] + dz + di[:, -1:])
    return valid & ordered & ~beats.any(1)


def recall_ref(z, dz, cand_ids, row_ids):
    """fp64 Recall@{1,5,10} hit counts of the similarity z [R, C >= 11] and, per k, the number of rows whose k-th and
    (k+1)-th largest values lie within twice the row's largest error, the only rows whose hit can differ"""
    top = z.topk(11, dim=1)
    hits = recall_hits_ref(top.indices[:, :10], cand_ids, row_ids)
    margin = 2 * dz.max(1).values
    near = [int((top.values[:, k - 1] - top.values[:, k] <= margin).sum()) for k in (1, 5, 10)]
    return hits, near


# ----------------------------------------------------------------------------------------------------------------------
# optimizer (module docstring, "Optimizer")
# ----------------------------------------------------------------------------------------------------------------------
ADAM_CHUNK = 8192               # opb_adam_chunk_elems()
NORM_GRID_CAP = 132 * 8         # grad_sumsq_kernel: grid = min(n_chunks, 1056)
U64 = 2.0 ** -53


def f32_rel(x):
    """relative error of rounding the Python double x to fp32 (0 for x = 0)"""
    x = float(x)
    return 0.0 if x == 0 else abs(float(np.float32(x)) - x) / abs(x)


def bias_correction(t, betas):
    """sqrt(1 - b2^t) / (1 - b1^t) in Python doubles, as the optimizers pass it to the kernel"""
    b1, b2 = betas
    return (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)


def adam_ref(p, g, m, v, *, t, lr, wd, betas, eps, grad_scale=None, grad_scale_err=0.0):
    """fp64 Adam step of ``adam_math`` on the operands the kernel reads (p: fp32 master or bf16 parameter; g fp32 or bf16;
    m, v fp32), t the step count after this step, lr including lr_scale, grad_scale a Python float (None = 1) with the
    absolute error ``grad_scale_err`` of its computed value.  Returns a namespace with m, m_err, v, v_err, p, p_err (the fp32
    p' of the master copy or an fp32 parameter) and upd, upd_err (lr bc m' / d)."""
    b1, b2 = betas
    assert 0.5 <= b1 < 1 and 0.5 <= b2 < 1, "1 - fp32(b) is exact only for 0.5 <= b < 1"
    u = U32
    P, G, M0, V0 = (x.double() for x in (p, g, m, v))
    s = 1.0 if grad_scale is None else float(grad_scale)
    c1, c2 = 1 - b1, 1 - b2
    e_c1 = abs((1 - float(np.float32(b1))) - c1) / c1
    e_c2 = abs((1 - float(np.float32(b2))) - c2) / c2
    X = G * s
    dX = G.abs() * (u * abs(s) + grad_scale_err)
    Mn = b1 * M0 + c1 * X
    dM = (b1 * M0).abs() * (f32_rel(b1) + u) + c1 * (X.abs() * (e_c1 + u) + dX) + u * Mn.abs()
    Vn = b2 * V0 + c2 * X * X
    dV = (b2 * V0).abs() * (f32_rel(b2) + u) + c2 * (X * X * (e_c2 + 2 * u) + 2 * X.abs() * dX) + u * Vn.abs()
    R = Vn.sqrt()
    dR = R - (Vn - dV).clamp_min(0.0).sqrt() + u * R
    D = R + eps
    dD = dR + eps * f32_rel(eps) + u * D
    Q = Mn / D
    dQ = dM / D + Q.abs() * dD / D + u * Q.abs()
    bc = bias_correction(t, betas)
    Upd = lr * bc * Q
    dUpd = lr * bc * dQ + Upd.abs() * (f32_rel(lr) + f32_rel(bc) + 2 * u)
    if float(np.float32(wd)) * float(np.float32(lr)) != 0.0:
        P1 = P * (1 - lr * wd)
        dP1 = (P * lr * wd).abs() * (f32_rel(lr) + f32_rel(wd) + 2 * u) + u * P1.abs()
    else:
        P1, dP1 = P, torch.zeros_like(P)
    Pn = P1 - Upd
    dPn = dP1 + dUpd + u * Pn.abs()
    return SimpleNamespace(m=Mn, m_err=dM, v=Vn, v_err=dV, p=Pn, p_err=dPn, upd=Upd, upd_err=dUpd)


def bf16_param_check(got, ref, err, what="bf16 parameter"):
    """bf16 parameter written without a master copy: bf16_rn of some fp32 value within ``err`` of ``ref``, i.e. between
    bf16_rn(ref - err) and bf16_rn(ref + err) (rounding is monotone).  Returns the number of elements where both
    neighbours were allowed (ref within err of a rounding midpoint)."""
    lo = (ref - err).bfloat16().double()
    hi = (ref + err).bfloat16().double()
    g = got.double()
    bad = ~((g >= lo) & (g <= hi))
    n_bad = int(bad.sum().item())
    if n_bad:
        i = int(bad.flatten().nonzero()[0].item())
        raise AssertionError(f"{what}: {n_bad} of {g.numel()} elements outside the bound; first at {i}: got "
                             f"{g.flatten()[i].item()!r}, allowed [{lo.flatten()[i].item()!r}, {hi.flatten()[i].item()!r}] "
                             f"(ref {ref.flatten()[i].item()!r} +- {err.flatten()[i].item():.3e})")
    return int((lo != hi).sum().item())


def norm_chunks(numels, chunk=ADAM_CHUNK):
    """the chunk table of ``optim.adam._Table``: [(tensor index, element offset, length)] in table order"""
    return [(i, o, min(chunk, n - o)) for i, n in enumerate(numels) for o in range(0, n, chunk)]


def clip_scale_ref(norm, norm_err, multiply_factor, max_norm, roundings=2):
    """grad_scale = multiply_factor * min(1, max_norm / (norm + 1e-6)) (multiply_factor alone for max_norm <= 0) from an fp64
    norm with absolute error ``norm_err``; ``roundings``: fp32 roundings between the norm and the coefficient (2 in the
    kernel: the sum and the division).  -> (grad_scale, bound)"""
    mf = float(multiply_factor)
    if max_norm <= 0:
        return mf, abs(mf) * f32_rel(mf)
    den = norm + 1e-6
    r = max_norm / den
    dr = r * ((norm_err + abs(float(np.float32(1e-6)) - 1e-6)) / den + f32_rel(max_norm) + roundings * U32)
    gs = mf * (1.0 if r >= 1.0 else r)          # clamp(max=1), keeping a NaN
    return gs, abs(mf) * dr + abs(gs) * (f32_rel(mf) + U32)


def grad_norm_ref(grads, multiply_factor=1.0, max_norm=0.0, chunk=ADAM_CHUNK):
    """fp64 ``opb_grad_norm_clip`` over the gradients in table order (module docstring, "Optimizer").  Returns a namespace
    with n_chunks, grid, depth (of the fp32 sum of squares), sumsq, norm (multiply_factor ||g||_2), norm_err, scale
    (out[1]) and scale_err."""
    n_chunks = len(norm_chunks([x.numel() for x in grads], chunk))
    grid = min(n_chunks, NORM_GRID_CAP)
    depth = 1 + 32 * -(-n_chunks // grid) + 5 + 8
    S = sum(float(x.double().square().sum()) for x in grads)
    raw = S ** 0.5
    mf = float(multiply_factor)
    N = mf * raw
    dN = abs(N) * (depth * U32 / 2 + 41 * U64 + 2 * U32 + f32_rel(mf))
    gs, dgs = clip_scale_ref(N, dN, mf, max_norm)
    return SimpleNamespace(n_chunks=n_chunks, grid=grid, depth=depth, sumsq=S, norm=N, norm_err=dN, scale=gs,
                           scale_err=dgs)
