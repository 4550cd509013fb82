"""fp64 restatement of the classification metrics (metrics/accuracy.py, metrics/map.py) and the error bounds of
csrc/metrics.cu, with no scikit-learn import.

argmax_ref: torch.argmax's rules per row: a NaN is the maximum (the first NaN wins), otherwise the first index of the
maximum; -0.0 == +0.0.

average_precision_ref: scikit-learn's average precision per class.  Sort by probability, descending; group equal
probabilities; with TP_g and FP_g counted through group g (exact integers),
    AP = sum_g (pos_g / P) * TP_g / (TP_g + FP_g)      (0 when P = 0, as scikit-learn 1.9 returns)
The terms are formed and summed in extended precision (np.longdouble, 64-bit significand) and divided by P last, so the
restatement is exact to a few 2^-64 relative, far below the bounds below.

Error contract (u = 2^-53), derived for the kernel's arithmetic:
* hyp, hard-label counts and the probabilities (hence the tie groups) are exact: there is no rounding in a comparison, a
  count or a bit-identical sigmoid.
* opb_average_precision forms t_g = pos_g * fl(TP_g / cnt_g) (two roundings: |t_g - exact| <= 2 u t_g), sums the G nonzero
  terms (at most G - 1 additions of nonzero operands, each rounding by at most u times the running sum, which is at most
  sum_g t_g = AP P) and divides by P (one more rounding), so |AP - exact| <= (2 + (G - 1) + 1) u AP + O(u^2) <= (G + 4) u
  since AP <= 1.  scikit-learn forms recall differences and NumPy pairwise sums instead; against it allow twice that.
* map: the C per-class errors average to at most their mean bound; the class-order sum of C terms adds (C - 1) u times the
  sum and the division by C one more rounding, so mean(AP bound) + (C + 1) u bounds |map - exact| (map <= 1).
* Soft score_sum: an fp64 sum of n fp32 scores in any fixed order is within (n - 1) u sum |s|; (n + 2) u sum |s| is allowed.
  The reference accumulates in fp32 (per-batch sums added into an fp32 counter: n + batches roundings of at most 2^-24 times
  the running sum), so against it (n + batches + 2) 2^-24 sum |s| is allowed.
"""
import numpy as np

U = 2.0 ** -53
U32 = 2.0 ** -24


def argmax_ref(x, mistake=None):
    """torch.argmax(x, 1) of an [n, C] array.  mistake: 'last_index' (the last maximal index wins) or 'nan_ignored' (NaN
    never wins)."""
    x = np.asarray(x, dtype=np.float64)
    nan = np.isnan(x)
    if mistake == "nan_ignored":
        nan = np.zeros_like(nan)
    xm = np.where(np.isnan(x), -np.inf, x)
    rowmax = xm.max(1, keepdims=True)
    hit = np.where(nan.any(1, keepdims=True), nan, xm == rowmax)
    if mistake == "last_index":
        return (x.shape[1] - 1 - hit[:, ::-1].argmax(1)).astype(np.int64)
    return hit.argmax(1).astype(np.int64)


def hard_hits(hyp, targets):
    """Accuracy's hard-label row scores: torch.eq of the int64 hypothesis with int64 or fp32 labels."""
    t = np.asarray(targets)
    if t.dtype.kind == "f":
        return (hyp.astype(np.float32) == t).astype(np.float64)
    return (hyp == t).astype(np.float64)


def average_precision_ref(probs, labels, mistake=None):
    """-> (AP fp64 [C], groups G int64 [C], positives P int64 [C]).  probs [N, C] are compared as given (fp32 or fp64);
    labels {0, 1}.  mistake: 'position' (ties broken by position instead of grouped), 'precision_first' (precision read at a
    group's first element), 'recall_over_N' (recall over N instead of P)."""
    probs = np.asarray(probs)
    labels = np.asarray(labels).astype(np.int64)
    N, C = probs.shape
    ap = np.zeros(C)
    G = np.zeros(C, np.int64)
    P = labels.sum(0).astype(np.int64)
    for c in range(C):
        p = probs[:, c].astype(np.float64)
        order = np.argsort(-p, kind="stable")
        ps, ys = p[order], labels[order, c]
        if mistake == "position":
            ends = np.arange(N)
        else:
            ends = np.flatnonzero(np.r_[ps[1:] != ps[:-1], True])
        cum = np.cumsum(ys)
        tp = cum[ends]
        starts = np.r_[0, ends[:-1] + 1]
        pos = tp - np.r_[0, tp[:-1]]
        if mistake == "precision_first":
            prec = cum[starts].astype(np.longdouble) / (starts + 1).astype(np.longdouble)
        else:
            prec = tp.astype(np.longdouble) / (ends + 1).astype(np.longdouble)
        G[c] = len(ends)
        denom = N if mistake == "recall_over_N" else P[c]
        if P[c] == 0:
            continue
        ap[c] = float(np.sum(pos.astype(np.longdouble) * prec) / np.longdouble(denom))
    return ap, G, P


def map_ref(ap, P, mistake=None):
    """The mean over classes of the restated AP (np.mean of map.py:43); mistake 'drop_no_positive' leaves classes without
    positives out of the mean."""
    a = np.asarray(ap, dtype=np.longdouble)
    if mistake == "drop_no_positive":
        a = a[np.asarray(P) > 0]
    return float(a.sum() / len(a))


def ap_bound(G):
    return (np.asarray(G, dtype=np.float64) + 4.0) * U


def map_bound(G):
    G = np.asarray(G, dtype=np.float64)
    return float(ap_bound(G).mean() + (len(G) + 1) * U)


def soft_sum_exact(scores):
    import math
    return math.fsum(np.asarray(scores, dtype=np.float64).tolist())


def soft_sum_bound(scores):
    s = np.asarray(scores, dtype=np.float64)
    return (len(s) + 2) * U * float(np.abs(s).sum())


def soft_sum_bound_fp32(scores, batches):
    s = np.asarray(scores, dtype=np.float64)
    return (len(s) + batches + 2) * U32 * float(np.abs(s).sum())


def sigmoid_f32(x):
    """1 / (1 + e) in fp32 operations with e = exp(-x) rounded to fp32: the route of torch.sigmoid's fp32 formula, elementwise
    (a function of x, within a few ulp of CUDA's expf-based result; it saturates to 1.0f above about 16.6 as that does)."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over="ignore"):
        e = np.exp(-x.astype(np.float64)).astype(np.float32)
        return (np.float32(1.0) / (np.float32(1.0) + e)).astype(np.float32)


def sigmoid_f64(x):
    """The planted mistake: the sigmoid in fp64, which splits the saturated group of fp32 probabilities."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-x))
