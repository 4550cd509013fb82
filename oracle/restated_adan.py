"""TEST INFRASTRUCTURE — the CPU oracle of the Adan optimizer, beside oracle/restated.py (its ``adam_step``).  Not product
code; only tests/ and scripts/ may import it.

PINNING: tests/test_adan_host_logic.py checks ``adan_step`` against tests/golden/adan.pt, produced by executing the
reference's unmodified optim/adan.py (oracle/make_golden_adan.py, run where the reference source tree exists).

All file:line citations are relative to the reference's one_peace/.
"""
import math


def adan_step(p, g, m, n, v, pre_grad, step, lr, betas, eps, weight_decay, no_prox=False):
    """optim/adan.py:197-220 (python Adan) for one parameter.  fp32 tensors; p, m (exp_avg), n (exp_avg_diff) and v
    (exp_avg_sq) are updated in place; `pre_grad` is the previous gradient, or None on the parameter's first step or at
    group step 1 (diff = 0); `step` is the GROUP's already-incremented step count.  Returns the new pre_grad (a copy of g)."""
    b1, b2, b3 = betas
    bc1, bc2, bc3 = 1.0 - b1 ** step, 1.0 - b2 ** step, 1.0 - b3 ** step
    if pre_grad is None or step == 1:
        pre_grad = g
    diff = g - pre_grad
    u = g + b2 * diff
    m.mul_(b1).add_(g, alpha=1 - b1)
    n.mul_(b2).add_(diff, alpha=1 - b2)
    v.mul_(b3).addcmul_(u, u, value=1 - b3)
    denom = (v.sqrt() / math.sqrt(bc3)).add_(eps)
    upd = (m / bc1 + b2 * n / bc2).div_(denom)
    if no_prox:
        p.mul_(1 - lr * weight_decay)
        p.add_(upd, alpha=-lr)
    else:
        p.add_(upd, alpha=-lr)
        p.div_(1 + lr * weight_decay)
    return g.clone()
