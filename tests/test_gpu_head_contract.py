"""GPU: the classification heads and criteria (``ClassifyHeadFn``, ``ClassifyLossFn``, ``RefcocoLossFn``, ``VitHeadFn`` of
one_peace_b200/autograd_classify.py) and the pretraining-path Functions (``BlockBiasFn``, ``RowGatherFn``, ``ZeroPadFn``,
``LinearFn``, ``FinalNormFn``, ``DclLossFn`` of one_peace_b200/autograd_general.py), forward and adjoint, stage by stage,
against the fp64 references and per-element bounds of tests/head_ref.py, at the model's widths (d = 1536, 24 heads,
head_scale_ratio 2).

The case builders are the CPU test's (tests/test_head_ref.py), run on the kernels behind its ``Recorder``, so each
backward stage is checked from the bf16 intermediate the device handed it.  Where the reference is exactly zero (the CLS
rows of dfeats, padded keys, the classifier's padded columns, the ViT CLS form's rows past the CLS row, padded rows,
student rows the DCL loss does not select, unused table rows) the bound is zero, so the device value must be exactly zero.

Every output must use at most its whole bound and, unless it can come out exact (a copy) or is a column reduction, at
least FLOOR of it: a bound that is never approached would not notice a mistake.  Each case runs twice, and every output
not summed by fp32 atomics must repeat bit for bit.  Each test prints the shares it saw (pytest -s)."""
import pytest
import torch

import test_head_ref as C
from test_classify_host_logic import HARD, HINGE, MULTI, SOFT

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
FLOOR = 1e-3


def check(what, case, args):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    r = C.run(case, args, kernels, dev="cuda")
    print(f"\n{what}: largest share of each bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(r.shares.items())))
    over = {k: v for k, v in r.shares.items() if not v <= 1.0}
    assert not over, f"{what}: outside the bound (share of the bound): {over}"
    low = {k: v for k, v in r.shares.items() if v < FLOOR and k not in r.exact and k not in r.reductions}
    assert not low, f"{what}: bound never approached (share below {FLOOR}): {low}"
    again = C.run(case, args, kernels, dev="cuda").outputs
    differ = [k for k, v in r.outputs.items() if k not in r.atomic and not torch.equal(v, again[k])]
    assert not differ, f"{what}: not bit-identical on a second run: {differ}"


D, H_RATIO = 1536, 2
CASES = {
    # ClassifyHeadFn
    "image head 384^2": ("classify", dict(B=4, S=577, d=D, ratio=H_RATIO, n_cls=1000, pooler=False, pads=None, seed=100)),
    "text head, pooler, ragged pads": ("classify", dict(B=8, S=73, d=D, ratio=H_RATIO, n_cls=3129, pooler=True,
                                                         pads=((1, 40), (3, 9), (5, 64), (7, 2)), seed=101)),
    "two images, pooler": ("classify", dict(B=4, S=577, d=D, ratio=H_RATIO, n_cls=2, pooler=True, two=True, pads=None,
                                            seed=102)),
    # VitHeadFn
    "ViT pooled S=577": ("vit", dict(B=8, S=577, d=D, n_cls=1000, pool=True, seed=103)),
    "ViT CLS S=1025": ("vit", dict(B=4, S=1025, d=D, n_cls=1000, pool=False, seed=104)),
    # ClassifyLossFn, RefcocoLossFn
    "classify loss hard 1000 strided": ("loss", dict(mode=HARD, rows=64, C=1000, ld=1008, seed=105)),
    "classify loss soft 3129 bf16": ("loss", dict(mode=SOFT, rows=64, C=3129, ld=3136, dtype=BF, eps=0.0, seed=106)),
    "classify loss multi-label 200": ("loss", dict(mode=MULTI, rows=64, C=200, ld=200, eps=0.0, seed=107)),
    "classify loss hinge": ("loss", dict(mode=HINGE, rows=64, C=1, ld=8, num_choices=4, eps=0.0, seed=108)),
    "refcoco loss": ("refcoco", dict(B=64, ld=8, ns=64, seed=109)),
    # autograd_general
    "DCL 16 x 65 rows": ("dcl", dict(B=16, S=65, d=D, pad_from=(None, 30, 61, None, 6) * 3 + (None,), seed=110)),
    "row gather canvas": ("gather", dict(form="canvas", B=8, S=257, K=65, d=768, seed=111)),
    "row gather preserve": ("gather", dict(form="preserve", B=8, S=257, K=65, d=D, seed=112)),
    "row gather audio repeat": ("gather", dict(form="repeat", B=8, S=257, K=65, d=D, seed=113)),
    "zero pad": ("zero_pad", dict(B=8, S=330, d=D, seed=114)),
    "block bias vl": ("block_bias", dict(H=24, n_t=73, n_i=65, Bb=8, L=257, seed=115)),
    "linear decoder embed": ("linear", dict(rows=8 * 257, n_in=D, n_out=768, seed=116)),
    "linear mask head bf16": ("linear", dict(rows=8 * 257, n_in=768, n_out=D, x_dtype=BF, seed=117)),
    "final norm": ("final_norm", dict(rows=8 * 257, d=D, seed=118)),
}


@pytest.mark.parametrize("what", list(CASES))
def test_head_contract(what):
    case, args = CASES[what]
    check(what, case, args)
