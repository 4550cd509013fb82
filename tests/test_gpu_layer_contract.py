"""GPU: the encoder stack of the training path (``EncoderStackFn``, ``layer_forward``, ``layer_backward`` of
one_peace_b200/autograd.py) at model width (d = 1536, 24 heads, F = 6144, two layers), forward and adjoint, stage by
stage, against the fp64 references and per-element bounds of tests/layer_ref.py.

The case builders are the CPU test's (tests/test_layer_ref.py), run on the kernels instead of their emulation: a text
pass with mixed key padding (one key live in a sample) and one shared LUT-form table, an image pass with one table per
layer, a 257-token pass (dense attention backward), concatenated text + image and text + audio sequences with per-sample
and batch-shared canvases, the decoder (no LayerScale, no bias), drop-path, and bf16 parameters; under kept activations,
the layer-by-layer recompute, and the recompute after the fused-LayerNorm forward.

Every output must use at most its whole bound and, unless it is exact (a row gather) or a column reduction (bias,
LayerNorm and LayerScale gradients, the bias tables), at least FLOOR of it.  Every case runs twice and repeats bit for
bit, except the bias-table gradients, which are summed with fp32 atomics.  Kept activations and the layer-by-layer
recompute give the same dx0 and parameter gradients bit for bit.  Each test prints the shares it saw (pytest -s)."""
import pytest
import torch

import test_layer_ref as C

pytestmark = pytest.mark.gpu
FLOOR = 1e-3
WIDE = dict(d=1536, H=24, F=6144, L=2, dev="cuda")
CASES = {
    "text": dict(form="text", S=72),
    "image": dict(form="image"),
    "long": dict(form="long"),
    "vl": dict(form="vl", parts=[("text", 72), ("image", 197)]),
    "al": dict(form="al", parts=[("text", 72), ("audio", 120)]),
    "decoder": dict(form="decoder", parts=[("text", 72), ("image", 197)]),
    "drop_path": dict(form="text", S=72, drop_path=0.5, seed=5),
    "text_bf16": dict(form="text", S=72, p_dtype=torch.bfloat16, seed=7),
}
FUSED = ("text", "image", "long")          # single-modality, every bias with a LUT form, no drop-path
RUNS = {}


def kernels():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels as K
    return K


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def run(case, policy):
    if (case, policy) not in RUNS:
        r = C.stack_case(kernels(), policy=policy, **{**WIDE, **CASES[case]})
        RUNS[(case, policy)] = C.NS(shares=r.shares, exempt=r.exempt, got=r.got)
    return RUNS[(case, policy)]


def check(what, r):
    sh = r.shares
    print(f"\n{what}: largest share of each bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(sh.items())))
    over = {k: v for k, v in sh.items() if not v <= 1.0}
    assert not over, f"{what}: outside the bound (share of the bound): {over}"
    low = {k: v for k, v in sh.items() if v < FLOOR and k not in r.exempt}
    assert not low, f"{what}: bound never approached (share below {FLOOR}): {low}"


@pytest.mark.parametrize("policy", ["keep", "recompute", "fused"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_stack(case, policy):
    if policy == "fused" and case not in FUSED:
        pytest.skip("the fused forward runs single-modality passes without drop-path")
    r = run(case, policy)
    check(f"{case} / {policy}", r)
    again = C.stack_case(kernels(), policy=policy, **{**WIDE, **CASES[case]})
    for k, v in r.got.items():
        if not k.endswith("dbias"):
            assert torch.equal(bits(v), bits(again.got[k])), f"{case} / {policy}: {k} differs between two runs"


@pytest.mark.parametrize("case", sorted(CASES))
def test_keep_equals_recompute(case):
    """the same gradients whether the activations were kept or recomputed layer by layer (bias tables aside: fp32
    atomics).  A single-modality recompute attends with the dense tables, the kept forward with their LUT form, which
    the attention kernels read to the same bits."""
    a, b = run(case, "keep"), run(case, "recompute")
    names = ["dx0"] + [k for k in a.got if k.startswith("L") and "." in k and k.count(".") <= 2
                       and k.split(".")[1] not in ("fwd", "recompute") and k.split(".")[-1] in C.LR.SHARED + C.LR.FFN]
    assert len(names) > 20
    for k in names:
        assert torch.equal(bits(a.got[k]), bits(b.got[k])), f"{case}: {k} differs between keep and recompute"
