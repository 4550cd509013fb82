"""CPU checks of the multi-scale deformable attention reference (tests/msda_ref.py) and of MSDeformAttn's host logic against
the reference module's fixture (tests/golden/msda.pt, oracle/make_golden_msda.py)."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import msda_ref as R  # noqa: E402
from kernel_ref import assert_within  # noqa: E402

from one_peace_b200.vision.ms_deform_attn import MSDeformAttn  # noqa: E402

GOLD = torch.load(os.path.join(HERE, "golden", "msda.pt"))
MISTAKES = ["align_corners", "swap_norm", "softmax_per_level", "clamp", "start_off_by_one"]
# each planted mistake must exceed the kernel's error bound by at least this factor somewhere
MISTAKE_FACTOR = 1000.0


def _proj_weights(st):
    w = torch.cat([st["sampling_offsets.weight"], st["attention_weights.weight"]])
    b = torch.cat([st["sampling_offsets.bias"], st["attention_weights.bias"]])
    return w, b


def _compose(c):
    """The module in fp64 around msda_ref: output and every gradient for the fixture's cotangent."""
    st = {k: v.double() for k, v in c["state"].items()}
    N, Lq, d = c["query"].shape
    S_in = c["input_flatten"].shape[1]
    H, P = c["config"]["n_heads"], c["config"]["n_points"]
    q = c["query"].double().reshape(N * Lq, d)
    x = c["input_flatten"].double().reshape(N * S_in, d)
    wp, bp = _proj_weights(st)
    value = x @ st["value_proj.weight"].T + st["value_proj.bias"]
    proj = q @ wp.T + bp
    ref = c["reference_points"].reshape(N * Lq, -1, 2)
    core = R.forward(value, proj, ref, c["shapes"], c["starts"], N, Lq, H, P)
    y = core @ st["output_proj.weight"].T + st["output_proj.bias"]
    dy = c["cotangent"].double().reshape(N * Lq, d)
    dcore = dy @ st["output_proj.weight"]
    dv, dp = R.backward(value, proj, ref, dcore, c["shapes"], c["starts"], N, Lq, H, P)
    n_off = 2 * H * len(c["shapes"]) * P
    dW, db = dp.T @ q, dp.sum(0)
    grads = {"sampling_offsets.weight": dW[:n_off], "sampling_offsets.bias": db[:n_off],
             "attention_weights.weight": dW[n_off:], "attention_weights.bias": db[n_off:],
             "value_proj.weight": dv.T @ x, "value_proj.bias": dv.sum(0),
             "output_proj.weight": dy.T @ core, "output_proj.bias": dy.sum(0)}
    return dict(output=y.view(N, Lq, d), d_query=(dp @ wp).view(N, Lq, d), d_input_flatten=(dv @ st["value_proj.weight"]).view(
        N, S_in, d), grads=grads, value=value, proj=proj, ref=ref)


@pytest.mark.parametrize("case", sorted(GOLD["cases"]))
def test_msda_ref_matches_reference_module(case):
    c = GOLD["cases"][case]
    got = _compose(c)
    for key in ("output", "d_query", "d_input_flatten"):
        want = c[key]
        assert (got[key] - want).abs().max().item() <= 1e-12 * (want.abs().max().item() + 1), key
    for k, want in c["grads"].items():
        assert (got["grads"][k] - want).abs().max().item() <= 1e-12 * (want.abs().max().item() + 1), k


@pytest.mark.parametrize("case", sorted(GOLD["cases"]))
def test_module_names_shapes_and_init(case):
    c = GOLD["cases"][case]
    torch.manual_seed(0)
    m = MSDeformAttn(**c["config"])
    assert [(k, tuple(p.shape)) for k, p in m.named_parameters()] == GOLD["keys"][case]
    assert m.im2col_step == 64
    sd = m.state_dict()
    assert list(sd) == list(GOLD["init"][case])
    for k, v in GOLD["init"][case].items():
        assert torch.equal(sd[k], v), k


def _inputs(N=1, Lq=3, d=64, shapes=((2, 3),), L_ref=1):
    len_in = sum(h * w for h, w in shapes)
    return torch.randn(N, Lq, d), torch.rand(N, Lq, L_ref, 2), torch.randn(N, len_in, d)


def test_refusals_before_any_kernel():
    m = MSDeformAttn(d_model=64, n_levels=1, n_heads=2, n_points=4)
    q, r, x = _inputs()
    with pytest.raises(NotImplementedError, match="padding"):
        m(q, r, x, [(2, 3)], [0], torch.zeros(1, 6, dtype=torch.bool))
    with pytest.raises(NotImplementedError, match="boxes"):
        m(q, torch.rand(1, 3, 1, 4), x, [(2, 3)], [0])
    with pytest.raises(ValueError):
        m(q, torch.rand(1, 3, 1, 3), x, [(2, 3)], [0])
    with pytest.raises(NotImplementedError, match="32 channels"):
        MSDeformAttn(d_model=64, n_levels=1, n_heads=4, n_points=4)(q, r, x, [(2, 3)], [0])
    with pytest.raises(NotImplementedError, match="32 channels"):
        MSDeformAttn(d_model=64, n_levels=1, n_heads=2, n_points=4, ratio=0.5)(q, r, x, [(2, 3)], [0])
    with pytest.raises(NotImplementedError, match="levels"):
        MSDeformAttn(d_model=64, n_levels=5, n_heads=2, n_points=4)(q, r, x, [(2, 3)], [0])
    with pytest.raises(NotImplementedError, match="points"):
        MSDeformAttn(d_model=64, n_levels=1, n_heads=2, n_points=9)(q, r, x, [(2, 3)], [0])
    with pytest.raises(NotImplementedError, match="reference points"):
        m(q, r.requires_grad_(True), x, [(2, 3)], [0])
    with pytest.raises(NotImplementedError, match="dtype"):
        m(q.half(), torch.rand(1, 3, 1, 2), x, [(2, 3)], [0])
    with pytest.raises(NotImplementedError, match="dtype"):
        m(q, torch.rand(1, 3, 1, 2), x.double(), [(2, 3)], [0])


def test_level_layout_checks():
    m = MSDeformAttn(d_model=64, n_levels=2, n_heads=2, n_points=4)
    q, r, x = _inputs(shapes=((2, 3), (1, 2)))
    with pytest.raises(ValueError, match="Len_in"):
        m(q, r, x, torch.tensor([[2, 3], [1, 3]]), torch.tensor([0, 6]))
    with pytest.raises(ValueError, match="running sum"):
        m(q, r, x, torch.tensor([[2, 3], [1, 2]]), torch.tensor([0, 5]))
    with pytest.raises(ValueError, match="pairs"):
        m(q, r, x, [(2, 3)], [0])
    with pytest.raises(ValueError, match="reference_points"):
        m(q, torch.rand(1, 3, 3, 2), x, [(2, 3), (1, 2)], [0, 6])


def test_planted_mistakes_exceed_the_bound():
    """Each mistake, made in the fp64 reference, lands far outside the error bound the kernel is held to."""
    c = GOLD["cases"]["injector"]
    g = _compose(c)
    N, Lq, _ = c["query"].shape
    H, P = c["config"]["n_heads"], c["config"]["n_points"]
    out, bound = R.forward(g["value"], g["proj"], g["ref"], c["shapes"], c["starts"], N, Lq, H, P, with_bound=True)
    for mistake in MISTAKES:
        bad = R.forward(g["value"], g["proj"], g["ref"], c["shapes"], c["starts"], N, Lq, H, P, mistake=mistake)
        with pytest.raises(AssertionError):
            assert_within(bad, out, bound, MISTAKE_FACTOR, torch.bfloat16, what=mistake)
