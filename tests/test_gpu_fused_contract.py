"""GPU: the fused-LayerNorm layer loops of inference (``TransformerEncoder.run_fused``, ``TransformerEncoderLayer.
forward_rows_fused``, the detection backbone's ``OnePeace.forward``, ``VideoLayer.forward_video``) at model width (d = 1536, 24 heads, F = 6144, two layers), stage by stage, against the fp64
references and per-element bounds of tests/fused_ref.py.

The case builders are the CPU test's (tests/test_fused_ref.py), run on the kernels instead of their emulation: a text pass
with mixed key padding (one key live in a sample) and one shared LUT-form table, the same at batch 2 (M = 144 <= 256: the
split-K workspace path of every GEMM), an image pass with one table per layer, an audio pass (the audio FFN), and a
257-token pass on the dense table (``attention`` with records); the detection backbone's forward on a 16 x 16 grid of two
images (the window-major gathers, layer 0 in 8 x 8 windows, layer 1 global, the decomposed relative-position terms); and
the video backbone's layer loop on one clip of 16 frames of 257 tokens, two clips of 5 frames of 17 tokens (M = 170:
split-K, and frames past T masked in the 16-frame temporal attention) and one clip of 32 frames of 17 tokens (the
32-frame temporal attention).

Every output must use at most its whole bound and, unless it is an exact copy (xb, the stack output), a record or a row
statistic, at least FLOOR of it.  Every case runs twice and repeats bit for bit: the loop has no atomics.  Three planted
mistakes of the CPU test also run on the kernels, to show that the bounds catch them there too.  Each test prints the
shares it saw (pytest -s)."""
import pytest
import torch

import test_fused_ref as C
from test_stem_ref import MISS

pytestmark = pytest.mark.gpu
FLOOR = 1e-3
WIDE = dict(d=1536, H=24, F=6144, L=2, dev="cuda")
CASES = {
    "text": dict(form="text", S=72),
    "text_small": dict(form="text", B=2, S=72),
    "image": dict(form="image"),
    "audio": dict(form="audio"),
    "long": dict(form="long"),
    "det": dict(form="det", B=2, bucket=16, window=8),
    "video": dict(form="video", Bv=1, T=16, N=257),
    "video_small": dict(form="video", Bv=2, T=5, N=17),
    "video_long_clip": dict(form="video", Bv=1, T=32, N=17),
}


def kernels():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels as K
    return K


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


@pytest.mark.parametrize("case", sorted(CASES))
def test_fused_loop(case):
    r = C.run(kernels(), **{**WIDE, **CASES[case]})
    sh = r.shares
    print(f"\n{case}: largest share of each bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(sh.items())))
    assert len(sh) == r.n_checks
    over = {k: v for k, v in sh.items() if not v <= 1.0}
    assert not over, f"{case}: outside the bound (share of the bound): {over}"
    low = {k: v for k, v in sh.items() if v < FLOOR and k not in r.exempt}
    assert not low, f"{case}: bound never approached (share below {FLOOR}): {low}"
    again = C.run(kernels(), **{**WIDE, **CASES[case]})
    for k, v in r.got.items():
        assert torch.equal(bits(v), bits(again.got[k])), f"{case}: {k} differs between two runs"


@pytest.mark.parametrize("name", ["FFN-LN records counted without the zero records",
                                  "detection: decomposed terms of the scaled q", "video: MLP adapter without scale"])
def test_planted_mistake_exceeds_bound(name):
    case, edit = C.MISTAKES[name]
    r = C.run(kernels(), edit=edit, **{**WIDE, **CASES[case]})
    sh = {k: v for k, v in r.shares.items() if k.split(".")[-1] not in ("xb", "xb0", "y")}
    worst = max(sh, key=sh.get)
    print(f"\n{name}: largest share {sh[worst]:.3g} ({worst})")
    assert sh[worst] >= MISS, f"{name}: largest share of a bound only {sh[worst]:.3g} ({worst})"
