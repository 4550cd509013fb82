"""GPU: the embedding stems and the retrieval head of the training path (``ImageEmbedFn``, ``AudioFeatFn``,
``AudioPosFn``, ``TextEmbedFn``, ``RelPosBiasFn``, ``HeadFn`` of one_peace_b200/autograd.py), forward and adjoint, stage by
stage, against the fp64 references and per-element bounds of tests/stem_ref.py.

Each Function's ``.apply`` is called directly with leaf tensors, so every gradient (positions, CLS, every weight) is
observable, with a random upstream gradient on every row, CLS and padded rows included.  The audio cases feed waveforms
through the feature extractor into the positional encoder.  The Functions run from a fresh copy of their module whose
kernels sit behind the CPU test's ``Recorder``, so each backward stage is checked from the bf16 intermediate the device
handed it.  Where the reference gradient is exactly zero (a padding token's row and unused rows of the embedding table,
relative-position buckets no position uses, the head's dx past the CLS row, padded rows) the bound is zero, so the device
value must be exactly zero.

Every output must use at most its whole bound and, unless it can come out exact (a copy, or a sum of one term) or is a
column reduction (``REDUCTION``), at least FLOOR of it: a bound that is never approached would not notice a mistake.  Each test prints the shares it saw (pytest -s).
The case builders are the CPU test's (tests/test_stem_ref.py), run on the kernels instead of their emulation."""
import re

import pytest
import torch

import restated
import test_stem_ref as C

pytestmark = pytest.mark.gpu
BF, F32 = torch.bfloat16, torch.float32
FLOOR = 1e-3
SPEC = tuple(restated.OracleConfig.feature_encoder_spec)     # the wav2vec extractor: 512 channels, 7 convolutions


def fns():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return C.functions(kernels)


# Column reductions over rows (bias gradients, LayerNorm dgamma / dbeta, batch sums): kernel_ref bounds their fp32 sums by
# the any-order worst case tau sum |terms|, which a sum of mixed-sign terms stays far below (1e-4 of it at 12608 rows), and
# a sum of a few bf16 terms is exact in fp32.  The floor holds every other output: each elementwise stage and each GEMM.
REDUCTION = re.compile(r"^(b\d?|proj_b|post_[wb]|ln\d?[wb]|ln[wb]\d|ln_[wb]|cls|cls_pos|pos)$")


def check(what, result):
    sh, exact = result
    print(f"\n{what}: largest share of each bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(sh.items())))
    over = {k: v for k, v in sh.items() if not v <= 1.0}
    assert not over, f"{what}: outside the bound (share of the bound): {over}"
    low = {k: v for k, v in sh.items() if v < FLOOR and k not in exact and not REDUCTION.match(k)}
    assert not low, f"{what}: bound never approached (share below {FLOOR}): {low}"


@pytest.mark.parametrize("dt", [(F32, F32), (BF, BF), (F32, BF)], ids=["f32", "bf16", "f32img_bf16par"])
@pytest.mark.parametrize("B,R,d", [(1, 32, 256), (3, 48, 256), (2, 224, 256), (2, 224, 1536)])
def test_image_embed(B, R, d, dt):
    check(f"image B={B} R={R} d={d}", C.image_case(fns(), B=B, R_=R, c4=d // 4, d=d, img_dtype=dt[0], p_dtype=dt[1],
                                                     seed=B * R + d, dev="cuda"))


@pytest.mark.parametrize("B,samples,d,pad_from", [
    (1, 16000, 256, (None,)),
    (2, 16000, 256, (None, 36)),                    # clip 1 padded from 3/4 of its 49 frames
    (3, 24000, 256, (None, 50, 1)),                 # different pad lengths, one clip with a single valid frame
    (2, 240000, 1536, (None, 600)),                 # the 15 s clip padded from frame 600
])
def test_audio(B, samples, d, pad_from):
    check(f"audio B={B} samples={samples} d={d}", C.audio_case(fns(), B=B, d=d, samples=samples, spec=SPEC,
                                                               pad_from=pad_from, seed=samples + d, dev="cuda"))


@pytest.mark.parametrize("d,p_dtype", [(256, F32), (1536, BF)])
def test_audio_pos_t37(d, p_dtype):
    check(f"audio_pos T=37 d={d}", C.audio_case(fns(), B=2, T=37, d=d, pad_from=(None, 20), p_dtype=p_dtype, seed=37,
                                                dev="cuda"))


@pytest.mark.parametrize("B,T,d,pads", [(8, 17, 256, ((1, 10), (5, 0), (7, 16))), (3, 72, 1536, ((0, 60), (2, 1)))])
def test_text_embed(B, T, d, pads):
    check(f"text B={B} T={T}", C.text_case(fns(), B=B, T=T, V=1000, d=d, pads=pads, seed=T, dev="cuda"))


@pytest.mark.parametrize("p_dtype", [F32, BF])
@pytest.mark.parametrize("B,S,d", [(1, 17, 256), (3, 197, 1536), (8, 17, 1536), (64, 197, 256), (1, 197, 1536),
                                   (3, 17, 256)])
def test_head(B, S, d, p_dtype):
    check(f"head B={B} S={S} d={d}", C.head_case(fns(), B=B, S=S, d=d, n=d, p_dtype=p_dtype, seed=B + S, dev="cuda"))


@pytest.mark.parametrize("H", [4, 24])
@pytest.mark.parametrize("S", [17, 72, 197])
def test_relpos_bias(S, H):
    if S == 197:
        bucket = restated.make_image_bucket_position(14)
    else:
        bucket = restated.make_token_bucket_position(256)[:S, :S].contiguous()
    NB = int(bucket.max()) + 4                      # three rows past the last bucket stay unused
    check(f"relpos S={S} H={H}", C.relpos_case(fns(), S=S, H=H, NB=NB, bucket=bucket, seed=S + H, dev="cuda"))
