"""GPU: the short-sequence attention forward (csrc/attention_wgmma.cu, S <= 224), where one CTA runs many (sample, head)
units in turn through two shared-memory buffers, at B * H = 1152 units, several times the SM count.  Each unit stages its
own LUT row and key-padding row, so padding that differs from sample to sample, per-sample dense tables and the
two-segment LUT show a stale buffer, a wrong barrier phase or a unit handed to the wrong buffer as wrong rows here.  Same
checks as tests/test_gpu_attention_contract.py: fp64 bounds, canaries, two launches bit-identical, LUT and dense forms of
the same values bit-identical."""
import pytest
import torch

import kernel_ref as R
from test_gpu_attention_contract import (check_fwd, dense_table, lut_form, make_bias, make_qkv, run_dense, run_lut, s_pad_for,
                                         same_bits, seed, twice)

pytestmark = pytest.mark.gpu
B, H = 48, 24
SEQ = [17, 72, 197, 214, 224]


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def ratios():
    seen = {}
    yield seen
    for k in sorted(seen):
        print(f"bound used: {k:<34s} {seen[k]:.3g}")


def ragged_pad(S, lo=1):
    """right padding of a different length in every sample (none in some); keys [0, lo) always live"""
    kp = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
    for b in range(B):
        n = (b * 37) % S
        kp[b, max(lo, S - n):] = 1
    return kp


@pytest.mark.parametrize("S", SEQ)
def test_lut_many_units(K, ratios, S):
    g = seed("persistent lut", S)
    qkv, kp = make_qkv(B, S, H, g), ragged_pad(S)
    rp, dense = lut_form(K, S, H, g)
    got = run_lut(K, qkv, rp, kp, B, S, H)
    check_fwd(ratios, "lut many units", got, R.attention_ref(qkv, dense, kp, B, S, H), B, S, H)
    same_bits(got, run_dense(K, qkv, dense_table(dense, s_pad_for(S, 1)), kp, B, S, H), "LUT vs dense table")


@pytest.mark.parametrize("S", SEQ)
def test_per_sample_table_many_units(K, ratios, S):
    g = seed("persistent per-sample", S)
    qkv, kp = make_qkv(B, S, H, g), ragged_pad(S)
    bias = make_bias((B, H, S, S), S, "stress", g)
    got = run_dense(K, qkv, dense_table(bias, s_pad_for(S, 2)), kp, B, S, H)
    check_fwd(ratios, "per-sample many units", got, R.attention_ref(qkv, bias, kp, B, S, H), B, S, H)


@pytest.mark.parametrize("S1,w", [(23, 7), (17, 14)])     # S = 73, 214
def test_two_segment_many_units(K, ratios, S1, w):
    import restated
    from one_peace_b200 import relpos
    S2 = w * w + 1
    S = S1 + S2
    g = seed("persistent two-segment", S1, w)
    b1 = restated.make_token_bucket_position(256)[:S1, :S1]
    b2 = restated.make_image_bucket_position(w)
    t1 = torch.randn(514, H, device="cuda", generator=g)
    t2 = torch.randn((2 * w - 1) ** 2 + 3, H, device="cuda", generator=g)
    rp = K.build_segmented_lut([(t1, relpos.build_lut_index(b1.numpy(), relpos.text_codes(S1)), S1),
                                (t2, relpos.build_lut_index(b2.numpy(), relpos.image_codes(S2, w)), S2)], "cuda")
    canvas = torch.zeros(H, S, S, device="cuda")
    canvas[:, :S1, :S1] = t1[b1.cuda()].permute(2, 0, 1)
    canvas[:, S1:, S1:] = t2[b2.cuda()].permute(2, 0, 1)
    kp = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
    for b in range(B):                  # text keys padded just before the image segment, a different count per sample
        n = b % S1
        kp[b, S1 - n:S1] = 1
    qkv = make_qkv(B, S, H, g)
    got = run_lut(K, qkv, rp, kp, B, S, H)
    check_fwd(ratios, "two-segment many units", got, R.attention_ref(qkv, canvas, kp, B, S, H), B, S, H)
    same_bits(got, run_dense(K, qkv, dense_table(canvas, s_pad_for(S, 2)), kp, B, S, H), "two-segment LUT vs its canvas")


def test_without_optional_outputs(K):
    """lse and ln_stats omitted (the inference stack passes ln_stats only): out has the same bits as with both"""
    S = 197
    g = seed("persistent no-lse", S)
    qkv, kp = make_qkv(B, S, H, g), ragged_pad(S)
    rp, _ = lut_form(K, S, H, g)
    full = run_lut(K, qkv, rp, kp, B, S, H)

    def launch():
        out, ob = R.canary_out((B * S, H * 64), rows_before=2, rows_after=2, dtype=torch.bfloat16)
        K.attention_tc(qkv, rp, kp, B, S, H, out=out)
        return {"out": (out, ob)}

    got = twice(launch)
    R.assert_canary(got["out"][1], got["out"][0], what="out without lse / ln_stats")
    assert torch.equal(got["out"][1].view(torch.int16), full["out"][1].view(torch.int16))
