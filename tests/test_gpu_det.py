"""GPU: the detection backbone's kernels and model.

opb_relpos_decomp_proj and opb_attention_decomp_fwd against tests/det_ref.py's fp64 bounds at S = 256 (B = 25, 50),
S = 6400 (B = 1, 2), an 8 x 8 grid and a 12 x 20 grid, rows in a shuffled grid order; outputs in NaN canaries and repeat
launches bit-identical; with zero decomposed terms the attention equals opb_attention_tc_fwd bit for bit.  OnePeace
against the reference's own onepeace.py (tests/golden/det.pt) and, at 1280^2 with 40 layers, against the fp32 torch
restatement oracle/restated_det.py on the same GPU after a strict load of a synthetic full state dict.  Autocast
invariance and the training refusal."""
import os

import pytest
import torch
import torch.nn.functional as F

import det_ref as D
import kernel_ref as R
import restated_det
import synth_det as sd_

pytestmark = pytest.mark.gpu
USED = {}          # largest share of each bound, printed at the end of the module (pytest -s)


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _record(name, ratio):
    USED[name] = max(USED.get(name, 0.0), ratio)


def _case(B, H, kh, kw, seed):
    """qkv (q carrying head_dim^-0.5 as the QKV epilogue stores it), tables, a LUT over the (2kh-1) x (2kw-1) offsets,
    shuffled grid positions."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    S, D_ = kh * kw, H * 64
    qkv = torch.randn(B * S, 3 * D_, device="cuda", generator=g)
    qkv[:, :D_] *= 0.125 * 1.5
    qkv = qkv.to(torch.bfloat16).contiguous()
    rph = 0.3 * torch.randn(2 * kh - 1, 64, device="cuda", generator=g)
    rpw = 0.3 * torch.randn(2 * kw - 1, 64, device="cuda", generator=g)
    order = torch.randperm(S, device="cuda", generator=g)
    pos_y, pos_x = (order // kw).int().contiguous(), (order % kw).int().contiguous()
    code = pos_y.long() * (2 * kw - 1) + pos_x.long()
    maxc = (kh - 1) * (2 * kw - 1) + kw - 1
    lut = 0.5 * torch.randn(H, (2 * kh - 1) * (2 * kw - 1), device="cuda", generator=g)
    from one_peace_b200 import kernels as K
    rp = K.RelPosBias(lut=lut.contiguous(), code_row=(code + maxc).int().contiguous(), code_col=code.int().contiguous())
    bias = lut[:, (code + maxc)[:, None] - code[None, :]]
    return qkv, rph, rpw, pos_y, pos_x, rp, bias


SHAPES = [(25, 24, 16, 16), (50, 4, 16, 16), (1, 2, 80, 80), (2, 1, 80, 80), (3, 2, 8, 8), (2, 3, 12, 20)]


@pytest.mark.parametrize("B,H,kh,kw", SHAPES)
def test_decomp_kernels_within_bounds(B, H, kh, kw):
    need_gpu()
    from one_peace_b200 import kernels as K
    S = kh * kw
    qkv, rph, rpw, py, px, rp, bias = _case(B, H, kh, kw, seed=B * 1000 + kh * 7 + kw)
    nh, nw = B * H * S * kh, B * H * S * kw
    buf_h = torch.full((nh + 64,), float("nan"), device="cuda")
    buf_w = torch.full((nw + 64,), float("nan"), device="cuda")
    rel_h, rel_w = buf_h[32:32 + nh].view(B, H, S, kh), buf_w[32:32 + nw].view(B, H, S, kw)
    K.relpos_decomp_proj(qkv, rph, rpw, py, px, B, S, H, kh, kw, rel_h=rel_h, rel_w=rel_w)
    for buf, n in ((buf_h, nh), (buf_w, nw)):
        assert torch.isnan(buf[:32]).all() and torch.isnan(buf[32 + n:]).all(), "write outside the terms"
    rh, eh, rw, ew = D.proj_ref(qkv, rph, rpw, py, px, B, S, H, kh, kw)
    _record("rel_h", R.assert_within(rel_h, rh, eh, 1.0, torch.float32, what="rel_h"))
    _record("rel_w", R.assert_within(rel_w, rw, ew, 1.0, torch.float32, what="rel_w"))
    again = K.relpos_decomp_proj(qkv, rph, rpw, py, px, B, S, H, kh, kw)
    assert torch.equal(again[0], rel_h) and torch.equal(again[1], rel_w)

    D_ = H * 64
    out, obuf = R.canary_out((B * S, D_), rows_before=3, rows_after=5, dtype=torch.bfloat16)
    lse = torch.full((B * H * S + 8,), float("nan"), device="cuda")
    st = torch.full((H * B * S * 2 + 8,), float("nan"), device="cuda")
    K.attention_decomp(qkv, rp, rel_h, rel_w, py, px, B, S, H, kh, kw, out=out, lse=lse[:B * H * S],
                       ln_stats=st[:H * B * S * 2])
    R.assert_canary(obuf, out, what="out")
    assert torch.isnan(lse[B * H * S:]).all() and torch.isnan(st[H * B * S * 2:]).all()
    ref = D.decomp_attention_ref(qkv, bias, rh, eh, rw, ew, py, px, B, S, H)
    _record("out", R.assert_within(out, ref.out, ref.out_err, 1.0, torch.bfloat16, what="out"))
    _record("lse", R.assert_within(lse[:B * H * S].view(B, H, S), ref.lse, ref.dlse, 1.0, torch.float32, what="lse"))
    _record("ln_stats", R.assert_within(st[:H * B * S * 2].view(H, B * S, 2), ref.stats, ref.stats_err, 1.0,
                                        torch.float32, what="ln_stats"))
    out2 = K.attention_decomp(qkv, rp, rel_h, rel_w, py, px, B, S, H, kh, kw)
    assert torch.equal(out2, out)


@pytest.mark.parametrize("B,H,kh,kw", [(4, 3, 16, 16), (1, 2, 80, 80)])
def test_zero_terms_equal_lut_attention(B, H, kh, kw):
    need_gpu()
    from one_peace_b200 import kernels as K
    S = kh * kw
    qkv, _, _, py, px, rp, _ = _case(B, H, kh, kw, seed=7)
    z_h = torch.zeros(B, H, S, kh, device="cuda")
    z_w = torch.zeros(B, H, S, kw, device="cuda")
    st_a = torch.empty(H * B * S * 2, device="cuda")
    st_b = torch.empty_like(st_a)
    a = K.attention_decomp(qkv, rp, z_h, z_w, py, px, B, S, H, kh, kw, ln_stats=st_a)
    b = K.attention_tc(qkv, rp, None, B, S, H, ln_stats=st_b)
    assert torch.equal(a, b) and torch.equal(st_a, st_b)


def _tiny_model(case):
    from one_peace_b200.vision.det import OnePeace
    bucket, window, pretrain, wbi = sd_.DET_CASES[case]
    torch.manual_seed(0)
    m = OnePeace(bucket_size=bucket, window_size=window, pretrain_bucket_size=pretrain, window_block_indexes=wbi,
                 **sd_.DET_TINY)
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    m.load_state_dict(sd_.det_state_dict(shapes, dict(m.named_buffers())), strict=True)
    return m.cuda().eval()


def _cos(a, b):
    return F.cosine_similarity(a.double().flatten(1), b.double().flatten(1), dim=1)


@pytest.mark.parametrize("case", list(sd_.DET_CASES))
def test_tiny_fixture(case, golden_dir):
    need_gpu()
    gold = torch.load(os.path.join(golden_dir, "det.pt"), weights_only=False)["cases"][case]["last_feat"]
    m = _tiny_model(case)
    img = sd_.det_images(sd_.DET_CASES[case][0]).cuda()
    with torch.no_grad():
        feat = m(img)["last_feat"]
    assert feat.dtype == torch.float32 and feat.shape == gold.shape
    cos = _cos(feat.cpu(), gold)
    assert (cos > 0.999).all(), cos


def test_autocast_invariance_and_training_refusal():
    need_gpu()
    m = _tiny_model("win4")
    img = sd_.det_images(8).cuda()
    with torch.no_grad():
        a = m(img)["last_feat"]
        with torch.autocast("cuda", dtype=torch.bfloat16):
            b = m(img)["last_feat"]
    assert b.dtype == torch.float32 and torch.equal(a, b)
    with pytest.raises(NotImplementedError, match="inference"):
        m(img)
    with torch.no_grad(), pytest.raises(ValueError):
        m(img[:, :, :64])


def test_production_backbone_1280():
    need_gpu()
    from one_peace_b200.vision.det import OnePeace
    lin = torch.linspace
    torch.linspace = lambda *a, **k: lin(*a, **{**k, "device": "cpu"})
    try:
        with torch.device("meta"):
            m = OnePeace(**sd_.PRODUCTION)
    finally:
        torch.linspace = lin
    m = m.to_empty(device="cuda")
    bufs = {"image_adapter.rp_bucket": restated_det.make_image_bucket_position(80, 159 * 159 + 3)[1:, 1:].contiguous(),
            "image_adapter.rp_bucket_window": restated_det.make_image_bucket_position(16, 31 * 31 + 3)[1:, 1:].contiguous()}
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    sd = sd_.det_state_dict(shapes, {k: v.cuda() for k, v in bufs.items()}, device="cuda")
    m.load_state_dict(sd, strict=True)
    m.eval()
    img = sd_.det_images(80, batch=1).cuda()
    with torch.no_grad():
        feat = m(img)["last_feat"]
        ref = restated_det.forward(sd, img, 24, 40, 80, 16, sd_.PRODUCTION["window_block_indexes"])
    assert feat.shape == (1, 1536, 80, 80) and torch.isfinite(feat).all()
    cos = _cos(feat, ref)
    print(f"\nproduction 1280^2 last_feat cosine {cos.item():.6f}")
    assert (cos >= 0.999).all(), cos


def test_zz_report_bound_shares():
    print("\nlargest share of each bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(USED.items())))
