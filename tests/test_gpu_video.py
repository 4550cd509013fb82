"""GPU: the video backbone's temporal-attention kernel and model.

opb_attention_temporal_fwd against tests/kernel_ref.py's fp64 attention bounds on the gathered (clip, token) sequences of
T frames, for T in {2, 5, 16, 31, 32}, N in {1, 17, 257} and (Bv, H) in {(1, 2), (4, 24)}; outputs and records inside NaN
canaries, repeat launches bit-identical.  OnePeaceViT against the reference's own onepeace.py (tests/golden/video.pt)
and, with 40 layers at 256^2 and T = 16, against the fp32 torch restatement oracle/restated_video.py on the same GPU after
a strict load of a synthetic full state dict with non-zero adapters.  Autocast invariance, bit-identical repeats and the
refusal under grad."""
import os

import pytest
import torch
import torch.nn.functional as F

import kernel_ref as R
import restated_video as RV
import synth_video as sv

pytestmark = pytest.mark.gpu
USED = {}          # largest share of each bound, printed at the end of the module (pytest -s)


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _record(name, ratio):
    USED[name] = max(USED.get(name, 0.0), ratio)


def _frame_major_index(Bv, T, N, device):
    """gathered row (b N + n) T + t -> frame-major row (b T + t) N + n"""
    b = torch.arange(Bv, device=device).view(Bv, 1, 1)
    n = torch.arange(N, device=device).view(1, N, 1)
    t = torch.arange(T, device=device).view(1, 1, T)
    return ((b * T + t) * N + n).reshape(-1)


@pytest.mark.parametrize("T", [2, 5, 16, 31, 32])
@pytest.mark.parametrize("N", [1, 17, 257])
@pytest.mark.parametrize("Bv,H", [(1, 2), (4, 24)])
def test_temporal_attention_against_fp64(T, N, Bv, H):
    need_gpu()
    from one_peace_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(T * 1000 + N * 10 + H)
    M, D = Bv * T * N, H * 64
    qkv = torch.randn(M, 3 * D, device="cuda", generator=g)
    qkv[:, :D] *= 0.125 * 2.0
    qkv = qkv.to(torch.bfloat16).contiguous()
    out, obuf = R.canary_out((M, D), rows_before=3, rows_after=5, dtype=torch.bfloat16)
    buf = torch.full((64 + H * M * 2 + 64,), float("nan"), device="cuda")
    st = buf[64:]
    K.attention_temporal(qkv, Bv, T, N, H, out=out, ln_stats=st[:H * M * 2])
    R.assert_canary(obuf, out, what="out")
    assert torch.isnan(buf[:64]).all() and torch.isnan(st[H * M * 2:]).all()
    idx = _frame_major_index(Bv, T, N, "cuda")
    ref = R.attention_ref(qkv[idx].contiguous(), None, None, Bv * N, T, H)
    _record("out", R.assert_within(out[idx], ref.out, ref.out_err, 1.0, torch.bfloat16, what="out"))
    stats = st[:H * M * 2].view(H, M, 2)[:, idx]
    _record("ln_stats", R.assert_within(stats, ref.stats, ref.stats_err, 1.0, torch.float32, what="ln_stats"))
    out2, st2 = K.attention_temporal(qkv, Bv, T, N, H)
    assert torch.equal(out2, out) and torch.equal(st2.view(-1), st[:H * M * 2])


def _model(T, device="cuda", **kw):
    from one_peace_b200.vision.video import OnePeaceViT
    torch.manual_seed(0)
    m = OnePeaceViT(num_frames=T, **{**sv.VIDEO_TINY, **kw})
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    m.load_state_dict(sv.video_state_dict(shapes, dict(m.named_buffers())), strict=True)
    return m.to(device).eval()


def _cos(a, b):
    return F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()


@pytest.mark.parametrize("case", list(sv.VIDEO_CASES))
def test_tiny_model_against_reference(case, golden_dir):
    need_gpu()
    gold = torch.load(os.path.join(golden_dir, "video.pt"), weights_only=False)["cases"][case]
    T, clips = sv.VIDEO_CASES[case]
    m = _model(T)
    x = sv.video_clips(T, clips, sv.VIDEO_TINY["bucket_size"]).cuda()
    with torch.no_grad():
        y = m(x)
        feats = m.forward_features(x)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y_ac = m(x)
        y2 = m(x)
    assert y.shape == gold["out"].shape and y.dtype == torch.float32
    assert feats.shape == gold["features"].shape
    c, cf = _cos(y.cpu(), gold["out"]), _cos(feats.cpu(), gold["features"])
    per_view = F.cosine_similarity(y.squeeze(-1).squeeze(-1).transpose(1, 2).reshape(-1, y.shape[1]).cpu().double(),
                                   gold["out"].squeeze(-1).squeeze(-1).transpose(1, 2).reshape(-1, y.shape[1]).double())
    print(f"{case}: cosine out {c:.6f} features {cf:.6f} worst frame {per_view.min().item():.6f}")
    assert c > 0.999 and cf > 0.999 and per_view.min().item() > 0.999
    assert torch.equal(y_ac, y) and torch.equal(y2, y)


def test_refusal_under_grad():
    need_gpu()
    m = _model(4)
    x = sv.video_clips(4, 1, sv.VIDEO_TINY["bucket_size"]).cuda()
    with pytest.raises(NotImplementedError):
        m(x)


@pytest.fixture
def strict_fp32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_production_backbone_against_fp32_restatement(strict_fp32):
    need_gpu()
    from one_peace_b200.vision.video import OnePeaceViT
    P = sv.PRODUCTION
    with torch.device("meta"):
        meta = OnePeaceViT(**P)
    shapes = {k: tuple(p.shape) for k, p in meta.named_parameters()}
    del meta
    torch.manual_seed(0)
    m = OnePeaceViT(**P)
    sd = sv.video_state_dict(shapes, {k: b.cuda() for k, b in m.named_buffers()}, device="cuda")
    m = m.cuda()
    m.load_state_dict(sd, strict=True)
    m.eval()
    x = sv.video_clips(P["num_frames"], 1, P["bucket_size"], device="cuda")
    with torch.no_grad():
        y = m(x)
        want = RV.forward(sd, x, P["attention_heads"], P["layers"], P["adapter_scale"])
    c = _cos(y, want)
    per_frame = F.cosine_similarity(y[0, :, :, 0, 0].t().double(), want[0, :, :, 0, 0].t().double())
    print(f"production backbone: cosine {c:.6f}, worst frame {per_frame.min().item():.6f}")
    assert y.shape == (1, P["embed_dim"], P["num_frames"], 1, 1)
    assert c >= 0.999 and per_frame.min().item() >= 0.999


def test_zz_report_bound_shares():
    print("largest share of each bound:", {k: round(v, 4) for k, v in USED.items()})
