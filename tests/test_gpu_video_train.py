"""GPU: fine-tuning the video backbone.

opb_attention_temporal_bwd against tests/kernel_ref.py's fp64 attention-backward bounds on the gathered (clip, token)
sequences, with lse = ref.lse + ref.dlse so that the bound covers the recomputed soft-max, for T in {2, 5, 16, 31, 32},
N in {1, 17, 257} and (Bv, H) in {(1, 2), (4, 24)}; dqkv inside NaN canaries, repeat launches bit-identical.  The GELU pair
against fp64.  OnePeaceViT in train mode against torch autograd through the fp32 train-mode restatement
(tests/video_train_ref.py) on the same GPU: the tiny model without and with drop-path (masks drawn again from the saved
CUDA RNG state), kept against recomputed activations, and the 40-layer backbone at T = 16.  The tiny model against the
reference's own train-mode output and gradients (tests/golden/video_train.pt, with the reference's drop-path masks), and
frozen parameters getting no gradient."""
import os

import pytest
import torch
import torch.nn.functional as F

import kernel_ref as R
import synth_video as sv
import video_train_ref as VT

pytestmark = pytest.mark.gpu
USED = {}


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _record(name, ratio):
    USED[name] = max(USED.get(name, 0.0), ratio)


def _frame_major_index(Bv, T, N, device):
    b = torch.arange(Bv, device=device).view(Bv, 1, 1)
    n = torch.arange(N, device=device).view(1, N, 1)
    t = torch.arange(T, device=device).view(1, 1, T)
    return ((b * T + t) * N + n).reshape(-1)


@pytest.mark.parametrize("T", [2, 5, 16, 31, 32])
@pytest.mark.parametrize("N", [1, 17, 257])
@pytest.mark.parametrize("Bv,H", [(1, 2), (4, 24)])
def test_temporal_attention_bwd_against_fp64(T, N, Bv, H):
    need_gpu()
    from one_peace_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(T * 1000 + N * 10 + H + 7)
    M, D = Bv * T * N, H * 64
    qkv = torch.randn(M, 3 * D, device="cuda", generator=g)
    qkv[:, :D] *= 0.25
    qkv = qkv.to(torch.bfloat16).contiguous()
    out, _ = K.attention_temporal(qkv, Bv, T, N, H)
    dout = torch.randn(M, D, device="cuda", generator=g).to(torch.bfloat16)
    q_scale = 0.125
    dqkv, buf = R.canary_out((M, 3 * D), rows_before=3, rows_after=5, dtype=torch.bfloat16)
    K.attention_temporal_bwd(qkv, out, dout, Bv, T, N, H, q_scale, dqkv=dqkv)
    R.assert_canary(buf, dqkv, what="dqkv")
    idx = _frame_major_index(Bv, T, N, "cuda")
    Bs = Bv * N
    f = R.attention_ref(qkv[idx].contiguous(), None, None, Bs, T, H)
    lse = (f.lse + f.dlse).reshape(-1)
    ref = R.attention_bwd_ref(qkv[idx].contiguous(), out[idx].contiguous(), dout[idx].contiguous(), lse, None, None, Bs, T,
                              H, q_scale)
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        _record(name, R.assert_within(dqkv[idx][:, sl], ref.dqkv[:, sl], ref.dqkv_err[:, sl], 1.0, torch.bfloat16, what=name))
    again = K.attention_temporal_bwd(qkv, out, dout, Bv, T, N, H, q_scale)
    assert torch.equal(again, dqkv)


def test_temporal_attention_bwd_refusals():
    need_gpu()
    from one_peace_b200 import _lib
    lib = _lib.load()
    t = torch.empty(64, dtype=torch.bfloat16, device="cuda")
    p = t.data_ptr()

    def call(**o):
        args = dict(qkv=p, out=p, dout=p, dqkv=p, Bv=1, T=16, N=257, H=24, qs=0.125, stream=0)
        args.update(o)
        return lib.opb_attention_temporal_bwd(*args.values())
    for bad in [dict(qkv=0), dict(out=0), dict(dout=0), dict(dqkv=0), dict(qkv=p + 8), dict(dqkv=p + 2), dict(T=1),
                dict(T=33), dict(Bv=0), dict(N=0), dict(H=0)]:
        assert call(**bad) == 1, bad


def test_gelu_pair_against_fp64():
    need_gpu()
    from one_peace_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(3)
    z = (3 * torch.randn(1000, 384, device="cuda", generator=g)).to(torch.bfloat16)
    dy = torch.randn(1000, 384, device="cuda", generator=g).to(torch.bfloat16)
    zd = z.double()
    y = K.gelu_fwd(z, torch.empty_like(z))
    dz = K.gelu_bwd(z, dy, torch.empty_like(z))
    ref_y = F.gelu(zd)
    cdf = 0.5 * (1 + torch.erf(zd / 2 ** 0.5))
    ref_dz = dy.double() * (cdf + zd * torch.exp(-0.5 * zd * zd) / (2 * torch.pi) ** 0.5)
    tau = 2.0 ** -20                 # fp32 erf / exp: a few ulp of the fp32 result, well below the bf16 output rounding
    _record("gelu", R.assert_within(y, ref_y, ref_y.abs() + zd.abs(), tau, torch.bfloat16, what="gelu"))
    _record("gelu_bwd", R.assert_within(dz, ref_dz, (dy.double().abs() * (1 + zd.abs())), tau, torch.bfloat16, what="gelu'"))


# ----------------------------------------------------------------------------------------------------------------
# the model
# ----------------------------------------------------------------------------------------------------------------
def _tiny(T, **kw):
    from one_peace_b200.vision.video import OnePeaceViT
    torch.manual_seed(0)
    m = OnePeaceViT(num_frames=T, **{**sv.VIDEO_TINY, **kw})
    sd = sv.video_state_dict({k: tuple(p.shape) for k, p in m.named_parameters()}, dict(m.named_buffers()))
    m.load_state_dict(sd, strict=True)
    return m.cuda().train(), {k: v.cuda() for k, v in sd.items()}


def _cos(a, b):
    return F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()


def _reference(sd, x, heads, layers, cot, masks=None, checkpoint=False, scale=0.5):
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and not k.endswith("rp_bucket") else v)
           for k, v in sd.items()}
    out = VT.forward(sdg, x, heads, layers, scale, masks=masks, checkpoint=checkpoint)
    (out * cot).sum().backward()
    return out.detach(), {k: v.grad for k, v in sdg.items() if torch.is_tensor(v) and v.requires_grad}


def _compare(m, y, want, grads, names=None, bar=0.99):
    c = _cos(y, want)
    worst, where = 1.0, None
    top = max(g.abs().max().item() for g in grads.values())
    for k, prm in m.named_parameters():
        if names is not None and not names(k):
            continue
        ref = grads[k]
        if ref.abs().max() == 0:
            assert prm.grad is None or prm.grad.abs().max().item() <= 1e-7 * top, (k, prm.grad.abs().max().item())
            continue
        assert prm.grad is not None, k
        ck = _cos(prm.grad, ref)
        if ck < worst:
            worst, where = ck, k
    return c, worst, where


@pytest.fixture
def strict_fp32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("case", list(sv.VIDEO_CASES))
def test_tiny_training_against_restatement(case, strict_fp32):
    need_gpu()
    T, clips = sv.VIDEO_CASES[case]
    m, sd = _tiny(T)
    x = sv.video_clips(T, clips, sv.VIDEO_TINY["bucket_size"]).cuda()
    y = m(x)
    cot = torch.randn(y.shape, generator=torch.Generator().manual_seed(5)).cuda()
    (y * cot).sum().backward()
    want, grads = _reference(sd, x, sv.VIDEO_TINY["attention_heads"], sv.VIDEO_TINY["layers"], cot)
    c, worst, where = _compare(m, y.detach(), want, grads)
    print(f"{case}: output cosine {c:.6f}, worst parameter-gradient cosine {worst:.5f} ({where})")
    assert c > 0.999 and worst > 0.99, (c, worst, where)


@pytest.mark.parametrize("case", ["plain", "drop_path"])
def test_tiny_training_against_reference_fixture(case, golden_dir, monkeypatch):
    """tests/golden/video_train.pt: the reference's own onepeace.py in train mode, fp64.  In the drop-path case the masks the
    reference drew replace this run's draw (per layer with p > 0: temporal, spatial, MLP adapter)."""
    need_gpu()
    from grad_codec import dequantise
    from one_peace_b200.vision import video
    gold = torch.load(os.path.join(golden_dir, "video_train.pt"), weights_only=False)
    rec = gold[case]
    T, clips = gold["T"], gold["clips"]
    m, _ = _tiny(T, drop_path_rate=rec["drop_path_rate"])
    if rec["masks"]:
        real = video.draw_row_scales

        def recorded(layers, Bv, T_, N_, device):
            it = iter(rec["masks"])
            return [trip if trip[0] is None else tuple(next(it).to(device).repeat_interleave(N_).contiguous()
                                                       for _ in range(3))
                    for trip in real(layers, Bv, T_, N_, device)]
        monkeypatch.setattr(video, "draw_row_scales", recorded)
    x = sv.video_clips(T, clips, sv.VIDEO_TINY["bucket_size"]).cuda()
    y = m(x)
    (y * gold["cot"].cuda()).sum().backward()
    grads = {k: v.cuda() for k, v in dequantise(rec["grads"]).items()}
    assert set(grads) == {k for k, _ in m.named_parameters()}
    c, worst, where = _compare(m, y.detach(), rec["out"].cuda(), grads)
    print(f"reference fixture, {case}: output cosine {c:.6f}, worst parameter-gradient cosine {worst:.5f} ({where})")
    assert c > 0.999 and worst > 0.99, (c, worst, where)


def test_frozen_parameters_get_no_gradient():
    """Adapter tuning with a frozen backbone: frozen parameters get None, the adapters the gradients of a full run."""
    need_gpu()
    T, clips = 4, 2
    x = sv.video_clips(T, clips, sv.VIDEO_TINY["bucket_size"]).cuda()
    m, _ = _tiny(T)
    m(x).sum().backward()
    full = {k: p.grad.clone() for k, p in m.named_parameters()}
    m, _ = _tiny(T)
    for k, p in m.named_parameters():
        p.requires_grad_("Adapter" in k)
    m(x).sum().backward()
    for k, p in m.named_parameters():
        if "Adapter" in k:
            assert p.grad is not None and torch.equal(p.grad, full[k]), k
        else:
            assert p.grad is None, k


def test_tiny_training_with_drop_path(strict_fp32):
    need_gpu()
    T, clips = 4, 2
    m, sd = _tiny(T, drop_path_rate=0.5)
    x = sv.video_clips(T, clips, sv.VIDEO_TINY["bucket_size"]).cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    state = torch.cuda.get_rng_state(dev)
    y = m(x)
    cot = torch.randn(y.shape, generator=torch.Generator().manual_seed(6)).cuda()
    (y * cot).sum().backward()
    masks = VT.row_scales([l.drop_path_prob for l in m.encoder.layers], T * clips, state, dev)
    assert any(r is not None and (r == 0).any() for trip in masks for r in trip), "no frame was dropped: pick another seed"
    want, grads = _reference(sd, x, sv.VIDEO_TINY["attention_heads"], sv.VIDEO_TINY["layers"], cot, masks=masks)
    c, worst, where = _compare(m, y.detach(), want, grads)
    print(f"drop-path: output cosine {c:.6f}, worst parameter-gradient cosine {worst:.5f} ({where})")
    assert c > 0.999 and worst > 0.99, (c, worst, where)


def test_keep_and_recompute_agree(monkeypatch):
    need_gpu()
    T, clips = 4, 2
    x = sv.video_clips(T, clips, sv.VIDEO_TINY["bucket_size"]).cuda()
    got = {}
    for mode in ("keep", "recompute"):
        monkeypatch.setenv("OPB_ACTIVATIONS", mode)
        m, _ = _tiny(T)
        y = m(x)
        y.sum().backward()
        got[mode] = (y.detach(), {k: p.grad.clone() for k, p in m.named_parameters()})
    assert torch.equal(got["keep"][0], got["recompute"][0])
    diff = {k: (got["keep"][1][k] - got["recompute"][1][k]).abs().max().item() for k in got["keep"][1]}
    inexact = {k: v for k, v in diff.items() if v != 0}
    print(f"keep vs recompute: output bit-identical, gradients differing: {inexact}")
    # only the table gradient may differ: the attention backward accumulates it with atomic adds
    assert set(inexact) <= {"image_adapter.rel_pos_table.weight"}, inexact
    if inexact:
        ref = got["keep"][1]["image_adapter.rel_pos_table.weight"]
        assert inexact["image_adapter.rel_pos_table.weight"] <= 1e-5 * ref.abs().max().item()


def test_eval_mode_still_refuses_under_grad():
    need_gpu()
    m, _ = _tiny(4)
    m.eval()
    x = sv.video_clips(4, 1, sv.VIDEO_TINY["bucket_size"]).cuda()
    with pytest.raises(NotImplementedError):
        m(x)


def test_production_backbone_training_against_fp32_restatement(strict_fp32):
    need_gpu()
    from one_peace_b200.vision.video import OnePeaceViT
    P = {**sv.PRODUCTION, "drop_path_rate": 0.0}
    with torch.device("meta"):
        meta = OnePeaceViT(**P)
    shapes = {k: tuple(p.shape) for k, p in meta.named_parameters()}
    del meta
    torch.manual_seed(0)
    m = OnePeaceViT(**P)
    sd = sv.video_state_dict(shapes, {k: b.cuda() for k, b in m.named_buffers()}, device="cuda")
    m = m.cuda()
    m.load_state_dict(sd, strict=True)
    m.train()
    x = sv.video_clips(P["num_frames"], 1, P["bucket_size"], device="cuda")
    y = m(x)
    cot = torch.randn(y.shape, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda")
    (y * cot).sum().backward()
    yd = y.detach()
    del y
    last = f"encoder.layers.{P['layers'] - 1}."
    checked = lambda k: (k.startswith("image_adapter.") or k.startswith("encoder.image_layer_norm") or
                         k.startswith("encoder.layers.0.") or k.startswith(last))
    want, grads = _reference(sd, x, P["attention_heads"], P["layers"], cot, checkpoint=True, scale=P["adapter_scale"])
    c, worst, where = _compare(m, yd, want, grads, names=checked)
    print(f"production backbone training: output cosine {c:.6f}, worst checked parameter-gradient cosine {worst:.5f} "
          f"({where})")
    assert c >= 0.999 and worst > 0.99, (c, worst, where)


def test_zz_report_bound_shares():
    print("largest share of each bound:", {k: round(v, 4) for k, v in USED.items()})
