"""CPU: the video backbone's training launch sequence, emulated in fp64 (tests/video_train_emul.py), against torch fp64
autograd through the train-mode restatement (tests/video_train_ref.py), on the tiny config with 2 clips of 4 frames and
explicit per-frame drop-path scales that differ between the frames of a clip.  Compared: the output, dL/d(stem rows),
and the gradient of the temporal embedding, the shared table, the final norm and every layer parameter.
- Exact arithmetic (rounding points off): |E - R| <= 1e-12 (|R| + rms(R)) element by element, rms over the tensor; each
  planted mistake exceeds this more than 100-fold.
- bf16 rounding points on: ||E - R|| <= 7 * 2^-8 ||R|| for every compared tensor (the worst tensor, the table gradient,
  uses 0.85 of it); each planted mistake exceeds this more than 30-fold on some tensor."""
import pytest
import torch

import restated_video as RV
import synth_video as sv

T, B, TAU_BF16 = 4, 2, 7 * 2.0 ** -8


@pytest.fixture(scope="module")
def case():
    from one_peace_b200.vision.video import OnePeaceViT
    torch.manual_seed(0)
    m = OnePeaceViT(num_frames=T, **sv.VIDEO_TINY)
    sd = sv.video_state_dict({k: tuple(p.shape) for k, p in m.named_parameters()}, dict(m.named_buffers()))
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    R = 16 * sv.VIDEO_TINY["bucket_size"]
    x = sv.video_clips(T, B, sv.VIDEO_TINY["bucket_size"]).double()
    p0 = RV.stem(sd, x.transpose(1, 2).reshape(B * T, 3, R, R), T)
    p0 = p0 - sd["image_adapter.temporal_embedding"][0, :T].repeat(B, 1)[:, None, :]
    rs = [tuple(((torch.arange(B * T) + i + j) % 3 != 0).double() * 1.5 for j in range(3))
          for i in range(sv.VIDEO_TINY["layers"])]
    cot = torch.randn(B, sv.VIDEO_TINY["embed_dim"], T, 1, 1, generator=torch.Generator().manual_seed(5)).double()
    return sd, p0, rs, cot


def _run(E, case, mistake=None):
    sd, p0, rs, cot = case
    return E.step(sd, p0, T, sv.VIDEO_TINY["attention_heads"], sv.VIDEO_TINY["layers"], rs, cot, mistake=mistake)


def _pairs(ref, got):
    (Ro, Rg, Rdp), (o, g, dp) = ref, got
    assert set(g) >= set(Rg), set(Rg) - set(g)
    return [("out", o, Ro), ("dp0", dp, Rdp)] + [(k, g[k], Rg[k]) for k in Rg]


def _elementwise(ref, got, tau):
    return max(((e - r).abs() / (tau * (r.abs() + r.pow(2).mean().sqrt()))).max().item() for _, e, r in _pairs(ref, got))


def _normwise(ref, got, tau):
    return max(((e - r).norm() / (tau * r.norm())).item() for _, e, r in _pairs(ref, got))


def test_training_sequence_emulation_and_planted_mistakes(case, monkeypatch):
    import video_train_emul as E
    sd, p0, rs, cot = case
    ref = E.reference(sd, p0, T, sv.VIDEO_TINY["attention_heads"], sv.VIDEO_TINY["layers"], rs, cot)
    assert len(ref[1]) == sum(1 for k, v in sd.items() if v.is_floating_point() and not k.startswith("image_adapter.embed")
                              and k not in ("image_adapter.cls_embedding", "image_adapter.pos_embed"))
    rounded = _normwise(ref, _run(E, case), TAU_BF16)
    assert rounded <= 1.0, rounded
    planted_rounded = {mk: _normwise(ref, _run(E, case, mk), TAU_BF16) for mk in E.MISTAKES}
    monkeypatch.setattr(E, "rb", lambda t: t)
    exact = _elementwise(ref, _run(E, case), 1e-12)
    assert exact <= 1.0, exact
    planted_exact = {mk: _elementwise(ref, _run(E, case, mk), 1e-12) for mk in E.MISTAKES}
    print(f"training emulation: {rounded:.3f} of the bf16 bound, {exact:.3f} of the exact bound; planted (bf16 bound) "
          f"{ {k: round(v, 1) for k, v in planted_rounded.items()} }")
    for mk in E.MISTAKES:
        assert planted_exact[mk] > 100.0, (mk, planted_exact[mk])
        assert planted_rounded[mk] > 30.0, (mk, planted_rounded[mk])
