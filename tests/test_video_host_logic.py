"""CPU: the video backbone's host logic.  oracle/restated_video.py against tests/golden/video.pt (the reference's own
onepeace.py); the production key / shape / dtype list and registration order; init_weights(pretrained=) and the adapter
zero-init after it; the refusals, which raise before any kernel runs; and the C ABI rejecting bad arguments of the temporal
attention."""
import json
import os
import pickle
import zlib

import pytest
import torch

import restated_video as RV
import synth_video as sv


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "video.pt"), weights_only=False)


def _tiny(T, **kw):
    from one_peace_b200.vision.video import OnePeaceViT
    torch.manual_seed(0)
    return OnePeaceViT(num_frames=T, **{**sv.VIDEO_TINY, **kw})


def _keys(m):
    return [(k, tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()]


def _state(m):
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    return sv.video_state_dict(shapes, dict(m.named_buffers()))


@pytest.mark.parametrize("case", list(sv.VIDEO_CASES))
def test_restatement_matches_reference(case, golden_dir):
    gold = _gold(golden_dir)["cases"][case]
    T, clips = sv.VIDEO_CASES[case]
    m = _tiny(T)
    assert _keys(m) == [tuple(k) for k in gold["keys"]]
    sd = _state(m)           # same names in the same order as the reference's: the same seeded values
    x = sv.video_clips(T, clips, sv.VIDEO_TINY["bucket_size"])
    heads, layers = sv.VIDEO_TINY["attention_heads"], sv.VIDEO_TINY["layers"]
    with torch.no_grad():
        out = RV.forward(sd, x, heads, layers)
        feats = RV.features(sd, x, heads, layers)
        feats = torch.nn.functional.layer_norm(feats, feats.shape[-1:], sd["encoder.image_layer_norm.weight"],
                                               sd["encoder.image_layer_norm.bias"]).transpose(0, 1)
    assert out.shape == gold["out"].shape and feats.shape == gold["features"].shape
    torch.testing.assert_close(out, gold["out"], rtol=0, atol=2e-4)
    torch.testing.assert_close(feats, gold["features"], rtol=0, atol=2e-4)


def test_production_keys_match_reference(golden_dir):
    from one_peace_b200.vision.video import OnePeaceViT
    prod = json.loads(zlib.decompress(_gold(golden_dir)["production_z"]))
    with torch.device("meta"):
        big = OnePeaceViT(**sv.PRODUCTION)
    assert _keys(big) == [(k, tuple(s), d) for k, s, d in prod["keys"]]
    assert sorted(big.no_weight_decay()) == prod["no_weight_decay"]
    assert big.get_num_layers() == prod["num_layers"]


def test_init_weights_pretrained_and_adapter_zero_init(golden_dir, tmp_path):
    gold = _gold(golden_dir)["pretrained"]
    path = tmp_path / "ckpt.pkl"
    with open(path, "wb") as f:
        pickle.dump({"model": {k: v.clone() for k, v in gold["ckpt"].items()}}, f)
    m = _tiny(4)
    m.init_weights(pretrained=str(path))
    st = m.state_dict()
    for k, v in gold["loaded"].items():
        assert torch.equal(st[k], v), k
    for layer in m.encoder.layers:
        for ad in (layer.S_Adapter, layer.T_Adapter, layer.MLP_Adapter):
            assert not ad.D_fc2.weight.any() and not ad.D_fc2.bias.any()
            assert ad.D_fc1.weight.any()


def test_init_weights_without_checkpoint():
    m = _tiny(4)
    m.init_weights()
    layer = m.encoder.layers[0]
    assert not layer.T_Adapter.D_fc2.weight.any() and layer.T_Adapter.D_fc1.weight.std() < 0.03
    assert torch.equal(layer.final_layer_norm.weight, torch.ones(128))
    with pytest.raises(TypeError):
        m.init_weights(pretrained=3)


def test_rel_pos_table_of_another_grid_is_resampled():
    m = _tiny(4)
    table = torch.randn(7 * 7 + 3, 2)
    sd = m.resize_rel_pos_embed({"image_adapter.rel_pos_table_list.0.weight": table, "image_adapter.rp_bucket": torch.zeros(1)})
    assert "image_adapter.rp_bucket" not in sd
    got = sd["image_adapter.rel_pos_table.weight"]
    assert got.shape == (7 * 7 + 3, 2) and torch.equal(got, table)      # 4 x 4 bucket -> 7 x 7 grid: nothing to resample
    sd = m.resize_rel_pos_embed({"image_adapter.rel_pos_table_list.0.weight": torch.randn(5 * 5 + 3, 2)})
    assert sd["image_adapter.rel_pos_table.weight"].shape == (7 * 7 + 3, 2)


@pytest.mark.parametrize("kw", [dict(dropout=0.1), dict(attention_dropout=0.1), dict(activation_dropout=0.1),
                                dict(rp_bias=True), dict(shared_rp_bias=False), dict(num_tadapter=2)])
def test_constructor_refusals(kw):
    with pytest.raises(NotImplementedError):
        _tiny(4, **kw)


def test_forward_refusals_raise_before_any_kernel():
    from one_peace_b200 import kernels as K
    m = _tiny(4).eval()
    n0 = K.LAUNCHES
    with torch.no_grad():
        for shape in [(1, 3, 5, 64, 64), (1, 3, 4, 32, 32), (1, 4, 4, 64, 64), (3, 4, 64, 64)]:
            with pytest.raises(ValueError):
                m(torch.zeros(shape))
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 4, 64, 64))              # parameters require grad
    for p in m.parameters():
        p.requires_grad_(False)
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 4, 64, 64, requires_grad=True))
    assert K.LAUNCHES == n0


def test_registration_falls_back_without_mmaction():
    from one_peace_b200.vision import video
    assert video.OnePeaceViT.__name__ == "OnePeaceViT" and "OnePeaceViT" in video.__all__


def test_abi_rejects_bad_arguments():
    from one_peace_b200 import _lib
    lib = _lib.load()
    INVALID = 1
    p, s = 256, 0          # any 16-byte-aligned non-null pointer: every check below fails before a launch
    call = lambda **o: lib.opb_attention_temporal_fwd(*[o.get(n, v) for n, v in [
        ("qkv", p), ("out", p), ("rec", p), ("Bv", 1), ("T", 16), ("N", 257), ("H", 24), ("stream", s)]])
    for bad in [dict(qkv=0), dict(out=0), dict(rec=0), dict(qkv=p + 8), dict(out=p + 2), dict(rec=p + 4), dict(T=1),
                dict(T=33), dict(T=0), dict(Bv=0), dict(N=0), dict(H=0), dict(Bv=-1)]:
        assert call(**bad) == INVALID, bad


def _emul_case():
    import video_emul  # noqa: F401
    from one_peace_b200.vision.video import OnePeaceViT
    T, B = 4, 2
    torch.manual_seed(0)
    m = OnePeaceViT(num_frames=T, **sv.VIDEO_TINY)
    sd = sv.video_state_dict({k: tuple(p.shape) for k, p in m.named_parameters()}, dict(m.named_buffers()))
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    return sd, sv.video_clips(T, B, sv.VIDEO_TINY["bucket_size"]).double()


def test_launch_sequence_emulation_and_planted_mistakes(monkeypatch):
    """The launch sequence of VideoLayer.forward_video, emulated in fp64 (tests/video_emul.py), against the reference's
    computation (restated_video.features in fp64) on 2 layers, 2 clips of 4 frames.
    - Exact arithmetic (rounding points off): |E - R| <= 1e-12 (|R| + rms_row(R)); each planted mistake exceeds it > 100-fold.
    - bf16 rounding points on: |E - R| <= 6 * 2^-8 (|R| + rms_row(R)); each planted mistake exceeds this bound > 30-fold."""
    import video_emul as E
    sd, x = _emul_case()
    heads, layers = sv.VIDEO_TINY["attention_heads"], sv.VIDEO_TINY["layers"]
    R = RV.features(sd, x, heads, layers)
    mag = R.abs() + R.pow(2).mean(-1, keepdim=True).sqrt()
    ratio = lambda got, tau: ((got - R).abs() / (tau * mag)).max().item()
    rounded = ratio(E.features(sd, x, heads, layers), 6 * 2.0 ** -8)
    assert rounded <= 1.0, rounded
    planted_rounded = {mk: ratio(E.features(sd, x, heads, layers, mistake=mk), 6 * 2.0 ** -8) for mk in E.MISTAKES}
    monkeypatch.setattr(E, "rb", lambda t: t)
    exact = ratio(E.features(sd, x, heads, layers), 1e-12)
    assert exact <= 1.0, exact
    planted_exact = {mk: ratio(E.features(sd, x, heads, layers, mistake=mk), 1e-12) for mk in E.MISTAKES}
    print(f"emulation: {rounded:.3f} of the bf16 bound, {exact:.3f} of the exact bound; planted (bf16 bound) "
          f"{ {k: round(v, 1) for k, v in planted_rounded.items()} }")
    for mk in E.MISTAKES:
        assert planted_exact[mk] > 100.0, (mk, planted_exact[mk])
        assert planted_rounded[mk] > 30.0, (mk, planted_rounded[mk])
