"""CPU: the video backbone's training path, host side.  Train-mode shape errors raise before any kernel runs, eval mode
keeps its refusal under grad, the C ABI rejects bad arguments of the temporal-attention backward and the GELU pair
before any launch, the drop-path draw order, and the parameter order of the layer adjoint."""
import pytest
import torch

import synth_video as sv


def _tiny(T, **kw):
    from one_peace_b200.vision.video import OnePeaceViT
    torch.manual_seed(0)
    return OnePeaceViT(num_frames=T, **{**sv.VIDEO_TINY, **kw})


def test_train_mode_shape_errors_raise_before_any_kernel():
    from one_peace_b200 import kernels as K
    m = _tiny(4).train()
    n0 = K.LAUNCHES
    for shape in [(1, 3, 5, 64, 64), (1, 3, 4, 32, 32), (1, 4, 4, 64, 64), (3, 4, 64, 64)]:
        with pytest.raises(ValueError):
            m(torch.zeros(shape))
        with pytest.raises(ValueError):
            m.forward_features(torch.zeros(shape))
    assert K.LAUNCHES == n0


def test_eval_mode_refusal_is_unchanged():
    from one_peace_b200 import kernels as K
    m = _tiny(4).eval()
    n0 = K.LAUNCHES
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 4, 64, 64))
    assert K.LAUNCHES == n0


def test_abi_rejects_bad_arguments():
    from one_peace_b200 import _lib
    lib = _lib.load()
    INVALID, p = 1, 256
    names = ["qkv", "out", "dout", "dqkv", "Bv", "T", "N", "H", "qs", "stream"]
    base = dict(qkv=p, out=p, dout=p, dqkv=p, Bv=1, T=16, N=257, H=24, qs=0.125, stream=0)
    call = lambda **o: lib.opb_attention_temporal_bwd(*[{**base, **o}[n] for n in names])
    for bad in [dict(qkv=0), dict(out=0), dict(dout=0), dict(dqkv=0), dict(qkv=p + 8), dict(out=p + 2), dict(dout=p + 4),
                dict(dqkv=p + 8), dict(T=1), dict(T=33), dict(T=0), dict(Bv=0), dict(N=0), dict(H=0), dict(Bv=-1)]:
        assert call(**bad) == INVALID, bad
    for bad in [(0, p, 4, 8), (p, 0, 4, 8), (p, p, 0, 8), (p, p, 4, 12), (p + 2, p, 4, 8), (p, p, 4, 0)]:
        assert lib.opb_gelu_fwd(*bad, None) == INVALID, bad
    for bad in [(0, p, p, 4, 8), (p, 0, p, 4, 8), (p, p, 0, 4, 8), (p, p, p, 4, 12), (p, p + 8, p, 4, 8), (p, p, p, -1, 8)]:
        assert lib.opb_gelu_bwd(*bad, None) == INVALID, bad


def test_drop_path_draw_order_and_scales():
    """Three per-frame draws per layer with p > 0, temporal, spatial, MLP adapter in that order, each repeated over the
    N rows of its frame; eval mode and p = 0 draw nothing."""
    from one_peace_b200.vision.video import draw_row_scales
    m = _tiny(4, drop_path_rate=0.5).train()
    Bv, T, N = 2, 4, 17
    torch.manual_seed(11)
    got = draw_row_scales(m.encoder.layers, Bv, T, N, torch.device("cpu"))
    torch.manual_seed(11)
    assert got[0] == (None, None, None)                          # linspace(0, 0.5, 2): layer 0 has p = 0
    p = m.encoder.layers[1].drop_path_prob
    for r in got[1]:
        want = ((torch.rand(Bv * T) < 1 - p).float() / (1 - p)).repeat_interleave(N)
        assert torch.equal(r, want)
    m.eval()
    assert all(t == (None, None, None) for t in draw_row_scales(m.encoder.layers, Bv, T, N, torch.device("cpu")))


def test_layer_gradient_order_names_every_parameter_once():
    from one_peace_b200.vision.video import video_params
    m = _tiny(4)
    for layer in m.encoder.layers:
        ps = video_params(layer)
        assert len(ps) == 33 and len({id(q) for q in ps}) == 33
        assert {id(q) for q in ps} == {id(q) for q in layer.parameters()}


def test_activation_bytes_per_row():
    from one_peace_b200.vision.video import video_row_bytes
    # 28 d (both passes' h1, qkv, att, a2, o) + 3 d (six d / 4 adapter tensors) + 10 d + 8 d (fp32 y, x1) + 8 F + 4 H
    assert video_row_bytes(1536, 6144, 24) == 49 * 1536 + 8 * 6144 + 96
