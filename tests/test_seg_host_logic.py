"""CPU: the segmentation backbone's host logic against tests/golden/seg.pt (the reference's own onepeace_adapter.py): the
refusals, the tiny and production key / shape / dtype lists and registration order, init_weights() with .pkl and .pth
checkpoints, the level layout and reference points, the per-layer LUT form of the bias, the BatchNorm fold and the
transposed-conv weight rearrangement."""
import json
import os
import pickle
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import synth_seg as ss
from one_peace_b200 import relpos
from one_peace_b200.vision import seg as S


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "seg.pt"), weights_only=False)


def _keys(m):
    return [(k, tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()]


def _tiny(**kw):
    torch.manual_seed(0)
    return S.OnePeaceAdapter(**{**ss.SEG_TINY, **kw})


@pytest.mark.parametrize("kw", [dict(dropout=0.1), dict(attention_dropout=0.1), dict(activation_dropout=0.1),
                                dict(rp_bias=False), dict(shared_rp_bias=True), dict(with_cffn=False),
                                dict(add_vit_feature=False), dict(interaction_indexes=[[0, 1], [3, 3]]),
                                dict(interaction_indexes=[[0, 1], [2, 2]]), dict(interaction_indexes=[[1, 3]]),
                                dict(interaction_indexes=None), dict(deform_ratio=1.0), dict(deform_num_heads=4),
                                dict(bucket_size=5)])
def test_constructor_refusals(kw):
    with pytest.raises(NotImplementedError):
        _tiny(**kw)


def test_forward_refusals():
    m = _tiny()
    with pytest.raises(ValueError):
        m(torch.zeros(1, 3, 48, 64))
    with pytest.raises(ValueError):
        m(torch.zeros(3, 64, 64))
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 64, 64))       # parameters require a gradient
    with torch.no_grad(), pytest.raises(NotImplementedError):
        m.train()(torch.zeros(1, 3, 64, 64))                   # BatchNorm runs only with its running statistics


@pytest.mark.parametrize("move", ["to_float64", "to_meta", "clone", "to_empty"])
def test_rp_bucket_stays_one_tensor(move):
    m = _tiny()
    if move == "to_float64":
        m.to(torch.float64)
    elif move == "to_meta":
        m.to("meta")
    elif move == "clone":
        m._apply(lambda t: t.clone())
    else:
        m.to_empty(device="cpu")
    layers = m.encoder.layers
    assert all(layer.rp_bucket is layers[0].rp_bucket for layer in layers)
    assert layers[0].rp_bucket.dtype == torch.int64
    sd = m.state_dict()
    ptr = layers[0].rp_bucket.untyped_storage().data_ptr()
    assert all(sd[f"encoder.layers.{i}.rp_bucket"].untyped_storage().data_ptr() == ptr for i in range(len(layers)))


def test_restatement_matches_reference(golden_dir):
    """oracle/restated_seg.py, the fp32 yardstick of the GPU tests, in fp64 against the reference's own backbone."""
    import restated_seg as RS
    gold = _gold(golden_dir)
    m = _tiny()
    sd = {k: v.double() if v.is_floating_point() else v for k, v in ss.seg_state_dict(m).items()}
    cfg = ss.SEG_TINY
    with torch.no_grad():
        fs = RS.forward(sd, ss.seg_images(2, cfg["bucket_size"]).double(), cfg["attention_heads"], cfg["deform_num_heads"],
                        cfg["n_points"], cfg["interaction_indexes"])
    for f, want in zip(fs, gold["maps"]):
        torch.testing.assert_close(f.float(), want, rtol=0, atol=1e-5)


def test_tiny_and_production_keys_match_reference(golden_dir):
    gold = _gold(golden_dir)
    assert _keys(_tiny()) == [tuple(k) for k in gold["keys"]]
    prod = json.loads(zlib.decompress(gold["production_z"]))
    with torch.device("meta"):
        big = S.OnePeaceAdapter(**ss.PRODUCTION)
    assert _keys(big) == [(k, tuple(s), d) for k, s, d in prod["keys"]]
    buckets = {layer.rp_bucket.data_ptr() for layer in _tiny().encoder.layers}
    assert len(buckets) == 1                   # one tensor under every layer's name


def test_strict_load_of_reference_state(golden_dir):
    m = _tiny()
    sd = ss.seg_state_dict(m)
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("ext", ["pkl", "pth"])
def test_init_weights_pretrained(ext, golden_dir, tmp_path):
    gold = _gold(golden_dir)["pretrained"]
    path = str(tmp_path / f"ckpt.{ext}")
    ckpt = {k: v.clone() for k, v in gold["ckpt"].items()}
    if ext == "pkl":
        with open(path, "wb") as f:
            pickle.dump({"model": ckpt}, f)
    else:
        torch.save({"state_dict": ckpt}, path)
    m = _tiny(pretrained=path)
    m.init_weights()
    st = m.state_dict()
    for k, v in gold[ext].items():
        torch.testing.assert_close(st[k], v, rtol=0, atol=2e-6, msg=k)


def test_level_layout_and_reference_points(golden_dir):
    d1, d2 = _gold(golden_dir)["deform_inputs"]
    side = ss.SEG_TINY["bucket_size"]
    shapes = S.level_shapes(side)
    assert d1[1].tolist() == [list(s) for s in shapes] and d2[1].tolist() == [[side, side]]
    assert d1[2].tolist() == [0, shapes[0][0] * shapes[0][1], shapes[0][0] * shapes[0][1] + shapes[1][0] * shapes[1][1]]
    assert torch.equal(S.reference_points([(side, side)]), d1[0].reshape(-1, 2))
    assert torch.equal(S.reference_points(shapes), d2[0].reshape(-1, 2))


@pytest.mark.parametrize("side", [4, 7])
def test_layer_lut_reproduces_embedding(side):
    n = (2 * side - 1) ** 2 + 3
    bucket = S.make_image_bucket_position(side, n)
    table = torch.randn(n, 3, generator=torch.Generator().manual_seed(side), dtype=torch.float64)
    S_ = side * side + 1
    idx, cr, cc = relpos.build_lut_index(bucket.numpy(), relpos.image_codes(S_, side))
    lut = table[torch.from_numpy(idx.astype(np.int64))].t()                      # relpos_lut_build: lut[h][l]
    dense = lut[:, torch.from_numpy(cr[:S_, None].astype(np.int64) - cc[None, :S_].astype(np.int64))]
    assert torch.equal(dense, F.embedding(bucket, table).permute(2, 0, 1))


def test_bn_fold_and_convt_rearrangement():
    g = torch.Generator().manual_seed(5)
    bn = torch.nn.BatchNorm2d(6).double().eval()
    with torch.no_grad():
        for t in (bn.weight, bn.bias, bn.running_mean):
            t.copy_(torch.randn(6, generator=g, dtype=torch.float64))
        bn.running_var.copy_(0.5 + torch.rand(6, generator=g, dtype=torch.float64))
    x = torch.randn(2, 6, 3, 3, generator=g, dtype=torch.float64)
    scale, shift = S.fold_bn(bn)
    torch.testing.assert_close(x * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1), bn(x), rtol=0, atol=1e-12)
    w = torch.randn(5, 4, 2, 2, generator=g, dtype=torch.float64)
    xs = torch.randn(2, 5, 3, 2, generator=g, dtype=torch.float64)
    y = (xs.permute(0, 2, 3, 1).reshape(-1, 5) @ S.convt_weight(w).t()).view(2, 3, 2, 2, 2, 4)   # (b, i, j, dy, dx, c)
    y = y.permute(0, 5, 1, 3, 2, 4).reshape(2, 4, 6, 4)
    torch.testing.assert_close(y, F.conv_transpose2d(xs, w, stride=2), rtol=0, atol=1e-12)
