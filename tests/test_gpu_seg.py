"""GPU: the segmentation kernels (csrc/seg.cu) against the fp64 references of tests/seg_ref.py with per-element bounds,
NaN canaries, bit-identical repeats and the argument checks; the tiny backbone against tests/golden/seg.pt (the reference's
own onepeace_adapter.py in fp64); the production backbone at 896^2; autocast leaving the outputs unchanged."""
import ctypes
import os

import pytest
import torch

import seg_ref as R
import synth_seg as ss

pytestmark = pytest.mark.gpu

DEV = "cuda"
LEVELS = {"tiny": [(8, 8), (4, 4), (2, 2)], "production": [(112, 112), (56, 56), (28, 28)],
          "non_square": [(6, 10), (3, 5), (2, 3)], "odd": [(7, 5), (3, 1)]}


def _share(err, bound):
    return (err / bound).max().item()


@pytest.mark.parametrize("levels", list(LEVELS))
@pytest.mark.parametrize("C", [32, 384])
@pytest.mark.parametrize("B", [1, 2])
def test_dwconv_gelu_against_fp64(levels, C, B):
    from one_peace_b200 import kernels as K
    shapes = LEVELS[levels]
    T = sum(h * w for h, w in shapes)
    g = torch.Generator().manual_seed(C + B)
    x = torch.randn(B * T, C, generator=g).to(torch.bfloat16)
    w = torch.randn(C, 1, 3, 3, generator=g) / 3
    b = 0.1 * torch.randn(C, generator=g)
    y, z, a = R.dwconv_gelu_ref(x.double(), w, b, shapes, B)
    wd = w.reshape(C, 9).t().contiguous().to(DEV)
    buf = torch.full((B * T + 64, C), float("nan"), dtype=torch.bfloat16, device=DEV)
    out = buf[32:32 + B * T]
    K.seg_dwconv_gelu(x.to(DEV), wd, b.to(DEV), shapes, B, out=out)
    got = out.double().cpu()
    share = _share((got - y).abs(), R.dwconv_gelu_bound(y, z, a))
    print(f"dwconv {levels} C={C} B={B}: largest share of the bound {share:.3f}")
    assert share <= 1.0
    assert torch.isnan(buf[:32].float()).all() and torch.isnan(buf[32 + B * T:].float()).all()
    again = K.seg_dwconv_gelu(x.to(DEV), wd, b.to(DEV), shapes, B)
    assert torch.equal(again, out)


MAPS = {"tiny_c1": (16, 16, 4, True), "tiny_c4": (2, 2, 4, False), "prod_c1": (224, 224, 56, True),
        "prod_c2": (112, 112, 56, False), "prod_c3": (56, 56, 56, False), "prod_c4": (28, 28, 56, False),
        "non_square": (12, 20, 5, True), "odd": (7, 3, 5, False)}


@pytest.mark.parametrize("case", list(MAPS))
@pytest.mark.parametrize("C", [32, 384])
@pytest.mark.parametrize("B", [1, 2])
def test_out_map_against_fp64(case, C, B):
    from one_peace_b200 import kernels as K
    H, W, gw, with_extra = MAPS[case]
    if B == 2 and C == 384 and case.startswith("prod"):
        C = 64
    g = torch.Generator().manual_seed(H + C + B)
    pad_c, pad_x = 3, 1                          # rows before each sample's map: the kernels index past them
    c = torch.randn(B, pad_c + H * W, C, generator=g)
    x = torch.randn(B, pad_x + gw * gw, C, generator=g)
    extra = torch.randn(B * (H // 2) * (W // 2), 4 * C, generator=g) if with_extra else None
    scale, shift = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    c_grid = c[:, pad_c:].transpose(1, 2).reshape(B, C, H, W)
    x_grid = x[:, pad_x:].transpose(1, 2).reshape(B, C, gw, gw)
    e_grid = None
    if with_extra:
        e_grid = extra.view(B, H // 2, W // 2, 2, 2, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, H, W)
    want, bound = R.out_map_ref(c_grid, x_grid, scale, shift, e_grid)
    buf = torch.full((B * C * H * W + 64,), float("nan"), device=DEV)
    out = buf[32:32 + B * C * H * W].view(B, C, H, W)
    args = (c.to(DEV).reshape(-1, C), pad_c + H * W, pad_c, x.to(DEV).reshape(-1, C), pad_x + gw * gw, pad_x, gw,
            scale.to(DEV), shift.to(DEV), B, H, W)
    ex = extra.to(DEV) if with_extra else None
    K.seg_out_map(*args, extra=ex, out=out)
    share = _share((out.double().cpu() - want).abs(), bound)
    print(f"out_map {case} C={C} B={B}: largest share of the bound {share:.3f}")
    assert share <= 1.0
    assert torch.isnan(buf[:32]).all() and torch.isnan(buf[32 + B * C * H * W:]).all()
    assert torch.equal(K.seg_out_map(*args, extra=ex), out)


def test_invalid_arguments_rejected_before_launch():
    from one_peace_b200 import _lib
    lib = _lib.load()
    t = torch.zeros(1024, dtype=torch.float32, device=DEV)
    p, q = t.data_ptr(), t.data_ptr() + 4                     # q: not 16-byte aligned
    hw = (ctypes.c_int32 * 2)(2, 2)
    bad_hw = (ctypes.c_int32 * 2)(0, 2)
    assert lib.opb_seg_dwconv_gelu(p, p, p, p, 1, 8, 1, hw, None) == 0
    torch.cuda.synchronize()
    for args in [(q, p, p, p, 1, 8, 1, hw), (p, p, p, None, 1, 8, 1, hw), (p, p, p, p, 1, 12, 1, hw),
                 (p, p, p, p, 0, 8, 1, hw), (p, p, p, p, 1, 8, 5, hw), (p, p, p, p, 1, 8, 1, bad_hw),
                 (p, p, p, p, 1, 8, 1, None)]:
        assert lib.opb_seg_dwconv_gelu(*args, None) == 1, args
    good = (p, 4, 0, p, 4, 0, 2, None, p, p, p, 1, 32, 2, 2)
    for i, v in [(0, None), (10, None), (12, 16), (13, 0), (1, 3), (4, 3), (6, 0)]:
        a = list(good)
        a[i] = v
        assert lib.opb_seg_out_map(*a, None) == 1, (i, v)
    a = list(good)
    a[7], a[13] = p, 3                                         # extra with an odd side
    assert lib.opb_seg_out_map(*a, None) == 1


def _tiny_model():
    """The fixture's tiny model, weights drawn on the CPU as the fixture's were, moved with .to()."""
    from one_peace_b200.vision.seg import OnePeaceAdapter
    torch.manual_seed(0)
    m = OnePeaceAdapter(**ss.SEG_TINY)
    m.load_state_dict(ss.seg_state_dict(m), strict=True)
    return m.to(DEV).eval().requires_grad_(False)


def _production_model():
    """The production config on the GPU with synth_seg's weights drawn there (built on the meta device: initialising 1.5 B
    parameters on the host would take minutes)."""
    from one_peace_b200.vision.seg import OnePeaceAdapter, make_image_bucket_position
    torch.manual_seed(0)
    with torch.device("meta"):
        m = OnePeaceAdapter(**ss.PRODUCTION)
    m = m.to_empty(device=DEV)
    layers = m.encoder.layers
    assert all(layer.rp_bucket is layers[0].rp_bucket for layer in layers)
    layers[0].rp_bucket.copy_(make_image_bucket_position(56, 111 ** 2 + 3))       # to_empty leaves buffers unset
    m.load_state_dict(ss.seg_state_dict(m, device=DEV), strict=True)
    return m.eval().requires_grad_(False)


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.double().flatten(), b.double().flatten(), dim=0).item()


def _check_layer_biases(m, layers):
    """Layer i's LUT-form bias (SegEncoder.biases) expanded to the dense (H, S, S) table equals its own
    F.embedding(rp_bucket, rel_pos_table) exactly."""
    biases = m.encoder.biases()
    for i in layers:
        layer, rp = m.encoder.layers[i], biases[i]
        S = layer.rp_bucket.shape[0]
        codes = rp.code_row[:S].long()[:, None] - rp.code_col[:S].long()[None, :]
        dense = rp.lut[:, codes]
        want = torch.nn.functional.embedding(layer.rp_bucket, layer.rel_pos_table.weight.float()).permute(2, 0, 1)
        assert torch.equal(dense, want), i


def test_tiny_model_against_reference(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "seg.pt"), weights_only=False)
    m = _tiny_model()
    _check_layer_biases(m, range(len(m.encoder.layers)))
    x = ss.seg_images(2, ss.SEG_TINY["bucket_size"]).to(DEV)
    for B in (2, 1):
        with torch.no_grad():
            got = m(x[:B])
        for i, (f, want) in enumerate(zip(got, gold["maps"])):
            want = want[:B]
            assert f.shape == want.shape and f.dtype == torch.float32
            f = f.double().cpu()
            cos = _cos(f, want)
            rel = ((f - want).abs().max() / want.double().pow(2).mean().sqrt()).item()
            print(f"tiny B={B} map {i + 1}: cosine {cos:.6f}, worst |error| / rms {rel:.4f}")
            assert cos >= 0.9999, (B, i, cos)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        again = m(x)
    with torch.no_grad():
        plain = m(x)
    for a, b in zip(again, plain):
        assert torch.equal(a, b)


def test_production_backbone_896_against_fp32_restatement():
    import restated_seg as RS
    m = _production_model()
    _check_layer_biases(m, (0, 39))
    x = ss.seg_images(2, 56, device=DEV)
    cfg = ss.PRODUCTION
    with torch.no_grad():
        one = m(x[:1])
        two = m(x)
        tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        try:
            want = RS.forward(m.state_dict(), x[:1], cfg["attention_heads"], cfg["deform_num_heads"], cfg["n_points"],
                              cfg["interaction_indexes"])
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    sides = [224, 112, 56, 28]
    for f1, f2, w, s in zip(one, two, want, sides):
        assert f1.shape == (1, 1536, s, s) and f2.shape == (2, 1536, s, s) and w.shape == f1.shape
        assert torch.isfinite(f2).all()
        cos, cos_b = _cos(f1, w), _cos(f1, f2[:1])
        rel = ((f1 - w).abs().max() / w.pow(2).mean().sqrt()).item()
        print(f"production {s}^2: cosine {cos:.6f} against the fp32 restatement, worst |error| / rms {rel:.4f}; "
              f"B=1 against sample 0 of B=2: cosine {cos_b:.7f}")
        assert cos >= 0.9999 and cos_b >= 0.9999
