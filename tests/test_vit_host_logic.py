"""CPU: OnePeaceViT's module tree against the reference's (tests/golden/vit.pt, made by oracle/make_golden_vit.py): state-dict
keys, shapes and dtypes of the tiny cases and of the four 4B variants, no_weight_decay() and the layer ids of lr_decay's
get_layer_id_for_vit; main_ft.py's loading of a converted pretraining checkpoint; the refusals; the C ABI of the head kernels
refusing bad arguments; and the fp64 head reference (tests/vit_ref.py) against an fp32 emulation and five planted mistakes."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import synth_vit as sv
import vit_ref as V


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "vit.pt"), weights_only=False)


def _keys(model):
    return [(k, tuple(v.shape), str(v.dtype)) for k, v in model.state_dict().items()]


def _meta(variant, **kw):
    from one_peace_b200.vision import models_vit as mv
    with torch.device("meta"):
        return getattr(mv, variant)(**kw)


@pytest.mark.parametrize("case", list(sv.VIT_CASES))
def test_tiny_keys_match_reference(golden_dir, case):
    from one_peace_b200.vision.models_vit import OnePeaceViT
    bucket, pool, _ = sv.VIT_CASES[case]
    m = OnePeaceViT(bucket_size=bucket, global_pool=pool, num_classes=sv.NUM_CLASSES, **sv.VIT_TINY)
    assert _keys(m) == _gold(golden_dir)["cases"][case]["keys"]


@pytest.mark.parametrize("variant", list(sv.BIG_VARIANTS))
@pytest.mark.parametrize("pool", [True, False])
def test_4b_keys_no_weight_decay_and_layer_ids(golden_dir, variant, pool):
    rec = sv.big_records(_gold(golden_dir))[(variant, pool)]
    m = _meta(variant, global_pool=pool)
    assert _keys(m) == rec["keys"]
    names = [k for k, _, _ in rec["keys"]]
    assert not any(s in k for k in names for s in ("version", "position_idx", "rel_pos_table_list"))
    assert ("encoder.layer_norm.weight" in names) == (not pool) and ("fc_norm.weight" in names) == pool
    assert sorted(m.no_weight_decay()) == rec["no_weight_decay"]
    assert isinstance(m.encoder.layers, torch.nn.ModuleList) and len(m.encoder.layers) == 40
    n_layers = len(m.encoder.layers) + 1

    def layer_id(name):                              # utils/lr_decay.py: get_layer_id_for_vit, restated
        if name.startswith("image_adapter"):
            return 0
        if name.startswith("encoder.layers"):
            return int(name.split(".")[2]) + 1
        return n_layers
    assert {n: layer_id(n) for n, _ in m.named_parameters()} == rec["layer_ids"]


def test_constructor_arguments_of_main_ft():
    """main_ft.py:269-275 passes these keywords; drop_path follows the linspace schedule."""
    from one_peace_b200.vision.models_vit import one_piece_g_256
    m = one_piece_g_256(num_classes=10, drop_path_rate=0.3, dropout=0.0, global_pool=True, use_checkpoint=True, layers=4,
                        embed_dim=256, ffn_embed_dim=1024, attention_heads=4)
    assert [layer.drop_path_prob for layer in m.encoder.layers] == pytest.approx([0.0, 0.1, 0.2, 0.3])
    assert all(float(layer.gamma_1.detach()[0]) == pytest.approx(1e-2) for layer in m.encoder.layers)
    w, b = m.head.weight.detach(), m.head.bias.detach()
    assert w.abs().max() <= 2.0 * 0.001 and 1.5e-5 < w.std() < 2.5e-5           # trunc_normal_(std=.02) * init_scale
    assert b.abs().max() <= 0.001 / 256 ** 0.5                                  # nn.Linear's bias init * init_scale


@pytest.mark.parametrize("kw", [dict(dropout=0.1), dict(attention_dropout=0.1), dict(activation_dropout=0.1),
                                dict(rp_bias=True), dict(shared_rp_bias=False)])
def test_refusals(kw):
    from one_peace_b200.vision.models_vit import OnePeaceViT
    with pytest.raises(NotImplementedError):
        OnePeaceViT(layers=1, embed_dim=256, ffn_embed_dim=1024, attention_heads=4, **kw)


@pytest.mark.parametrize("shape", [(1, 3, 128, 128), (1, 3, 64, 48), (1, 3, 80, 80)])
def test_resolution_refused_before_any_kernel(shape):
    from one_peace_b200 import kernels as K
    from one_peace_b200.vision.models_vit import OnePeaceViT
    m = OnePeaceViT(layers=1, embed_dim=256, ffn_embed_dim=1024, attention_heads=4, bucket_size=4).eval()
    before = K.LAUNCHES
    with pytest.raises(ValueError):
        m(torch.zeros(shape))
    assert K.LAUNCHES == before


def _converted_checkpoint(src_bucket, d=256, heads=4, layers=2):
    """A converted pretraining checkpoint (convert_to_vision.py's layout): per-layer table list, rp_bucket of the pretraining
    grid, pos_embed of a src_bucket^2 grid."""
    g = torch.Generator().manual_seed(7)
    nrd = (2 * src_bucket - 1) ** 2 + 3
    m = _meta_free_tiny(src_bucket, d, heads, layers)
    ck = {k: torch.randn(v.shape, generator=g) if v.is_floating_point() else v.clone() for k, v in m.state_dict().items()}
    ck["image_adapter.rel_pos_table_list.0.weight"] = ck.pop("image_adapter.rel_pos_table.weight")
    assert ck["image_adapter.rel_pos_table_list.0.weight"].shape == (nrd, heads)
    del ck["head.weight"], ck["head.bias"]
    return ck


def _meta_free_tiny(bucket, d=256, heads=4, layers=2, **kw):
    from one_peace_b200.vision.models_vit import OnePeaceViT
    return OnePeaceViT(bucket_size=bucket, layers=layers, embed_dim=d, ffn_embed_dim=4 * d, attention_heads=heads, **kw)


def test_main_ft_loading_path():
    """main_ft.py:285-294 restated: pop rp_bucket, interpolate pos_embed bicubically (utils/pos_embed.py), copy
    rel_pos_table_list.0 to rel_pos_table and resample it onto the larger grid, then a non-strict load."""
    from one_peace_b200.adapter.image import geometric_sequence_interpolation
    ck = _converted_checkpoint(4)
    model = _meta_free_tiny(6, num_classes=5)
    ck.pop("image_adapter.rp_bucket", None)
    pe = ck["image_adapter.pos_embed"]
    n_new = model.image_adapter.bucket_size
    n_old = int((pe.shape[0] - 1) ** 0.5)
    tok = pe[1:].reshape(-1, n_old, n_old, pe.shape[1]).permute(0, 3, 1, 2)
    tok = F.interpolate(tok, size=(n_new, n_new), mode="bicubic", align_corners=False).permute(0, 2, 3, 1).flatten(0, 2)
    ck["image_adapter.pos_embed"] = torch.cat([pe[:1], tok], 0)
    rel = ck["image_adapter.rel_pos_table_list.0.weight"].clone()
    src = int((rel.shape[0] - 3) ** 0.5)
    dst = int((model.state_dict()["image_adapter.rel_pos_table.weight"].shape[0] - 3) ** 0.5)
    new = geometric_sequence_interpolation(src, dst, rel[:-3], rel.shape[1])
    ck["image_adapter.rel_pos_table.weight"] = torch.cat([new, rel[-3:]], 0)
    missing, unexpected = model.load_state_dict(ck, strict=False)
    assert sorted(missing) == ["head.bias", "head.weight", "image_adapter.rp_bucket"]
    assert unexpected == ["image_adapter.rel_pos_table_list.0.weight"]
    t = model.image_adapter.rel_pos_table.weight.detach()
    assert t.shape == ((2 * 6 - 1) ** 2 + 3, 4) and torch.equal(t[-3:], rel[-3:])
    # the resampled grid passes through the source offsets: the centre (offset 0, 0) is kept
    assert torch.allclose(t[:-3].view(11, 11, 4)[5, 5], rel[:-3].view(7, 7, 4)[3, 3], atol=1e-5)
    assert model.image_adapter.pos_embed.shape == (37, 256)


def test_strict_load_of_a_full_state_dict():
    m = _meta_free_tiny(4, global_pool=False, num_classes=3)
    sd = {k: torch.zeros_like(v) for k, v in m.state_dict().items()}
    m.load_state_dict(sd, strict=True)


def _abi():
    from one_peace_b200 import _lib
    return _lib.load()


def test_abi_rejects_bad_arguments_without_a_gpu():
    """Every refusal returns status 1 before any CUDA call (the checks need no device)."""
    lib = _abi()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    p16 = (p + 15) // 16 * 16
    assert lib.opb_token_mean_ln_ws_floats(0, 17, 256) == -1
    assert lib.opb_token_mean_ln_ws_floats(2, 1, 256) == -1
    assert lib.opb_token_mean_ln_ws_floats(2, 17, 254) == -1
    assert lib.opb_token_mean_ln_ws_floats(70000, 17, 256) == -1
    assert lib.opb_token_mean_ln_ws_floats(2, 17, 256) > 0
    ws_need = lib.opb_token_mean_ln_ws_floats(2, 17, 256)

    def fwd(x=p16, ld=256, B=2, S=17, d=256, eps=1e-5, ws=p16, n_ws=ws_need, m=p16):
        return lib.opb_token_mean_ln_fwd(x, ld, B, S, d, p, p, eps, ws, n_ws, m, p, p, p, None)
    for bad in (dict(x=None), dict(m=None), dict(ld=255), dict(ld=258), dict(B=0), dict(S=1), dict(d=6), dict(eps=-1.0),
                dict(eps=float("nan")), dict(x=p16 + 4), dict(ws=p16 + 4), dict(n_ws=ws_need - 1)):
        assert fwd(**bad) == 1, bad

    def bwd(dy=p, B=2, S=17, d=256, ws=p16, dx=p16, ld=256):
        return lib.opb_token_mean_ln_bwd(dy, p, p, p, p, B, S, d, p, p, ws, dx, ld, None)
    for bad in (dict(dy=None), dict(dx=None), dict(ws=None), dict(B=0), dict(S=1), dict(d=10), dict(ld=100), dict(ld=262),
                dict(dx=p16 + 8), dict(ws=p16 + 4)):
        assert bwd(**bad) == 1, bad


def test_wrappers_refuse_bad_layouts():
    from one_peace_b200 import kernels as K
    with pytest.raises(RuntimeError):             # CPU tensors: no CPU path
        K.token_mean_ln_fwd(torch.zeros(2, 17, 256), torch.ones(256), torch.zeros(256), 1e-5)


# ---- the fp64 reference and its bounds ----
def _case(B, S, d, seed, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, d, generator=g) + offset * torch.randn(1, 1, d, generator=g)
    gamma = 1.0 + 0.2 * torch.randn(d, generator=g)
    beta = 0.1 * torch.randn(d, generator=g)
    dy = torch.randn(B, d, generator=g)
    return x.float(), gamma.float(), beta.float(), dy.float()


@pytest.mark.parametrize("B,S,d", [(1, 17, 256), (4, 257, 256), (3, 577, 1536), (2, 1025, 1536)])
def test_fp32_emulation_within_bounds(B, S, d):
    x, gamma, beta, dy = _case(B, S, d, seed=B * S + d, offset=1.0)
    r = V.head_fwd(x, gamma, beta, 1e-5)
    y, m, mean, rstd = V.emulate_fwd(x, gamma, beta, 1e-5)
    assert V.excess(m, r["m"], r["b_m"]) <= 1.0
    assert V.excess(mean, r["mean"], r["b_mean"]) <= 1.0
    assert V.excess(rstd, r["rstd"], r["b_rstd"]) <= 1.0
    assert V.excess(y, r["y"], r["b_y"]) <= 1.0
    rb = V.head_bwd(dy, m, mean, rstd, gamma, S)
    dx, dgamma, dbeta = V.emulate_bwd(dy, m, mean, rstd, gamma, S)
    assert V.excess(dx, rb["dx"], rb["b_dx"]) <= 1.0
    assert V.excess(dgamma, rb["dgamma"], rb["b_dgamma"]) <= 1.0
    assert V.excess(dbeta, rb["dbeta"], rb["b_dbeta"]) <= 1.0


def test_reference_matches_autograd():
    """The fp64 reference is the reference's expression: x[:, 1:].mean(1) -> LayerNorm, and its autograd adjoint."""
    x, gamma, beta, dy = _case(3, 17, 256, seed=3)
    xd = x.double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    y = F.layer_norm(xd[:, 1:].mean(1), (256,), gd, bd, 1e-5)
    (y * dy.double()).sum().backward()
    r = V.head_fwd(x, gamma, beta, 1e-5)
    assert torch.allclose(r["y"], y.detach(), rtol=1e-12, atol=1e-12)
    rb = V.head_bwd(dy, r["m"], r["mean"], r["rstd"], gamma, 17)
    assert torch.allclose(rb["dx"], xd.grad, rtol=1e-10, atol=1e-13)
    assert torch.equal(rb["dx"][:, 0], torch.zeros(3, 256, dtype=torch.float64))
    assert torch.allclose(rb["dgamma"], gd.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(rb["dbeta"], bd.grad, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("mistake", sorted(set(V.MISTAKES_FWD + V.MISTAKES_BWD)))
def test_planted_mistakes_exceed_a_bound(mistake):
    B, S, d = 4, 17, 256
    x, gamma, beta, dy = _case(B, S, d, seed=11, offset=1.0)
    r = V.head_fwd(x, gamma, beta, 1e-5)

    def fwd_excess(planted):
        y, m, mean, rstd = V.emulate_fwd(x, gamma, beta, 1e-5, planted)
        return max(V.excess(m, r["m"], r["b_m"]), V.excess(mean, r["mean"], r["b_mean"]),
                   V.excess(rstd, r["rstd"], r["b_rstd"]), V.excess(y, r["y"], r["b_y"]))
    y, m, mean, rstd = V.emulate_fwd(x, gamma, beta, 1e-5)
    rb = V.head_bwd(dy, m, mean, rstd, gamma, S)

    def bwd_excess(planted):
        dx, dgamma, dbeta = V.emulate_bwd(dy, m, mean, rstd, gamma, S, planted)
        return max(V.excess(dx, rb["dx"], rb["b_dx"]), V.excess(dgamma, rb["dgamma"], rb["b_dgamma"]),
                   V.excess(dbeta, rb["dbeta"], rb["b_dbeta"]))
    assert fwd_excess(None) <= 1.0 and bwd_excess(None) <= 1.0
    worst = max(fwd_excess(mistake) if mistake in V.MISTAKES_FWD else 0.0, bwd_excess(mistake) if mistake in V.MISTAKES_BWD else 0.0)
    assert worst > 100.0, (mistake, worst)


def test_timm_criteria_restatement():
    """synth_vit's timm formulas: label smoothing is torch's cross_entropy(label_smoothing=s), which is what the kernel's
    hard-label mode computes; soft targets reduce to the hard loss for one-hot targets."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(8, 37, generator=g, dtype=torch.float64)
    lab = torch.randint(0, 37, (8,), generator=g)
    assert torch.allclose(sv.label_smoothing_ce(x, lab), F.cross_entropy(x, lab, label_smoothing=sv.SMOOTHING))
    assert torch.allclose(sv.soft_target_ce(x, F.one_hot(lab, 37).double()), F.cross_entropy(x, lab))
    assert np.isfinite(sv.soft_target_ce(x, torch.softmax(x, 1)).item())
