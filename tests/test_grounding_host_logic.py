"""CPU: the fp64 reference of the grounding kernels (tests/grounding_ref.py) against torchvision and torch.autograd, its error
bounds against an fp32 emulation of the kernel arithmetic and six planted mistakes, the image adapter's checkpoint upgrade
against the reference's (tests/golden/refcoco.pt, made by oracle/make_golden_grounding.py), and the names of the
criterion, its registration and the metric."""
import os

import pytest
import torch

import grounding_ref as G
import synth_grounding as sg


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "refcoco.pt"), weights_only=False)


def boxes_case(B, seed, kind="mixed"):
    """logits fp32 [B, 4] and target boxes [B, 4]; kind: 'mixed' (random logits), 'valid' (p0 < p2, p1 < p3 for every row),
    'invalid' (no row valid)."""
    g = torch.Generator().manual_seed(seed)
    z = 1.5 * torch.randn(B, 4, generator=g)
    if kind != "mixed":
        lo = torch.minimum(z[:, :2], z[:, 2:]) - 0.05
        hi = torch.maximum(z[:, :2], z[:, 2:]) + 0.05
        z = torch.cat([lo, hi], 1) if kind == "valid" else torch.cat([hi, lo], 1)
    return z.float(), sg.random_boxes(g, B).float()


def planted_case():
    """Random rows plus rows that expose the planted mistakes: ties p0 == p2 (validity is strict) and reversed predictions
    against reversed targets (the enclosing box's extents are negative, so only its clamp keeps GIoU from a finite value)."""
    z, t = boxes_case(64, 11)
    tie = torch.tensor([[0.3, -0.4, 0.3, 0.8], [-0.2, -1.0, -0.2, 0.1]])
    rev_z = torch.tensor([[2.2, 2.2, -2.2, -2.2]])
    rev_t = torch.tensor([[0.8, 0.8, 0.2, 0.2]])
    z = torch.cat([z, tie, rev_z]).float()
    t = torch.cat([t, sg.random_boxes(torch.Generator().manual_seed(5), 2), rev_t]).float()
    return z, t


@pytest.mark.parametrize("kind", ["mixed", "valid", "invalid"])
def test_reference_matches_torchvision_and_autograd(kind):
    z, t = boxes_case(200, 1, kind)
    r = G.refcoco(z, t, 200)
    loss, dz, giou, valid = G.refcoco_autograd(z, t, 200)
    assert torch.equal(valid, r["valid"])
    assert (r["giou"] - giou).abs().max() <= 1e-12
    assert torch.allclose(r["dlogits"], dz, rtol=1e-10, atol=1e-15)
    if kind == "invalid":
        assert r["n_valid"] == 0 and torch.isnan(loss) and torch.isnan(r["loss"])
        assert torch.isfinite(dz).all()
    else:
        assert abs(r["loss"].item() - loss.item()) <= 1e-12 * abs(loss.item())


def test_reference_tie_gradient_is_torchs():
    """At p_j == t_j the L1 gradient is 0 and max / min split theirs in half, as torch's autograd does."""
    t = torch.tensor([[0.25, 0.25, 0.75, 0.75]])
    z = torch.log(t / (1 - t)).float()
    z[0, 1] = -0.2                                 # only column 1 off its target
    t = torch.sigmoid(z.double()).float().clone()
    t[0, 1] = 0.1
    r = G.refcoco(z, t, 1)
    _, dz, _, _ = G.refcoco_autograd(z, t, 1)
    assert torch.allclose(r["dlogits"], dz, rtol=1e-10, atol=1e-15)


@pytest.mark.parametrize("kind", ["mixed", "valid", "invalid"])
@pytest.mark.parametrize("B", [1, 4, 37, 300])
def test_fp32_emulation_within_bounds(B, kind):
    z, t = boxes_case(B, 100 + B, kind)
    r = G.refcoco(z, t, B)
    p, valid, giou, loss, dz = G.emulate(z, t, B)
    keep = ~r["unsure"]
    assert torch.equal(valid[keep], r["valid"][keep])
    assert G.excess(p, r["p"], r["b_p"]) <= 1.0
    assert G.excess(giou, r["giou"], r["b_giou"]) <= 1.0
    assert G.excess(dz, r["dlogits"], r["b_dlogits"]) <= 1.0
    if r["n_valid"]:
        assert G.excess(loss, r["loss"], r["b_loss"]) <= 1.0
    else:
        assert torch.isnan(loss)


@pytest.mark.parametrize("mistake", ["nvalid_as_B", "valid_le", "no_sigmoid_grad", "unclamped_enclosing", "l1_sign",
                                     "invalid_giou_grad"])
def test_planted_mistakes_exceed_a_bound(mistake):
    z, t = planted_case()
    B = z.shape[0]
    r = G.refcoco(z, t, B)
    assert 0 < r["n_valid"] < B
    p, valid, giou, loss, dz = G.emulate(z, t, B)
    clean = max(G.excess(giou, r["giou"], r["b_giou"]), G.excess(loss, r["loss"], r["b_loss"]),
                G.excess(dz, r["dlogits"], r["b_dlogits"]))
    assert clean <= 1.0
    p, valid, giou, loss, dz = G.emulate(z, t, B, mistake)
    worst = max(G.excess(giou, r["giou"], r["b_giou"]), G.excess(loss, r["loss"], r["b_loss"]),
                G.excess(dz, r["dlogits"], r["b_dlogits"]))
    assert worst > 100.0, (mistake, worst)


def test_iou_hits_restatement_matches_golden(golden_dir):
    io = _gold(golden_dir)["iou_acc"]
    hyps, refs = sg.iou_boxes()
    assert torch.equal(hyps, io["hyps"]) and torch.equal(refs, io["refs"])
    hits = G.iou_hits(hyps, refs).to(torch.int32)
    assert torch.equal(hits, io["row_hit"])
    assert int(hits.sum()) == int(io["merged"]["score_sum"])
    # the constructed cases: exactly 0.5 is a hit; one ulp of the reference box wider mostly is not (the fp32 areas round
    # some of them back to 0.5, which is what the reference counts)
    n = hyps.shape[0]
    assert hits[n - 128:n - 64].all() and hits[n - 32:].all() and int(hits[n - 64:n - 32].sum()) < 16


def _ref_adapter(rel_bucket=24, bucket=16):
    from types import SimpleNamespace
    from one_peace_b200.adapter.image import ImageAdapter
    cfg = SimpleNamespace(vision_encoder_type="hmlp", layernorm_embedding=False, add_type_embedding=False, shrink_alpha=1.0,
                          bucket_size=bucket, use_attn_bias=True, rel_bucket_size=rel_bucket)
    return ImageAdapter(cfg, sg.GROUNDING_TINY["embed_dim"], sg.GROUNDING_TINY["heads"], num_layers=sg.GROUNDING_TINY["layers"])


def test_image_table_upgrade_matches_reference(golden_dir):
    gold = _gold(golden_dir)["upgrade"]
    sd = sg.small_table_state_dict()
    p = "encoder_wrapper.image_adapter."
    up = {k: v.clone() for k, v in sd.items() if k.startswith(p)}
    assert up[p + "rel_pos_table_list.0.weight"].shape[0] == 27 ** 2 + 3
    ad = _ref_adapter()
    ad.upgrade_state_dict_named(up, p[:-1])
    got = up[p + "rel_pos_table_list.0.weight"]
    assert got.shape == gold["rel_pos_table"].shape == (47 ** 2 + 3, sg.GROUNDING_TINY["heads"])
    assert torch.allclose(got, gold["rel_pos_table"], rtol=1e-6, atol=1e-6)
    assert torch.equal(got[-3:], sd[p + "rel_pos_table_list.0.weight"][-3:])
    assert torch.allclose(up[p + "pos_embed"], gold["pos_embed"], rtol=1e-6, atol=1e-7)
    assert torch.equal(up[p + "rp_bucket"], ad.rp_bucket) and torch.equal(up[p + "position_idx"], ad.position_idx)
    ad.load_state_dict({k[len(p):]: v for k, v in up.items() if k[len(p):] in ad.state_dict()}, strict=False)


def test_classify_model_upgrade_resizes_then_copies(golden_dir):
    from one_peace_b200.one_peace.one_peace_classify import OnePeaceClassifyConfig, OnePeaceClassifyModel
    from one_peace_b200.one_peace.hub_interface import _Dictionary
    from one_peace_b200.unify_model_config import one_peace_4b_encoder_config
    gold = _gold(golden_dir)["upgrade"]
    T = sg.GROUNDING_TINY
    cfg = OnePeaceClassifyConfig(attn_pooling=True, head_scale_ratio=sg.HEAD_SCALE_RATIO, use_image_features=True)
    cfg.encoder = one_peace_4b_encoder_config(T["layers"], T["embed_dim"], T["ffn"], T["heads"], sg.PATCH)
    m = OnePeaceClassifyModel(cfg, _Dictionary(), "vl", 4)
    sd = sg.small_table_state_dict()
    m.upgrade_state_dict_named(sd, "")
    m.load_state_dict(sd, strict=True)
    ad = m.encoder_wrapper.image_adapter
    for t in ad.rel_pos_table_list:
        assert torch.allclose(t.weight.detach(), gold["rel_pos_table"], rtol=1e-6, atol=1e-6)
    assert torch.allclose(gold["rel_pos_table_last"], gold["rel_pos_table"])
    assert torch.allclose(ad.pos_embed.detach(), gold["pos_embed"], rtol=1e-6, atol=1e-7)


def test_parameter_order_matches_reference(golden_dir):
    from one_peace_b200.one_peace.one_peace_classify import OnePeaceClassifyConfig, OnePeaceClassifyModel
    from one_peace_b200.one_peace.hub_interface import _Dictionary
    from one_peace_b200.unify_model_config import one_peace_4b_encoder_config
    rec = _gold(golden_dir)["cases"]["boxes"]
    T = sg.GROUNDING_TINY
    cfg = OnePeaceClassifyConfig(attn_pooling=True, head_scale_ratio=sg.HEAD_SCALE_RATIO, use_image_features=True)
    cfg.encoder = one_peace_4b_encoder_config(T["layers"], T["embed_dim"], T["ffn"], T["heads"], sg.PATCH)
    m = OnePeaceClassifyModel(cfg, _Dictionary(), "vl", 4)
    assert [n for n, _ in m.named_parameters()] == rec["param_order"]


def test_registry_and_protocol():
    from one_peace_b200.criterions import RefCOCOCriterion
    from one_peace_b200.criterions.refcoco_loss import RefCOCOCriterionConfig
    from one_peace_b200.metrics import IouAcc
    from one_peace_b200 import fairseq_compat as fc
    assert RefCOCOCriterion.logging_outputs_can_be_summed() is True
    assert [f for f in RefCOCOCriterionConfig.__dataclass_fields__ if f != "_name"] == []
    reg = getattr(fc, "REGISTRY", None)
    if reg is not None:
        assert reg["refcoco_criterion"] is RefCOCOCriterion
    for name in ("initialize", "compute", "merge_results"):
        assert callable(getattr(IouAcc, name))
    logged = []
    orig = fc.metrics.log_scalar
    fc.metrics.log_scalar = lambda k, v, *a, **kw: logged.append((k, v))
    try:
        RefCOCOCriterion.reduce_metrics([{"loss": 3.0, "nsentences": 4, "sample_size": 1},
                                         {"loss": 1.0, "nsentences": 3, "sample_size": 1}])
    finally:
        fc.metrics.log_scalar = orig
    assert logged == [("loss", 2.0), ("nsentences", 7), ("sample_size", 2)]
