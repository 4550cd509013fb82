"""TEST INFRASTRUCTURE.  Generates tests/golden/refcoco.pt by executing the reference's OWN files (one_peace_classify.py with
head_type vl, 4 outputs and attention pooling at patch_image_size 384; criterions/refcoco_loss.py; metrics/iou_acc.py;
models/adapter/image.py's upgrade_state_dict_named; via oracle/ref_stub.py) on the seeded cases of oracle/synth_grounding.py.
It needs the reference source tree:

    python oracle/make_golden_grounding.py

Two stand-ins are installed, and recorded in the fixture:
  * scipy.interpolate.interp2d, removed in SciPy 1.14, becomes its gridded-data equivalent: the s = 0 bicubic spline
    RectBivariateSpline(y, x, z) evaluated as f(dy, dx);
  * one_peace.utils.data_utils (imported by iou_acc.py for its distributed all_gather, which a single process never calls)
    becomes an empty module, and IouAcc runs on the CPU with initialize()'s tensors created there.
The fixture is committed; the tests read only the fixture.
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402
import synth  # noqa: E402
import synth_grounding as sg  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
INTERP2D_STANDIN = "RectBivariateSpline(y, x, z, kx=3, ky=3, s=0)(new_y, new_x) for interp2d(x, y, z, kind='cubic')(new_x, new_y)"


class _Interp2dStandin:
    def __init__(self, x, y, z, kind="cubic"):
        from scipy.interpolate import RectBivariateSpline
        assert kind == "cubic"
        self.f = RectBivariateSpline(y, x, z, kx=3, ky=3, s=0)

    def __call__(self, new_x, new_y):
        return self.f(new_y, new_x)


def _install():
    ref_stub.install()
    from scipy import interpolate
    interpolate.interp2d = _Interp2dStandin
    if "one_peace.utils" not in sys.modules:
        u = types.ModuleType("one_peace.utils")
        u.__path__ = []
        sys.modules["one_peace.utils"] = u
        sys.modules["one_peace.utils.data_utils"] = types.ModuleType("one_peace.utils.data_utils")
        sys.modules["one_peace.utils.data_utils"].all_gather = None
    if "one_peace.metrics" not in sys.modules:
        m = types.ModuleType("one_peace.metrics")
        m.__path__ = [os.path.join(ref_stub.REF_PKG, "metrics")]
        sys.modules["one_peace.metrics"] = m


def build_reference_grounding(seed=0):
    """The reference OnePeaceClassifyModel of the RefCOCO recipe (run_scripts/visual_grounding/base.yaml: head_type vl,
    num_classes 4, attn_pooling, no pooler, use_image_features, head_scale_ratio 2, patch_image_size 384) at the tiny width,
    4B encoder flags, drop-path 0 so that the forward is deterministic."""
    _install()
    ref_stub.ref_module("one_peace.models.components").has_flash = False
    ref_stub.ref_module("one_peace.models.transformer.multihead_attention").has_xformers = False
    cls_mod = ref_stub.ref_module("one_peace.models.one_peace.one_peace_classify")
    T = sg.GROUNDING_TINY
    cfg = cls_mod.OnePeaceClassifyConfig()
    cfg.attn_pooling, cfg.use_pooler, cfg.use_image_features, cfg.head_scale_ratio = True, False, True, sg.HEAD_SCALE_RATIO
    enc = cfg.encoder
    enc.embed_dim, enc.ffn_embed_dim, enc.layers, enc.attention_heads = T["embed_dim"], T["ffn"], T["layers"], T["heads"]
    enc.normalize_before, enc.learned_pos = True, True
    enc.drop_path_rate = 0.0
    enc.dropout = enc.attention_dropout = enc.activation_dropout = 0.0
    enc.magneto_scale_attn, enc.scale_attn, enc.scale_fc, enc.scale_heads = True, False, True, False
    enc.use_layer_scale, enc.layer_scale_init_value = True, 1e-6
    enc.checkpoint_activations = False
    enc.text_adapter.bucket_size, enc.text_adapter.use_attn_bias = 256, True
    enc.image_adapter.bucket_size, enc.image_adapter.use_attn_bias = 16, True
    enc.image_adapter.rel_bucket_size = sg.PATCH // 16
    enc.image_adapter.vision_encoder_type = "hmlp"
    enc.audio_adapter.bucket_size, enc.audio_adapter.use_attn_bias = 512, True
    torch.manual_seed(seed)
    model = cls_mod.OnePeaceClassifyModel(cfg, ref_stub._Dictionary(50264), "vl", num_classes=4, use_two_images=False)
    model.eval()
    return model


def _load(m, sd):
    sd = dict(sd)
    for mod in ("text", "image"):                              # per-layer tables (adapter/{text,image}.py upgrade_state_dict_named)
        getattr(m.encoder_wrapper, f"{mod}_adapter").upgrade_state_dict_named(sd, f"encoder_wrapper.{mod}_adapter")
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.endswith(("rp_bucket", "position_idx", "version")) for k in missing), (missing, unexpected)


def grounding():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    _install()
    rloss = ref_stub.ref_module("one_peace.criterions.refcoco_loss")
    out = {"config": dict(sg.GROUNDING_TINY, patch_image_size=sg.PATCH, head_scale_ratio=sg.HEAD_SCALE_RATIO),
           "interp2d_standin": INTERP2D_STANDIN, "cases": {}}
    for name in sg.GROUNDING_CASES:
        case, sd, sample = sg.grounding_case(name)
        m = build_reference_grounding()
        _load(m, sd)
        rec = dict(case=case, param_order=[n for n, _ in m.named_parameters()])
        with torch.no_grad():
            rec["logits"] = m(**sample["net_input"]).detach()
        for q in m.parameters():
            q.requires_grad_(True)
        m.zero_grad(set_to_none=True)
        loss, sample_size, log = rloss.RefCOCOCriterion(task=None)(m, sample)
        loss.backward()
        p = rec["logits"].sigmoid()
        rec["n_valid"] = int((p[:, :2] < p[:, 2:]).all(1).sum())
        rec["loss"] = loss.detach().clone()
        rec["sample_size"] = sample_size
        rec["log"] = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in log.items()}
        rec["grads"] = {n: synth.grad_summary(n, q.grad) for n, q in m.named_parameters() if q.grad is not None}
        out["cases"][name] = rec
        print(name, rec["loss"].item(), "n_valid", rec["n_valid"])

    # the image adapter's checkpoint upgrade: 224^2-sized tables into the 384^2 model
    m = build_reference_grounding()
    sd = sg.small_table_state_dict()
    ad = m.encoder_wrapper.image_adapter
    p = "encoder_wrapper.image_adapter."
    up = {k: v.clone() for k, v in sd.items() if k.startswith(p)}
    ad.upgrade_state_dict_named(up, p[:-1])
    out["upgrade"] = {"rel_pos_table": up[p + "rel_pos_table_list.0.weight"].clone(),
                      "rel_pos_table_last": up[p + f"rel_pos_table_list.{len(ad.rel_pos_table_list) - 1}.weight"].clone(),
                      "pos_embed": up[p + "pos_embed"].clone()}
    print("upgrade", tuple(out["upgrade"]["rel_pos_table"].shape), tuple(out["upgrade"]["pos_embed"].shape))

    # IouAcc on seeded boxes, per row and merged over uneven batches
    iou_mod = ref_stub.ref_module("one_peace.metrics.iou_acc")
    hyps, refs = sg.iou_boxes()

    def fresh():
        a = iou_mod.IouAcc()
        a.ids, a.hyps = torch.Tensor([]), torch.Tensor([])
        a.score_sum, a.score_cnt = torch.FloatTensor([0]), torch.IntTensor([0])
        return a
    row_hit = []
    for r in range(hyps.shape[0]):
        a = fresh()
        a.compute(torch.tensor([r]), hyps[r:r + 1], refs[r:r + 1])
        row_hit.append(int(a.score_sum.item()))
    a = fresh()
    ids = torch.arange(1000, 1000 + hyps.shape[0])
    cuts = [0, 7, 64, 65, 200, hyps.shape[0]]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        a.compute(ids[lo:hi], hyps[lo:hi], refs[lo:hi])
    merged = a.merge_results(output_predict=True)
    out["iou_acc"] = {"hyps": hyps, "refs": refs, "ids": ids, "cuts": cuts, "row_hit": torch.tensor(row_hit, dtype=torch.int32),
                      "merged": merged}
    print("iou_acc", merged["score_sum"], merged["score_cnt"], merged["iou_acc"])
    torch.save(out, os.path.join(OUT, "refcoco.pt"))
    print("refcoco.pt", os.path.getsize(os.path.join(OUT, "refcoco.pt")))


if __name__ == "__main__":
    grounding()
