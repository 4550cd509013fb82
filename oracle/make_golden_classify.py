"""TEST INFRASTRUCTURE.  Generates tests/golden/classify.pt by executing the reference's OWN model and criterion files
(one_peace_classify.py, one_peace_base.py:132-235, classify_loss.py, hinge_loss.py; via oracle/ref_stub.py) on the seeded
cases of oracle/synth_classify.py.  It needs the reference source tree:

    python oracle/make_golden_classify.py

Tiny config (2 layers, d=256, ffn=1024, 4 heads).  The fixture is committed; the tests read only the fixture.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402
import synth  # noqa: E402
import synth_classify as sc  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def build_reference_classify(embed_dim=256, ffn=1024, layers=2, heads=4, head_type="audio", num_classes=2, use_pooler=False,
                             use_two_images=False, use_image_features=False, patch_image_size=224, text_bucket=256,
                             image_bucket=16, audio_bucket=512, seed=0, vocab=50264):
    """Instantiate the reference OnePeaceClassifyModel with the attention-pooling head of the fine-tuning recipes (4B encoder
    flags, drop-path 0 so that the forward is deterministic)."""
    ref_stub.install()
    ref_stub.ref_module("one_peace.models.components").has_flash = False
    ref_stub.ref_module("one_peace.models.transformer.multihead_attention").has_xformers = False
    cls_mod = ref_stub.ref_module("one_peace.models.one_peace.one_peace_classify")
    cfg = cls_mod.OnePeaceClassifyConfig()
    cfg.attn_pooling, cfg.use_pooler, cfg.use_image_features = True, use_pooler, use_image_features
    enc = cfg.encoder
    enc.embed_dim, enc.ffn_embed_dim, enc.layers, enc.attention_heads = embed_dim, ffn, layers, heads
    enc.normalize_before, enc.learned_pos = True, True
    enc.drop_path_rate = 0.0
    enc.dropout = enc.attention_dropout = enc.activation_dropout = 0.0
    enc.magneto_scale_attn, enc.scale_attn, enc.scale_fc, enc.scale_heads = True, False, True, False
    enc.use_layer_scale, enc.layer_scale_init_value = True, 1e-6
    enc.checkpoint_activations = False
    enc.text_adapter.bucket_size, enc.text_adapter.use_attn_bias = text_bucket, True
    enc.image_adapter.bucket_size, enc.image_adapter.use_attn_bias = image_bucket, True
    enc.image_adapter.rel_bucket_size = patch_image_size // 16
    enc.image_adapter.vision_encoder_type = "hmlp"
    enc.audio_adapter.bucket_size, enc.audio_adapter.use_attn_bias = audio_bucket, True
    torch.manual_seed(seed)
    model = cls_mod.OnePeaceClassifyModel(cfg, ref_stub._Dictionary(vocab), head_type, num_classes=num_classes,
                                          use_two_images=use_two_images)
    model.eval()
    return model


def classify():
    """tests/golden/classify.pt: one_peace_classify with the attention-pooling head through the reference's own model and
    criterion files (one_peace_classify.py, one_peace_base.py:132-235, classify_loss.py, hinge_loss.py) on the seeded cases of
    synth_classify.CLASSIFY_CASES: logits, loss, logging output and every parameter's grad_summary, the reference's parameter order, and
    the key set upgrade_state_dict_named leaves of a full 'val'-style state dict."""
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    closs = ref_stub.ref_module("one_peace.criterions.classify_loss")
    hloss = ref_stub.ref_module("one_peace.criterions.hinge_loss")
    full = synth.make_state_dict(**sc.CLASSIFY_TINY, seed=0)
    out = {"config": sc.CLASSIFY_TINY, "cases": {}}
    for name in sc.CLASSIFY_CASES:
        case, sd, sample = sc.classify_case(name)
        m = build_reference_classify(**sc.CLASSIFY_TINY, head_type=case["head_type"], num_classes=case["num_classes"],
                                              use_pooler=case["use_pooler"], use_two_images=case["use_two_images"],
                                              use_image_features=case["use_image_features"])
        sd = dict(sd)
        for mod in ("text", "image", "audio"):                     # per-layer relative-position tables (adapter/text.py:166-185)
            ad = getattr(m.encoder_wrapper, f"{mod}_adapter", None)
            if ad is not None:
                ad.upgrade_state_dict_named(sd, f"encoder_wrapper.{mod}_adapter")
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not unexpected and all(k.endswith(("rp_bucket", "position_idx", "version")) for k in missing), (missing, unexpected)
        up = {k: v.clone() for k, v in full.items()}
        m.upgrade_state_dict_named(up, "")
        rec = dict(case=case, param_order=[n for n, _ in m.named_parameters()], upgraded_keys=sorted(up))
        crit = case["criterion"]
        if crit is None:
            with torch.no_grad():
                rec["logits"] = m(**sample["net_input"]).detach()
        else:
            for q in m.parameters():
                q.requires_grad_(True)
            m.zero_grad(set_to_none=True)
            if crit[0] == "hinge":
                c = hloss.HingeLoss(task=None, margin=1.0, num_choices=crit[1])
                ni = sample["net_input"]
                with torch.no_grad():
                    rec["logits"] = m(src_tokens=ni["src_tokens"], src_audios=ni["src_audios"].repeat_interleave(crit[1], 0),
                                      audio_padding_masks=ni["audio_padding_masks"].repeat_interleave(crit[1], 0)).detach()
            else:
                c = closs.ClassifyCriterion(task=None, use_multi_label=crit[0] == "multi",
                                            label_smoothing=crit[1] if crit[0] == "hard" else 0.0)
                with torch.no_grad():
                    rec["logits"] = m(**sample["net_input"]).detach()
            loss, _, log = c(m, sample)
            loss.backward()
            rec["loss"] = loss.detach().clone()
            rec["log"] = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in log.items()}
            rec["grads"] = {n: synth.grad_summary(n, q.grad) for n, q in m.named_parameters() if q.grad is not None}
        out["cases"][name] = rec
        print(name, rec.get("loss"))
    torch.save(out, os.path.join(OUT, "classify.pt"))
    print("classify.pt", os.path.getsize(os.path.join(OUT, "classify.pt")))


if __name__ == "__main__":
    classify()
