"""TEST INFRASTRUCTURE.  Seeded head parameters and samples of one_peace_classify (one_peace_classify.py with the
attention-pooling head, classify_loss.py / hinge_loss.py), shared by the golden-vector generator
(oracle/make_golden_classify.py) and the classification tests.  Encoder weights and raw inputs come from
oracle/synth.py; everything is drawn from seeded CPU generators in a fixed order."""
import torch

from synth import _tn, make_state_dict, tiny_inputs

CLASSIFY_TINY = dict(embed_dim=256, ffn=1024, layers=2, heads=4)

# name -> (head_type, num_classes, criterion, options); criterion: ("hard", eps) | ("multi",) | ("soft",) | ("hinge", choices)
# | None (forward only)
CLASSIFY_CASES = {
    "audio_hard": ("audio", 7, ("hard", 0.1), {}),
    "audio_multi": ("audio", 5, ("multi",), {}),
    "vl_pooler_multi": ("vl", 11, ("multi",), dict(use_pooler=True)),
    "vl_two_images": ("vl", 2, ("hard", 0.0), dict(use_two_images=True)),
    "al_hinge": ("al", 1, ("hinge", 4), {}),
    "text_soft": ("text", 6, ("soft",), {}),
    "image_peaky": ("image", 5, ("hard", 0.0), dict(q_std=1.0)),
    "vl_image_features": ("vl", 3, None, dict(use_image_features=True)),
}


def make_classify_head_state_dict(embed_dim, heads, num_classes, use_pooler=False, use_two_images=False, head_scale_ratio=1,
                                  q_std=0.02, seed=0):
    """classify_head.* of OnePeaceClassifyHead with attention pooling, in the reference's registration order."""
    g = torch.Generator().manual_seed(1000 + seed)
    d = embed_dim
    sd = {}

    def lin(prefix, out_f, in_f, bias=True, std=0.05):
        sd[prefix + "weight"] = _tn(g, (out_f, in_f), std)
        if bias:
            sd[prefix + "bias"] = 0.1 * torch.randn(out_f, generator=g)

    def ln(prefix, n):
        sd[prefix + "weight"] = 1.0 + 0.2 * torch.randn(n, generator=g)
        sd[prefix + "bias"] = 0.1 * torch.randn(n, generator=g)
    h = "classify_head."
    ln(h + "norm.", d)
    lin(h + "attn_pooling_func.k_proj.", d, d, bias=False)
    lin(h + "attn_pooling_func.v_proj.", d, d)
    lin(h + "attn_pooling_func.out_proj.", d, d)
    sd[h + "attn_pooling_func.q"] = _tn(g, (1, 1, heads, d // heads), q_std) if q_std <= 0.02 else \
        q_std * torch.randn(1, 1, heads, d // heads, generator=g)
    if use_pooler:
        lin(h + "pooler.1.", d, d)
    inner = int(d * head_scale_ratio)
    lin(h + "classifier.0.", inner, 2 * d if use_two_images else d)
    ln(h + "classifier.1.", inner)
    lin(h + "classifier.3.", num_classes, inner)
    return sd


def classify_case(name, seed=0):
    """-> (case dict, state dict of the whole model, sample) for one CLASSIFY_CASES entry; the sample is what the criterion
    receives (net_input, target, nsentences)."""
    head_type, n_cls, crit, opts = CLASSIFY_CASES[name]
    mods = {"text": ("text",), "image": ("image",), "audio": ("audio",), "vl": ("text", "image"), "al": ("text", "audio")}[head_type]
    sd = make_state_dict(**CLASSIFY_TINY, modalities=mods, seed=seed)
    sd.pop("logit_scale")
    for m in mods:
        sd.pop(f"{m}_proj.weight")
        sd.pop(f"{m}_proj.bias")
    sd.update(make_classify_head_state_dict(CLASSIFY_TINY["embed_dim"], CLASSIFY_TINY["heads"], n_cls,
                                            use_pooler=opts.get("use_pooler", False), use_two_images=opts.get("use_two_images", False),
                                            q_std=opts.get("q_std", 0.02), seed=seed))
    g = torch.Generator().manual_seed(2000 + seed)
    tok, img, aud, apm = tiny_inputs(seed=seed + 7, n_text=8, n_img=2, n_audio=2)
    B = 2
    ni = {}
    if head_type in ("text", "vl", "al"):
        ni["src_tokens"] = tok[:8] if head_type == "al" else (tok[:4] if head_type == "text" else tok[:B])
    if head_type in ("image", "vl"):
        ni["src_images"] = img
        if opts.get("use_two_images"):
            ni["src_images_2"] = torch.randn(img.shape, generator=g)
    if head_type in ("audio", "al"):
        ni["src_audios"], ni["audio_padding_masks"] = aud, apm
    rows = ni["src_tokens"].shape[0] if head_type == "text" else B
    target = None
    if crit is not None:
        if crit[0] == "hard":
            target = torch.randint(0, n_cls, (rows,), generator=g)
        elif crit[0] == "multi":
            target = (torch.rand(rows, n_cls, generator=g) < 0.3).float()
            target[:, 0] = 1.0
        elif crit[0] == "soft":
            target = torch.softmax(2.0 * torch.randn(rows, n_cls, generator=g), dim=1)
        else:
            target = torch.randint(0, crit[1], (B,), generator=g)
    sample = {"net_input": ni, "target": target, "nsentences": rows}
    case = dict(name=name, head_type=head_type, num_classes=n_cls, criterion=crit, use_pooler=opts.get("use_pooler", False),
                use_two_images=opts.get("use_two_images", False), use_image_features=opts.get("use_image_features", False))
    return case, sd, sample
