"""TEST INFRASTRUCTURE.  Seeded weights, samples and boxes of the visual-grounding path (one_peace_classify with head_type vl,
4 outputs and attention pooling at patch_image_size 384, criterions/refcoco_loss.py, metrics/iou_acc.py), shared by the
golden-vector generator (oracle/make_golden_grounding.py) and the grounding tests.  Everything is drawn from seeded CPU
generators in a fixed order."""
import torch

from synth import make_state_dict, tiny_inputs
from synth_classify import CLASSIFY_TINY, make_classify_head_state_dict

GROUNDING_TINY = CLASSIFY_TINY
PATCH = 384                      # the RefCOCO recipe's patch_image_size: rel_bucket_size 24, 577 image tokens
HEAD_SCALE_RATIO = 2
TEXT_LEN = 20

# name -> bias of the 4 box logits: "boxes" makes every row valid (p0 < p2 and p1 < p3); "mixed" puts the y-validity
# threshold between the rows (three of the four stay valid, every row at least 0.07 from the threshold in logit);
# "all_invalid" turns every row around so the loss is NaN and only the L1 gradient flows
GROUNDING_CASES = {
    "boxes": (-0.6, -0.6, 0.6, 0.6),
    "mixed": (-0.6, 0.34, 0.6, 0.0),
    "all_invalid": (1.5, 1.5, -1.5, -1.5),
}


def random_boxes(g, n):
    """n target boxes (x0, y0, x1, y1) in [0, 1] with x0 < x1 and y0 < y1."""
    lo = 0.6 * torch.rand(n, 2, generator=g)
    hi = lo + 0.05 + (1.0 - lo - 0.05) * torch.rand(n, 2, generator=g)
    return torch.cat([lo, hi], 1)


def grounding_case(name, seed=0, B=4):
    """-> (case dict, state dict of the whole model, sample) for one GROUNDING_CASES entry."""
    sd = make_state_dict(**GROUNDING_TINY, modalities=("text", "image"), image_rel_bucket=PATCH // 16, seed=seed)
    sd.pop("logit_scale")
    for m in ("text", "image"):
        sd.pop(f"{m}_proj.weight")
        sd.pop(f"{m}_proj.bias")
    sd.update(make_classify_head_state_dict(GROUNDING_TINY["embed_dim"], GROUNDING_TINY["heads"], 4,
                                            head_scale_ratio=HEAD_SCALE_RATIO, seed=seed))
    sd["classify_head.classifier.3.bias"] = torch.tensor(GROUNDING_CASES[name], dtype=torch.float32)
    tok, img, _, _ = tiny_inputs(seed=seed + 11, n_text=B, text_len=TEXT_LEN, n_img=B, res=PATCH, n_audio=1)
    g = torch.Generator().manual_seed(3000 + seed)
    sample = {"net_input": {"src_tokens": tok, "src_images": img}, "target": random_boxes(g, B), "nsentences": B}
    case = dict(name=name, head_type="vl", num_classes=4, use_pooler=False, use_two_images=False, use_image_features=True,
                head_scale_ratio=HEAD_SCALE_RATIO, patch_image_size=PATCH)
    return case, sd, sample


def small_table_state_dict(seed=5):
    """A text + image state dict whose image tables come from a 224^2 / 14-bucket model: 27^2 + 3 relative-position rows and a
    14^2 + 1 row pos_embed, for loading into the 384^2 model (24 buckets, pos_embed bucket 16)."""
    sd = make_state_dict(**GROUNDING_TINY, modalities=("text", "image"), image_rel_bucket=14, image_bucket=14, seed=seed)
    sd.pop("logit_scale")
    return sd


def iou_boxes(seed=0):
    """(hyps, refs) fp32 [n, 4] covering overlapping, disjoint, nested and degenerate pairs, pairs with two negative extents
    whose product is a positive area, and pairs constructed to have iou == 0.5 exactly (dyadic coordinates)."""
    g = torch.Generator().manual_seed(4000 + seed)
    rows = []
    # overlapping / disjoint / nested: random boxes and jittered copies
    a = random_boxes(g, 96)
    b = a + 0.25 * (torch.rand(96, 4, generator=g) - 0.5)
    rows.append((a, b))
    far = random_boxes(g, 32)
    rows.append((far, far + torch.tensor([2.0, 2.0, 2.0, 2.0])))                  # disjoint
    inner = a[:32].clone()
    c = (inner[:, :2] + inner[:, 2:]) / 2
    half = (inner[:, 2:] - inner[:, :2]) / 4
    rows.append((inner, torch.cat([c - half, c + half], 1)))                     # nested
    # degenerate: zero width / height, reversed corners, both extents negative
    d = random_boxes(g, 16)
    zw = d.clone()
    zw[:, 2] = zw[:, 0]
    rows.append((zw, d))
    rev = d[:, [2, 3, 0, 1]].contiguous()
    rows.append((rev, rev.clone()))
    rows.append((rev, d))
    # iou == 0.5 exactly: [0, 0, w, h] against [0, 0, 2w, h] (area_i = wh, union = 2wh), and scaled / shifted dyadic variants
    k = torch.arange(1, 33, dtype=torch.float32)
    w = k / 64.0
    h = (33 - k) / 32.0
    x0 = (k % 5) / 8.0
    y0 = (k % 3) / 16.0
    hp = torch.stack([x0, y0, x0 + w, y0 + h], 1)
    rp = torch.stack([x0, y0, x0 + 2 * w, y0 + h], 1)
    rows.append((hp, rp))
    rows.append((rp, hp))
    # just above / below 0.5 by one ulp of the reference's box
    up = rp.clone()
    up[:, 2] = torch.nextafter(up[:, 2], torch.full_like(up[:, 2], 10.0))
    rows.append((hp, up))
    dn = rp.clone()
    dn[:, 2] = torch.nextafter(dn[:, 2], torch.zeros_like(dn[:, 2]))
    rows.append((hp, dn))
    hyps = torch.cat([r[0] for r in rows]).float().contiguous()
    refs = torch.cat([r[1] for r in rows]).float().contiguous()
    return hyps, refs
