"""Seeded cases of the OnePeaceViT fixture (tests/golden/vit.pt, oracle/make_golden_vit.py): the tiny config, a state dict that
gives every parameter a visible effect (random relative-position table, layer scales of 0.1, a head whose logits are O(1)),
images and targets.  Shared by the fixture generator and the tests, so the fixture stores outputs only."""
import json
import zlib

import torch

VIT_TINY = dict(layers=2, embed_dim=256, ffn_embed_dim=1024, attention_heads=4)
NUM_CLASSES = 37                                   # not a multiple of 8: the head GEMM's padded rows are exercised
BATCH = 4
# name -> (bucket_size, global_pool, criterion): buckets 4 (64^2, S = 17) and 16 (256^2, S = 257), both heads, both criteria
VIT_CASES = {
    "b4_pool_soft": (4, True, "soft"),
    "b4_cls_smooth": (4, False, "smooth"),
    "b16_pool_smooth": (16, True, "smooth"),
    "b16_cls_soft": (16, False, "soft"),
}
SMOOTHING = 0.1
BIG_VARIANTS = {"one_piece_g_256": 16, "one_piece_g_384": 24, "one_piece_g_448": 28, "one_piece_g_512": 32}


def _norm_param(name):
    return any(t in name for t in ("layer_norm.", "self_attn.ln.", "image_ffn.2.", "fc_norm."))


def vit_state_dict(shapes, buffers, seed=0, device="cpu"):
    """shapes: {name: shape} of the parameters, buffers: {name: tensor} copied as they are -> fp32 state dict on `device`
    (the values depend on the device's generator: the fixture's are the CPU's)."""
    sd = {}
    for name, shape in shapes.items():
        g = torch.Generator(device=device).manual_seed(zlib.crc32(name.encode()) + seed)
        r = torch.randn(*shape, generator=g, device=device)
        if _norm_param(name):
            v = 1.0 + 0.1 * r if name.endswith("weight") else 0.05 * r
        elif "gamma_" in name:
            v = 0.1 + 0.02 * r
        elif "rel_pos_table" in name:
            v = 0.5 * r
        elif name.endswith(("cls_embedding", "pos_embed")):
            v = shape[-1] ** -0.5 * r
        elif name.endswith("bias"):
            v = 0.02 * r if not name.startswith("head.") else 0.1 * r
        else:                                       # Linear / Conv2d weights: unit-variance outputs
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            v = fan_in ** -0.5 * r
        sd[name] = v.float()
    for name, b in buffers.items():
        sd[name] = b.clone()
    return sd


def vit_inputs(bucket, seed=0):
    """images fp32 [BATCH, 3, 16 * bucket, 16 * bucket], soft targets fp32 [BATCH, NUM_CLASSES] (rows sum to 1), labels int64."""
    g = torch.Generator().manual_seed(1000 + bucket + seed)
    R = 16 * bucket
    img = torch.randn(BATCH, 3, R, R, generator=g)
    soft = torch.softmax(2.0 * torch.randn(BATCH, NUM_CLASSES, generator=g), dim=1)
    labels = torch.randint(0, NUM_CLASSES, (BATCH,), generator=g)
    return img, soft, labels


def soft_target_ce(x, target):
    """timm.loss.SoftTargetCrossEntropy: mean over rows of sum_c -target_c * log_softmax(x)_c."""
    return torch.sum(-target * torch.log_softmax(x, dim=-1), dim=-1).mean()


def label_smoothing_ce(x, target, smoothing=SMOOTHING):
    """timm.loss.LabelSmoothingCrossEntropy: mean over rows of (1 - s) * nll + s * mean_c(-log_softmax(x)_c)."""
    logprobs = torch.log_softmax(x, dim=-1)
    nll = -logprobs.gather(dim=-1, index=target.unsqueeze(1)).squeeze(1)
    return ((1.0 - smoothing) * nll + smoothing * -logprobs.mean(dim=-1)).mean()


def criterion(kind, x, soft, labels):
    return soft_target_ce(x, soft) if kind == "soft" else label_smoothing_ce(x, labels)


def big_records(fixture):
    """The fixture's 4B records, {(variant, global_pool): dict(keys=[(name, shape, dtype)], no_weight_decay, layer_ids)}."""
    recs = json.loads(zlib.decompress(fixture["big_z"]).decode())
    return {(r["variant"], r["pool"]): dict(keys=[(k, tuple(shape), dt) for k, shape, dt in r["keys"]],
                                             no_weight_decay=r["no_weight_decay"], layer_ids=r["layer_ids"]) for r in recs}
