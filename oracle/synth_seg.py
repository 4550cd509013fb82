"""TEST INFRASTRUCTURE.  Seeded cases of the segmentation-backbone fixture (oracle/make_golden_seg.py ->
tests/golden/seg.pt) and the synthetic weights the tests and scripts/bench_seg.py load.  Every parameter is non-zero and
every BatchNorm has non-trivial statistics: the reference initialises the injectors' gamma to 1e-6 and the tables to zero,
and a fixture built that way could not see the injectors or the relative-position bias."""
import torch
import torch.nn as nn

SEG_TINY = dict(conv_inplane=16, n_points=4, deform_num_heads=2, init_values=1e-6, cffn_ratio=0.25, deform_ratio=0.5,
                interaction_indexes=[[0, 0], [1, 1], [2, 2], [3, 3]], attention_heads=2, bucket_size=4, embed_dim=128,
                ffn_embed_dim=512, layers=4, drop_path_rate=0.0)
PRODUCTION = dict(conv_inplane=64, n_points=4, deform_num_heads=24, init_values=1e-6, cffn_ratio=0.25, deform_ratio=0.5,
                  interaction_indexes=[[0, 9], [10, 19], [20, 29], [30, 39]], attention_heads=24, bucket_size=56,
                  embed_dim=1536, ffn_embed_dim=6144, layers=40, drop_path_rate=0.4, rp_bias=True, shared_rp_bias=False)


def seg_state_dict(model, seed=1, device="cpu"):
    """Seeded fp32 values for every floating entry of model.state_dict(), drawn in its order; integer buffers copied."""
    g = torch.Generator(device=device).manual_seed(seed)
    kinds = {n: m for n, m in model.named_modules()}
    sd = {}
    for name, t in model.state_dict().items():
        if not t.is_floating_point():
            sd[name] = t.clone().to(device)
            continue
        r = torch.randn(*t.shape, generator=g, device=device)
        owner, leaf = (name.rsplit(".", 1) + [""])[:2] if "." in name else ("", name)
        norm = isinstance(kinds.get(owner), (nn.LayerNorm, nn.modules.batchnorm._BatchNorm))
        if norm and leaf == "weight":
            v = 1.0 + 0.1 * r
        elif norm and leaf == "running_var":
            v = 0.5 + r.abs()
        elif norm and leaf in ("bias", "running_mean"):
            v = 0.05 * r
        elif leaf in ("gamma_1", "gamma_2", "gamma"):
            v = 0.3 + 0.1 * r
        elif name.endswith("rel_pos_table.weight"):
            v = 0.5 * r
        elif leaf in ("pos_embed", "level_embed", "cls_embedding"):
            v = 0.1 * r
        elif leaf == "bias":
            v = 0.02 * r
        else:
            fan_in = 1
            for s in t.shape[1:]:
                fan_in *= s
            if isinstance(kinds.get(owner), nn.ConvTranspose2d):
                fan_in = t.shape[0] * t.shape[2] * t.shape[3]
            v = r * fan_in ** -0.5
        sd[name] = v.float()
    return sd


def seg_images(B, bucket, seed=2, device="cpu"):
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(B, 3, 16 * bucket, 16 * bucket, generator=g, device=device)
