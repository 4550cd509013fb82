"""TEST INFRASTRUCTURE.  Seeded cases of the detection-backbone fixture (oracle/make_golden_det.py -> tests/golden/det.pt)
and the synthetic weights the GPU tests and scripts/bench_det.py load: every parameter non-zero, so the relative-position
table, rel_pos_h / rel_pos_w and LayerScale all move the output."""
import torch

DET_TINY = dict(attention_heads=4, embed_dim=256, ffn_embed_dim=1024, layers=4, dropout=0.0, drop_path_rate=0.0,
                rp_bias=False, use_decomposed_rel_pos=True, shared_rp_bias=True)
# name -> (bucket_size, window_size, pretrain_bucket_size, window_block_indexes)
DET_CASES = {
    "win4": (8, 4, 4, (0, 1, 2)),
    "win4_pretrain2": (8, 4, 2, (0, 1, 2)),
    "global_only": (8, 4, 4, ()),
}
BATCH = 2

PRODUCTION = dict(attention_heads=24, bucket_size=80, pretrain_bucket_size=16, dropout=0.0, drop_path_rate=0.6,
                  embed_dim=1536, ffn_embed_dim=6144, layers=40, out_feature="last_feat", rp_bias=False,
                  use_decomposed_rel_pos=True, shared_rp_bias=True, use_checkpoint=True, window_size=16,
                  window_block_indexes=tuple(i for i in range(40) if i % 4 != 3))


def det_state_dict(shapes, buffers, seed=1, device="cpu"):
    """shapes: {name: shape} of the parameters; buffers: {name: tensor} copied as they are."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for name, shape in shapes.items():
        r = torch.randn(*shape, generator=g, device=device)
        if name.endswith("gamma_1") or name.endswith("gamma_2"):
            v = 0.3 + 0.1 * r
        elif "layer_norm" in name or name.endswith(".ln.weight") or ".image_ffn.2." in name:
            v = (1.0 + 0.1 * r) if name.endswith("weight") else 0.05 * r
        elif name.endswith("rel_pos_table.weight"):
            v = 0.5 * r
        elif "rel_pos_h" in name or "rel_pos_w" in name:
            v = 0.1 * r
        elif name.endswith("pos_embed"):
            v = 0.02 * r
        elif name.endswith("bias"):
            v = 0.02 * r
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            v = r * fan_in ** -0.5
        sd[name] = v.float()
    sd.update({k: b.clone() for k, b in buffers.items()})
    return sd


def det_images(bucket, batch=BATCH, seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, 3, 16 * bucket, 16 * bucket, generator=g)
