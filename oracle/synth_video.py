"""TEST INFRASTRUCTURE.  Seeded cases of the video-backbone fixture (oracle/make_golden_video.py -> tests/golden/video.pt)
and the synthetic weights the GPU tests and scripts/bench_video.py load: every parameter non-zero, the adapters' D_fc2
included (the reference zero-initialises them, and a fixture built that way could not see the adapters)."""
import torch

VIDEO_TINY = dict(attention_heads=2, embed_dim=128, ffn_embed_dim=512, layers=2, bucket_size=4, dropout=0.0,
                  drop_path_rate=0.0, adapter_scale=0.5, rp_bias=False, shared_rp_bias=True)
# name -> (num_frames, clips)
VIDEO_CASES = {"t4_b2": (4, 2), "t16_b1": (16, 1)}

PRODUCTION = dict(attention_heads=24, bucket_size=16, num_frames=16, dropout=0.0, drop_path_rate=0.4, embed_dim=1536,
                  ffn_embed_dim=6144, layers=40, adapter_scale=0.5, rp_bias=False, shared_rp_bias=True,
                  use_checkpoint=False)


def video_state_dict(shapes, buffers, seed=1, device="cpu"):
    """shapes: {name: shape} of the parameters; buffers: {name: tensor} copied as they are."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for name, shape in shapes.items():
        r = torch.randn(*shape, generator=g, device=device)
        if name.endswith("gamma_1") or name.endswith("gamma_2"):
            v = 0.3 + 0.1 * r
        elif "layer_norm" in name or name.endswith(".ln.weight") or name.endswith(".ln.bias") or ".image_ffn.2." in name:
            v = (1.0 + 0.1 * r) if name.endswith("weight") else 0.05 * r
        elif name.endswith("rel_pos_table.weight"):
            v = 0.5 * r
        elif name.endswith("pos_embed") or name.endswith("temporal_embedding"):
            v = 0.1 * r
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


def video_clips(num_frames, clips, bucket, seed=2, device="cpu"):
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(clips, 3, num_frames, 16 * bucket, 16 * bucket, generator=g, device=device)
