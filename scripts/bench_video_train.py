"""Fine-tuning step of the Kinetics-400 video backbone (one_peace_b200.vision.video.OnePeaceViT in train mode) on one GPU:
40 layers, d = 1536, synthetic non-zero weights and adapters (oracle/synth_video.py), drop_path_rate 0.4, 2 clips at
T = 16 (the recipe's per-GPU batch) and at T = 32.  One step is forward + backward of sum(out * cotangent).

The baseline is a torch eager bf16 autograd restatement (tests/video_train_ref.py with SDPA, the bias passed as a float
mask, the same drop-path draw) with per-layer checkpointing, alternated with ours in the same process.  Also the
temporal-attention backward kernel alone at B = 2, T = 16 against its HBM floor (it reads qkv, out and d_out and writes
dqkv: 8 D bf16 per row).

    python scripts/bench_video_train.py [--layers 40] [--iters 3] [--out DIR]

Prints one JSON line per measurement, and the card name and power limit read in the same process.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench_video as BV  # noqa: E402
import restated_video as RV  # noqa: E402
import synth_video as sv  # noqa: E402
import video_train_ref as VT  # noqa: E402
from one_peace_b200 import kernels as K  # noqa: E402
from one_peace_b200.vision.video import OnePeaceViT  # noqa: E402


def bench_temporal_bwd(rounds=5, iters=50):
    Bv, T, N, H = 2, 16, 257, 24
    D, M = H * 64, Bv * T * N
    qkv = (torch.randn(M, 3 * D, device="cuda") * 0.5).to(torch.bfloat16)
    out, _ = K.attention_temporal(qkv, Bv, T, N, H)
    dout = torch.randn(M, D, device="cuda").to(torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    run = lambda: K.attention_temporal_bwd(qkv, out, dout, Bv, T, N, H, 0.125, dqkv=dqkv)
    run()
    ts = [BV.timed(run, iters) for _ in range(rounds)]
    moved = 8 * D * 2 * M
    floor_us = 1e6 * moved / BV.HBM_BYTES_PER_S
    us = 1e3 * min(ts)
    return dict(what="temporal_attention_bwd", Bv=Bv, T=T, N=N, H=H, kernel_us=round(us, 2),
                kernel_us_spread=[round(1e3 * v, 2) for v in (min(ts), max(ts))], bytes=moved,
                hbm_floor_us=round(floor_us, 2), floor_fraction=round(floor_us / us, 3))


def bench_step(T, clips, layers, iters):
    P = dict(sv.PRODUCTION, num_frames=T, layers=layers, drop_path_rate=0.4)
    with torch.device("meta"):
        meta = OnePeaceViT(**P)
    shapes = {k: tuple(p.shape) for k, p in meta.named_parameters()}
    del meta
    m = OnePeaceViT(**P)
    sd = sv.video_state_dict(shapes, {k: b.cuda() for k, b in m.named_buffers()}, device="cuda")
    m = m.cuda()
    m.load_state_dict(sd, strict=True)
    m.train()
    sd16 = {k: (v.to(torch.bfloat16).requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    del sd
    x = sv.video_clips(T, clips, P["bucket_size"], device="cuda")
    x16 = x.to(torch.bfloat16)
    cot = torch.randn(clips, P["embed_dim"], T, 1, 1, device="cuda")
    probs = [layer.drop_path_prob for layer in m.encoder.layers]
    dev = torch.device("cuda", torch.cuda.current_device())
    RV._attn = BV._attn_sdpa

    def ours():
        for p in m.parameters():
            p.grad = None
        (m(x) * cot).sum().backward()

    def eager():
        for v in sd16.values():
            if torch.is_tensor(v) and v.requires_grad:
                v.grad = None
        masks = VT.row_scales(probs, clips * T, torch.cuda.get_rng_state(dev), dev)
        masks = [tuple(None if r is None else r.to(torch.bfloat16) for r in trip) for trip in masks]
        y = VT.forward(sd16, x16, P["attention_heads"], layers, P["adapter_scale"], masks=masks, checkpoint=True)
        (y.float() * cot).sum().backward()

    N = P["bucket_size"] ** 2 + 1
    ours()
    eager()
    t_ours, t_eager = [], []
    for _ in range(3):
        t_ours.append(BV.timed(ours, iters))
        t_eager.append(BV.timed(eager, iters))
    policy = m.encoder.activations                 # what the timed steps' VideoStackFn chose
    fl = 3 * BV.encoder_flops(clips, T, N, P["embed_dim"], P["ffn_embed_dim"], P["attention_heads"], layers)
    ms, ms_e = min(t_ours), min(t_eager)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del m, sd16
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return dict(what="backbone_train_step", T=T, clips=clips, layers=layers, drop_path_rate=0.4,
                activations=policy, ms_per_step=round(ms, 2),
                ms_spread=[round(v, 2) for v in (min(t_ours), max(t_ours))],
                encoder_tflops_3x_fwd=round(fl / ms * 1e-9, 1), eager_bf16_sdpa_checkpointed_ms=round(ms_e, 2),
                eager_ms_spread=[round(v, 2) for v in (min(t_eager), max(t_eager))], speedup_vs_eager=round(ms_e / ms, 2),
                peak_gib=round(peak, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_video_train.py measures on the GPU"
    res = [dict(what="card", card=BV.card())]
    print(json.dumps(res[-1]), flush=True)
    res.append(bench_temporal_bwd())
    print(json.dumps(res[-1]), flush=True)
    for T, clips in ((16, 2), (32, 2)):
        res.append(bench_step(T, clips, a.layers, a.iters))
        print(json.dumps(res[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_video_train.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
