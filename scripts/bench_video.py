"""Evaluation throughput of the Kinetics-400 video backbone (one_peace_b200.vision.video.OnePeaceViT) on one GPU, with
synthetic non-zero weights (oracle/synth_video.py), against a torch eager bf16 restatement with SDPA in the same process,
alternating the two; and the temporal-attention kernel alone at the production shape against the gather path it replaces
(row_gather of qkv into (b n) t order -> the sequence attention at S = T -> row_gather back).

    python scripts/bench_video.py [--layers 40] [--iters 5] [--out DIR]

Prints one JSON line per measurement, and the card name and power limit read in the same process.  FLOPs are derived from
shapes (encoder GEMMs + both attentions); the temporal kernel's HBM floor counts qkv in, out and records out.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import restated_video as RV  # noqa: E402
import synth_video as sv  # noqa: E402
from one_peace_b200 import kernels as K  # noqa: E402
from one_peace_b200.vision.video import OnePeaceViT  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def encoder_flops(views, T, N, d, F_, H, layers):
    M = views * T * N
    gemm = 2 * M * d * (2 * 3 * d + 2 * d + 6 * (d // 4) + 2 * F_ + F_)
    attn = 4 * views * (N * H * T * T + T * H * N * N) * 64
    return layers * (gemm + attn)


def _attn_sdpa(x, sd, p, heads, bias=None):
    B, L, d = x.shape
    hd = d // heads
    q = (RV._lin(x, sd, p + ".q_proj") * hd ** -0.5).view(B, L, heads, hd).transpose(1, 2)
    k = RV._lin(x, sd, p + ".k_proj", bias=False).view(B, L, heads, hd).transpose(1, 2)
    v = RV._lin(x, sd, p + ".v_proj").view(B, L, heads, hd).transpose(1, 2)
    mask = None if bias is None else bias.to(q.dtype).unsqueeze(0).expand(B, -1, -1, -1)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=1.0).transpose(1, 2).reshape(B, L, d)
    return RV._lin(RV._ln(o, sd, p + ".ln"), sd, p + ".out_proj")


def timed(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_temporal(rounds=5, iters=50):
    Bv, T, N, H = 4, 16, 257, 24
    D, M = H * 64, Bv * T * N
    qkv = (torch.randn(M, 3 * D, device="cuda") * 0.5).to(torch.bfloat16)
    out = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    rec = torch.empty(H, M, 2, device="cuda")
    b = torch.arange(Bv, device="cuda").view(Bv, 1, 1)
    n = torch.arange(N, device="cuda").view(1, N, 1)
    t = torch.arange(T, device="cuda").view(1, 1, T)
    idx = ((b * T + t) * N + n).reshape(-1).contiguous()
    inv = torch.empty_like(idx)
    inv[idx] = torch.arange(M, device="cuda")
    g_qkv = torch.empty_like(qkv)
    g_out = torch.empty_like(out)

    def new():
        K.attention_temporal(qkv, Bv, T, N, H, out=out, ln_stats=rec)

    def old():
        K.row_gather(qkv, idx, out=g_qkv)
        K.attention(g_qkv, None, None, Bv * N, T, H, out=g_out, ln_stats=rec)
        K.row_gather(g_out, inv, out=out)

    for f in (new, old):
        f()
    ts_new, ts_old = [], []
    for _ in range(rounds):
        ts_new.append(timed(new, iters))
        ts_old.append(timed(old, iters))
    us_new, us_old = 1e3 * min(ts_new), 1e3 * min(ts_old)
    moved = qkv.numel() * 2 + out.numel() * 2 + rec.numel() * 4
    floor_us = 1e6 * moved / HBM_BYTES_PER_S
    return dict(what="temporal_attention", Bv=Bv, T=T, N=N, H=H, kernel_us=round(us_new, 2),
                kernel_us_spread=[round(1e3 * v, 2) for v in (min(ts_new), max(ts_new))], gather_path_us=round(us_old, 2),
                gather_path_us_spread=[round(1e3 * v, 2) for v in (min(ts_old), max(ts_old))], bytes=moved,
                hbm_floor_us=round(floor_us, 2), floor_fraction=round(floor_us / us_new, 3))


def bench_backbone(T, views, layers, iters):
    P = dict(sv.PRODUCTION, num_frames=T, layers=layers)
    with torch.device("meta"):
        meta = OnePeaceViT(**P)
    shapes = {k: tuple(p.shape) for k, p in meta.named_parameters()}
    del meta
    m = OnePeaceViT(**P)
    sd = sv.video_state_dict(shapes, {k: b.cuda() for k, b in m.named_buffers()}, device="cuda")
    m = m.cuda()
    m.load_state_dict(sd, strict=True)
    m.eval().requires_grad_(False)
    sd16 = {k: (v.to(torch.bfloat16) if v.is_floating_point() else v) for k, v in sd.items()}
    del sd
    x = sv.video_clips(T, views, P["bucket_size"], device="cuda")
    x16 = x.to(torch.bfloat16)
    RV._attn = _attn_sdpa
    ours = lambda: m(x)
    eager = lambda: RV.forward(sd16, x16, P["attention_heads"], layers, P["adapter_scale"])
    with torch.no_grad():
        y, ye = ours(), eager()
        cos = F.cosine_similarity(y.flatten().double(), ye.flatten().double(), dim=0).item()
        t_ours, t_eager = [], []
        for _ in range(3):
            t_ours.append(timed(ours, iters))
            t_eager.append(timed(eager, iters))
    N = P["bucket_size"] ** 2 + 1
    fl = encoder_flops(views, T, N, P["embed_dim"], P["ffn_embed_dim"], P["attention_heads"], layers)
    ms, ms_e = min(t_ours), min(t_eager)
    del m, sd16
    torch.cuda.empty_cache()
    return dict(what="backbone_eval", T=T, views=views, layers=layers, ms_per_view=round(ms / views, 3),
                views_per_s=round(1e3 * views / ms, 3), encoder_tflops=round(fl / ms * 1e-9, 1),
                tflop_per_view=round(fl / views * 1e-12, 2), eager_bf16_sdpa_ms_per_view=round(ms_e / views, 3),
                speedup_vs_eager=round(ms_e / ms, 2), ms_spread=[round(v, 2) for v in (min(t_ours), max(t_ours))],
                cosine_vs_eager=round(cos, 6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_video.py measures on the GPU"
    res = [dict(what="card", card=card())]
    print(json.dumps(res[-1]), flush=True)
    res.append(bench_temporal())
    print(json.dumps(res[-1]), flush=True)
    for T, views in ((16, 1), (16, 4), (32, 1)):
        res.append(bench_backbone(T, views, a.layers, a.iters))
        print(json.dumps(res[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_video.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
