"""Times OnePeaceViT (one_piece_g_*, 40 layers, d = 1536, 24 heads) on ImageNet-shaped work:

  - eval images/s at 256^2 / 384^2 / 512^2 (S = 257 / 577 / 1025), B = 64, against a torch eager bf16 restatement of the
    same forward (F.scaled_dot_product_attention with the bias as its mask), alternating the two, two rounds each;
  - one fine-tuning step at 384^2, B = 8, drop-path 0.4, soft targets, AdamW-style AdjustAdam with layer decay 0.85 (the
    1k recipe's settings);
  - the pooled-head kernels alone at B = 64, S = 1025, d = 1536 against their HBM floor (bytes / 3.35 TB/s).

Prints one JSON line (with the card's name and power limit) and writes it to --out if given.

    python scripts/bench_vit.py [--iters 3] [--warmup 2] [--layers 40] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:                     # the number is still reported, without the card line
        return f"unknown ({e})"


def time_cuda(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters          # ms


def eager_bf16_forward(P, img, heads, eps=1e-5):
    """models_vit.py's eval forward (global_pool) in torch eager bf16 on the parameters P (name -> bf16 tensor)."""
    pre = "image_adapter.embed_images."
    d = P["image_adapter.pos_embed"].shape[1]

    def ln2d(x, i):
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), P[f"{pre}{i}.layer_norm.weight"],
                            P[f"{pre}{i}.layer_norm.bias"], eps).permute(0, 3, 1, 2)
    x = F.gelu(ln2d(F.conv2d(img, P[pre + "0.weight"], P[pre + "0.bias"], stride=4), 1))
    x = F.gelu(ln2d(F.conv2d(x, P[pre + "3.weight"], P[pre + "3.bias"], stride=2), 4))
    x = F.conv2d(x, P[pre + "6.weight"], P[pre + "6.bias"], stride=2).flatten(2).transpose(1, 2)
    B = x.shape[0]
    x = torch.cat([P["image_adapter.cls_embedding"].expand(B, -1, -1), x], 1) + P["image_adapter.pos_embed"][None]
    S = x.shape[1]
    bias = F.embedding(P["image_adapter.rp_bucket"], P["image_adapter.rel_pos_table.weight"]).permute(2, 0, 1)[None]
    i = 0
    while f"encoder.layers.{i}.gamma_1" in P:
        L = lambda n: P[f"encoder.layers.{i}.{n}"]                      # noqa: E731
        h = F.layer_norm(x, (d,), L("self_attn_layer_norm.weight"), L("self_attn_layer_norm.bias"), eps)
        q = F.linear(h, L("self_attn.q_proj.weight"), L("self_attn.q_proj.bias"))
        k = F.linear(h, L("self_attn.k_proj.weight"))
        v = F.linear(h, L("self_attn.v_proj.weight"), L("self_attn.v_proj.bias"))
        q, k, v = (t.view(B, S, heads, -1).transpose(1, 2) for t in (q, k, v))
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=bias.expand(B, -1, -1, -1))
        a = F.layer_norm(a.transpose(1, 2).reshape(B, S, d), (d,), L("self_attn.ln.weight"), L("self_attn.ln.bias"), eps)
        x = x + L("gamma_1") * F.linear(a, L("self_attn.out_proj.weight"), L("self_attn.out_proj.bias"))
        h = F.layer_norm(x, (d,), L("final_layer_norm.weight"), L("final_layer_norm.bias"), eps)
        u = F.gelu(F.linear(h, L("image_ffn.0.wi_0.weight"))) * F.linear(h, L("image_ffn.0.wi_1.weight"))
        u = F.layer_norm(u, (u.shape[-1],), L("image_ffn.2.weight"), L("image_ffn.2.bias"), eps)
        x = x + L("gamma_2") * F.linear(u, L("image_ffn.3.weight"), L("image_ffn.3.bias"))
        i += 1
    z = F.layer_norm(x[:, 1:].mean(1), (d,), P["fc_norm.weight"], P["fc_norm.bias"], eps)
    return F.linear(z, P["head.weight"], P["head.bias"]).float()


def flops_per_image(S, d=1536, ffn=6144, layers=40):
    """Multiply-adds x 2 of the encoder: QKV, out_proj, GeGLU (two halves), fc2, and the two attention products."""
    return 2 * layers * S * (3 * d * d + d * d + 2 * d * ffn + ffn * d + 2 * S * d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit.py needs a CUDA device")
    from one_peace_b200 import kernels as K
    from one_peace_b200.optim.adam import AdjustAdam
    from one_peace_b200.vision import models_vit as mv
    from one_peace_b200.vision.losses import SoftTargetCrossEntropy

    torch.manual_seed(0)
    res = dict(metric="vit", card=card(), layers=a.layers)
    B = 64
    for variant, R in (("one_piece_g_256", 256), ("one_piece_g_384", 384), ("one_piece_g_512", 512)):
        with torch.device("cuda"):
            m = getattr(mv, variant)(num_classes=1000, layers=a.layers).eval()
        P = {k: (v.detach().bfloat16() if v.is_floating_point() else v) for k, v in m.state_dict().items()}
        img = torch.randn(B, 3, R, R, device="cuda")
        img16 = img.bfloat16()
        S = (R // 16) ** 2 + 1
        with torch.no_grad():
            ours = lambda: m(img)                                  # noqa: E731
            eager = lambda: eager_bf16_forward(P, img16, 24)       # noqa: E731
            for _ in range(a.warmup):
                ours()
                eager()
            rounds = []
            for _ in range(2):                                     # alternate the two, twice
                rounds.append((time_cuda(ours, a.iters), time_cuda(eager, a.iters)))
        o, e = min(r[0] for r in rounds), min(r[1] for r in rounds)
        res[f"eval_{R}"] = dict(S=S, batch=B, ms=[round(r[0], 1) for r in rounds], eager_bf16_ms=[round(r[1], 1) for r in rounds],
                               images_per_s=round(B / o * 1e3, 1), eager_images_per_s=round(B / e * 1e3, 1),
                               encoder_tflops=round(flops_per_image(S, layers=a.layers) * B / o / 1e9, 1))
        del m, P, img, img16
        torch.cuda.empty_cache()

    # one fine-tuning step at 384^2
    Bt = 8
    with torch.device("cuda"):
        m = mv.one_piece_g_384(num_classes=1000, drop_path_rate=0.4, layers=a.layers)
    m.train()
    n_layers = len(m.encoder.layers) + 1
    groups = {}
    for n, p in m.named_parameters():
        lid = 0 if n.startswith("image_adapter") else (int(n.split(".")[2]) + 1 if n.startswith("encoder.layers") else n_layers)
        nd = p.ndim == 1 or n in m.no_weight_decay()
        groups.setdefault((lid, nd), dict(params=[], lr_scale=0.85 ** (n_layers - lid), weight_decay=0.0 if nd else 0.05))
        groups[(lid, nd)]["params"].append(p)
    opt = AdjustAdam(SimpleNamespace(lr=[5e-4], adam_betas=(0.9, 0.999), adam_eps=1e-8, weight_decay=0.05), list(groups.values()))
    opt.set_lr(5e-4)
    crit = SoftTargetCrossEntropy()
    img = torch.randn(Bt, 3, 384, 384, device="cuda")
    target = torch.softmax(torch.randn(Bt, 1000, device="cuda"), 1)

    def step():
        opt.optimizer.zero_grad(set_to_none=True)
        crit(m(img), target).backward()
        opt.step()
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    step_ms = min(time_cuda(step, a.iters) for _ in range(2))
    res["finetune_384"] = dict(batch=Bt, drop_path=0.4, step_ms=round(step_ms, 1), images_per_s=round(Bt / step_ms * 1e3, 1))
    del m, opt, groups
    torch.cuda.empty_cache()

    # the head kernels alone
    Bh, Sh, d = 64, 1025, 1536
    x = torch.randn(Bh, Sh, d, device="cuda")
    gamma, beta = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
    _, mm, mean, rstd = K.token_mean_ln_fwd(x, gamma, beta, 1e-5)
    dy = torch.randn(Bh, d, device="cuda")
    dx = torch.empty_like(x)
    for _ in range(5):
        K.token_mean_ln_fwd(x, gamma, beta, 1e-5)
        K.token_mean_ln_bwd(dy, mm, mean, rstd, gamma, dx)
    fwd_us = time_cuda(lambda: K.token_mean_ln_fwd(x, gamma, beta, 1e-5), 50) * 1e3
    bwd_us = time_cuda(lambda: K.token_mean_ln_bwd(dy, mm, mean, rstd, gamma, dx), 50) * 1e3
    floor_us = x.numel() * 4 / HBM * 1e6
    res["head_kernels"] = dict(B=Bh, S=Sh, d=d, MB=round(x.numel() * 4 / 1e6, 1), fwd_us=round(fwd_us, 1), bwd_us=round(bwd_us, 1),
                               floor_us=round(floor_us, 1), fwd_share=round(floor_us / fwd_us, 3),
                               bwd_share=round(floor_us / bwd_us, 3))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
