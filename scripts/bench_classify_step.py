"""Times the VGGSound-shaped fine-tuning step of one_peace_classify at 4B width (40 layers, d = 1536, 24 heads; 8 clips of
15 s; 309 classes; drop-path 0.6; AdjustAdam with layer decay 0.95), and the attention-pooling kernels alone next to their HBM
floors (bytes the kernel must move / 3.35 TB/s).  Prints one JSON line and writes it to --out if given.

    python scripts/bench_classify_step.py [--steps 10] [--warmup 3] [--layers 40] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

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
    return start.elapsed_time(end) / iters * 1e3          # us


def layer_decay_groups(model, lr, decay, n_layers):
    """lr_scale per parameter as the reference's utils/layer_decay.py assigns it: adapters are layer 0, encoder layer i is
    layer i + 1, everything else (final norms, classify_head) layer n_layers + 1."""
    groups = {}
    for name, p in model.named_parameters():
        if name.startswith("encoder_wrapper.fusion_model.layers."):
            lid = int(name.split(".")[3]) + 1
        elif "_adapter." in name:
            lid = 0
        else:
            lid = n_layers + 1
        scale = decay ** (n_layers + 1 - lid)
        groups.setdefault(scale, []).append(p)
    return [{"params": ps, "lr_scale": s, "lr": lr * s} for s, ps in groups.items()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_classify_step.py needs a CUDA device")
    from one_peace_b200 import kernels as K
    from one_peace_b200.criterions import ClassifyCriterion
    from one_peace_b200.one_peace.hub_interface import from_pretrained
    from one_peace_b200.optim.adam import AdjustAdam

    torch.manual_seed(0)
    B, n_cls, secs = 8, 309, 15
    hub = from_pretrained(model_type="one_peace_classify", head_type="audio", num_classes=n_cls, layers=a.layers, device="cuda")
    m = hub.model
    m.train()
    L = len(m.encoder_wrapper.fusion_model.layers)
    for i, layer in enumerate(m.encoder_wrapper.fusion_model.layers):
        layer.drop_path_prob = 0.6 * i / max(L - 1, 1)
    for p in m.parameters():
        p.requires_grad_(True)
    opt = AdjustAdam(SimpleNamespace(lr=[2e-5], adam_betas=(0.9, 0.999), adam_eps=1e-8, weight_decay=0.05),
                     layer_decay_groups(m, 2e-5, 0.95, L))
    wav = torch.nn.functional.layer_norm(torch.randn(B, 16000 * secs, device="cuda"), (16000 * secs,))
    frames = 16000 * secs
    for _, k, s in ((512, 10, 5),) + ((512, 3, 2),) * 4 + ((512, 2, 2),) * 2:
        frames = (frames - k) // s + 1
    pad = torch.zeros(B, frames + 1, dtype=torch.bool, device="cuda")
    pad[1, 1 + frames * 2 // 3:] = True
    sample = {"net_input": {"src_audios": wav, "audio_padding_masks": pad}, "target": torch.randint(0, n_cls, (B,), device="cuda"),
              "nsentences": B}
    crit = ClassifyCriterion(task=None, label_smoothing=0.1)

    def step():
        opt.optimizer.zero_grad(set_to_none=True)
        loss, n, _ = crit(m, sample)
        (loss / n).backward()
        opt.step()
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    step_ms = time_cuda(step, a.steps) / 1e3

    # the pooling kernels alone at the step's shape: T = frames keys, d = 1536
    d, T = m.encoder_wrapper.fusion_model.layers[0].embed_dim, frames
    kv = torch.randn(B * T, 2 * d, device="cuda").bfloat16()
    q = 0.02 * torch.randn(d // 64, 64, device="cuda")
    kp = pad[:, 1:].to(torch.uint8).contiguous()
    out, lse = K.attn_pool_fwd(kv, q, kp, B, T)
    dout = torch.randn(B, d, device="cuda").bfloat16()
    for _ in range(5):
        K.attn_pool_fwd(kv, q, kp, B, T)
        K.attn_pool_bwd(kv, q, kp, lse, dout, B, T)
    fwd_us = time_cuda(lambda: K.attn_pool_fwd(kv, q, kp, B, T), 200)
    bwd_us = time_cuda(lambda: K.attn_pool_bwd(kv, q, kp, lse, dout, B, T), 200)
    kv_bytes = kv.numel() * 2
    fwd_floor = kv_bytes / HBM * 1e6
    bwd_floor = 2 * kv_bytes / HBM * 1e6
    res = dict(metric="classify_step", card=card(), layers=L, batch=B, seconds=secs, classes=n_cls, step_ms=round(step_ms, 2),
               samples_per_s=round(B / step_ms * 1e3, 2), pool_T=T, kv_MB=round(kv_bytes / 1e6, 1),
               pool_fwd_us=round(fwd_us, 1), pool_fwd_floor_us=round(fwd_floor, 1), pool_fwd_share=round(fwd_floor / fwd_us, 3),
               pool_bwd_us=round(bwd_us, 1), pool_bwd_floor_us=round(bwd_floor, 1), pool_bwd_share=round(bwd_floor / bwd_us, 3))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
