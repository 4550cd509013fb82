"""Times the RefCOCO-shaped visual-grounding fine-tuning step of one_peace_classify at 4B width (40 layers, d = 1536, 24 heads;
head_type vl, 4 outputs, attention pooling, image features, head_scale_ratio 2; 4 image-text pairs at 384^2 with 20-token
texts, so the concatenated sequence is 577 + 21 = 598 tokens; drop-path 0.4; AdjustAdam with layer decay 0.9), its peak
memory, and the refcoco_criterion kernel alone next to eager torch + torchvision computing the same loss and gradient on the
same logits.  Prints one JSON line and writes it to --out if given.

    python scripts/bench_grounding_step.py [--steps 10] [--warmup 3] [--layers 40] [--out result.json]
"""
import argparse
import json
import os
import sys
from types import SimpleNamespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_classify_step import card, layer_decay_groups, time_cuda  # noqa: E402


def eager_loss(z, t, ns):
    """criterions/refcoco_loss.py:36-46 in eager torch + torchvision, forward and backward (the baseline the kernel replaces)."""
    from torchvision.ops import generalized_box_iou
    z = z.detach().requires_grad_(True)
    p = z.sigmoid()
    loss = torch.nn.functional.l1_loss(p, t, reduction="sum") / ns
    valid = (p[:, :2] < p[:, 2:]).all(1)
    loss = loss + (1 - torch.diag(generalized_box_iou(p[valid], t[valid]))).mean()
    loss.backward()
    return loss, z.grad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grounding_step.py needs a CUDA device")
    from one_peace_b200.autograd_classify import RefcocoLossFn
    from one_peace_b200.criterions import RefCOCOCriterion
    from one_peace_b200.one_peace.hub_interface import from_pretrained
    from one_peace_b200.optim.adam import AdjustAdam

    torch.manual_seed(0)
    B, res, text_len = 4, 384, 20
    hub = from_pretrained(model_type="one_peace_classify", head_type="vl", num_classes=4, layers=a.layers, device="cuda",
                          patch_image_size=res, head_scale_ratio=2, use_image_features=True)
    m = hub.model
    m.train()
    L = len(m.encoder_wrapper.fusion_model.layers)
    for i, layer in enumerate(m.encoder_wrapper.fusion_model.layers):
        layer.drop_path_prob = 0.4 * i / max(L - 1, 1)
    for p in m.parameters():
        p.requires_grad_(True)
    opt = AdjustAdam(SimpleNamespace(lr=[1.5e-4], adam_betas=(0.9, 0.999), adam_eps=1e-8, weight_decay=0.05),
                     layer_decay_groups(m, 1.5e-4, 0.9, L))
    tok = torch.randint(4, 50000, (B, text_len), device="cuda")
    tok[:, -1] = 2
    img = torch.randn(B, 3, res, res, device="cuda")
    lo = 0.5 * torch.rand(B, 2, device="cuda")
    tgt = torch.cat([lo, lo + 0.1 + 0.4 * torch.rand(B, 2, device="cuda")], 1)
    sample = {"net_input": {"src_tokens": tok, "src_images": img}, "target": tgt, "nsentences": B}
    crit = RefCOCOCriterion(task=None)

    def step():
        opt.optimizer.zero_grad(set_to_none=True)
        loss, _, _ = crit(m, sample)
        loss.backward()
        opt.step()
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    step_ms = time_cuda(step, a.steps) / 1e3
    peak_gb = torch.cuda.max_memory_allocated() / 2 ** 30

    # the criterion alone on the logits the model produces: [B, 4] view of the 8-wide padded classifier output
    with torch.no_grad():
        z = m(**sample["net_input"]).detach()
    z8 = torch.zeros(B, 8, device="cuda")
    z8[:, :4] = z
    zv = z8[:, :4].requires_grad_(True)

    def kernel():
        loss, _, _ = RefcocoLossFn.apply(zv, tgt, B)
        loss.backward()

    def eager():
        eager_loss(z, tgt, B)
    for _ in range(10):
        kernel()
        eager()
    kern_us = time_cuda(kernel, 200)
    eager_us = time_cuda(eager, 200)
    res_line = dict(metric="grounding_step", card=card(), layers=L, batch=B, image=res, text_len=text_len,
                    seq=(res // 16) ** 2 + 1 + text_len + 1, step_ms=round(step_ms, 2), pairs_per_s=round(B / step_ms * 1e3, 2),
                    peak_mem_GB=round(peak_gb, 2), loss_fn_us=round(kern_us, 1), eager_torchvision_us=round(eager_us, 1))
    line = json.dumps(res_line)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
