"""Times the fused Adan step on the parameters of the VGGSound-shaped one_peace_classify at 4B width (head_type audio, 40
layers, d = 1536, 309 classes) with layer-decay groups (0.95), against its HBM floor (bytes the step must move / 3.35 TB/s:
38 B per parameter with bf16 p and g, 44 B with fp32 p and g or with a master copy) and against the reference's eager
arithmetic (oracle/restated_adan.py ``adan_step``, one parameter at a time) on the same parameters; checks that fused and eager
parameters agree after a few steps; and times the whole fine-tuning step (bench_classify_step.py's workload) with `adan`
next to `adjust_adam`.  Prints one JSON line and writes it to --out if given.

    python scripts/bench_adan_step.py [--steps 10] [--warmup 3] [--layers 40] [--out result.json]
"""
import argparse
import json
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_classify_step import HBM, card, layer_decay_groups, time_cuda  # noqa: E402

BETAS = (0.98, 0.92, 0.99)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adan_step.py needs a CUDA device")
    import restated_adan as restated
    from one_peace_b200.criterions import ClassifyCriterion
    from one_peace_b200.one_peace.hub_interface import from_pretrained
    from one_peace_b200.optim import Adan, AdjustAdam, FairseqAdan

    torch.manual_seed(0)
    B, n_cls, secs = 8, 309, 15
    hub = from_pretrained(model_type="one_peace_classify", head_type="audio", num_classes=n_cls, layers=a.layers, device="cuda")
    m = hub.model
    m.train()
    L = len(m.encoder_wrapper.fusion_model.layers)
    for i, layer in enumerate(m.encoder_wrapper.fusion_model.layers):
        layer.drop_path_prob = 0.6 * i / max(L - 1, 1)
    params = list(m.parameters())
    for p in params:
        p.requires_grad_(True)
    n_par = sum(p.numel() for p in params)
    p_dtype = params[0].dtype

    # ---- the optimizer step alone: synthetic gradients on every parameter ----
    gen = torch.Generator(device="cuda").manual_seed(1)
    for p in params:
        p.grad = (torch.randn(p.shape, device="cuda", generator=gen) * 1e-3).to(p.dtype)
    groups = layer_decay_groups(m, 2e-5, 0.95, L)
    opt = Adan(groups, lr=2e-5, betas=BETAS, weight_decay=0.05)
    opt.step()                               # state allocated, first step
    torch.cuda.synchronize()
    fused_us = time_cuda(opt.step, 20)
    bytes_per = 38 if p_dtype == torch.bfloat16 else 44
    floor_us = n_par * bytes_per / HBM * 1e6

    # ---- eager reference arithmetic on the same parameters (one python loop over every parameter) ----
    def snapshot():
        return {p: (p.detach().float().clone(), {k: opt.state[p][k].clone() for k in ("exp_avg", "exp_avg_diff",
                                                                                      "exp_avg_sq", "pre_grad")})
                for p in params}

    def eager_step(store):
        for g in opt.param_groups:
            t = g["step"] + 1
            for p in g["params"]:
                p32, st = store[p]
                st["pre_grad"] = restated.adan_step(p32, p.grad.float(), st["exp_avg"], st["exp_avg_diff"], st["exp_avg_sq"],
                                                    st["pre_grad"], t, g["lr"], BETAS, 1e-8, g["weight_decay"])
    snap = snapshot()
    eager_step(snap)
    torch.cuda.synchronize()
    eager_us = time_cuda(lambda: eager_step(snap), 3)
    del snap

    # ---- fused vs eager parameters after a few steps, from the same starting state ----
    store = snapshot()
    worst = 0.0
    for _ in range(3):
        eager_step(store)
        opt.step()
        for p in params:
            want = store[p][0].to(p.dtype).float()
            store[p] = (want.clone(), store[p][1])
            scale = want.abs().max().clamp_min(1e-30)
            worst = max(worst, float(((p.detach().float() - want).abs().max() / scale)))
    del store, opt
    for p in params:
        p.grad = None
    torch.cuda.empty_cache()

    # ---- the whole fine-tuning step with adan and with adjust_adam ----
    wav = torch.nn.functional.layer_norm(torch.randn(B, 16000 * secs, device="cuda"), (16000 * secs,))
    frames = 16000 * secs
    for _, k, s in ((512, 10, 5),) + ((512, 3, 2),) * 4 + ((512, 2, 2),) * 2:
        frames = (frames - k) // s + 1
    pad = torch.zeros(B, frames + 1, dtype=torch.bool, device="cuda")
    pad[1, 1 + frames * 2 // 3:] = True
    sample = {"net_input": {"src_audios": wav, "audio_padding_masks": pad}, "target": torch.randint(0, n_cls, (B,), device="cuda"),
              "nsentences": B}
    crit = ClassifyCriterion(task=None, label_smoothing=0.1)
    step_ms = {}
    for name in ("adan", "adjust_adam"):
        if name == "adan":
            fo = FairseqAdan(SimpleNamespace(lr=[2e-5], adan_betas=BETAS, adan_eps=1e-8, weight_decay=0.05,
                                             fp16_adan_stats=False), layer_decay_groups(m, 2e-5, 0.95, L))
        else:
            fo = AdjustAdam(SimpleNamespace(lr=[2e-5], adam_betas=(0.9, 0.999), adam_eps=1e-8, weight_decay=0.05),
                            layer_decay_groups(m, 2e-5, 0.95, L))

        def step():
            fo.optimizer.zero_grad(set_to_none=True)
            loss, n, _ = crit(m, sample)
            (loss / n).backward()
            fo.step()
        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        step_ms[name] = time_cuda(step, a.steps) / 1e3
        del fo
        torch.cuda.empty_cache()

    res = dict(metric="adan_step", card=card(), layers=L, params=n_par, param_dtype=str(p_dtype).replace("torch.", ""),
               groups=len(groups), fused_us=round(fused_us, 1), floor_us=round(floor_us, 1),
               floor_share=round(floor_us / fused_us, 3), eager_us=round(eager_us, 1),
               eager_over_fused=round(eager_us / fused_us, 1), fused_vs_eager_max_rel=float(f"{worst:.3g}"),
               step_ms_adan=round(step_ms["adan"], 2), step_ms_adjust_adam=round(step_ms["adjust_adam"], 2))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
