"""Multi-scale deformable attention core at the segmentation recipe's shapes (896^2, N = 1): the sm_90a kernels
(opb_ms_deform_attn_fwd / _bwd), the reference's compiled op (oracle/_ref/, fp32, when built) and an eager torch grid_sample
restatement (fp32), forward and forward + backward, timed alternately in one process with CUDA events.

    python scripts/bench_msda.py [--iters 50] [--rounds 3] [--out results.json]

Every variant starts from the value_proj output and the [offsets | logits] projection, so each includes what it must do to
turn those into the output: ours fuses the soft-max and the locations, the other two run them as torch ops.  "bytes" is what
the op must move at least: value once (bf16 for ours, fp32 for the others), proj, ref and the output; the backward adds
d_out, d_value (fp32, read and written) and d_proj.  "hbm share" is that over 3.35 TB/s, over the measured time.
"""
import argparse
import glob
import importlib.machinery
import importlib.util
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from one_peace_b200 import kernels as K  # noqa: E402

HBM = 3.35e12
SHAPES = {   # name -> (Lq, H, level shapes, P, L_ref)
    "injector": (3136, 24, [(112, 112), (56, 56), (28, 28)], 4, 1),
    "extractor": (16464, 24, [(56, 56)], 4, 1),
    "pixel_decoder": (16464, 32, [(112, 112), (56, 56), (28, 28)], 4, 3),
}


def ref_op():
    hits = sorted(glob.glob(os.path.join(ROOT, "oracle", "_ref", "MultiScaleDeformableAttention*.so")))
    if not hits:
        return None
    loader = importlib.machinery.ExtensionFileLoader("MultiScaleDeformableAttention", hits[0])
    mod = importlib.util.module_from_spec(importlib.util.spec_from_loader("MultiScaleDeformableAttention", loader))
    loader.exec_module(mod)
    return mod


def locations(proj, ref, shapes, Lq, H, P):
    L = len(shapes)
    pr = proj.view(1, Lq, -1)
    off = pr[..., :2 * H * L * P].reshape(1, Lq, H, L, P, 2)
    attn = torch.softmax(pr[..., 2 * H * L * P:].reshape(1, Lq, H, L * P), -1).view(1, Lq, H, L, P)
    wh = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float32, device=proj.device)
    loc = ref.view(1, Lq, 1, ref.shape[1], 1, 2) + off / wh[None, None, None, :, None]
    return loc.contiguous(), attn.contiguous()


def torch_core(value, loc, attn, shapes, starts):
    N, S_in, H, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    out = 0
    for l, ((h, w), s0) in enumerate(zip(shapes, starts)):
        img = value[:, s0:s0 + h * w].permute(0, 2, 3, 1).reshape(N * H, D, h, w)
        grid = loc[:, :, :, l].permute(0, 2, 1, 3, 4).reshape(N * H, Lq, P, 2) * 2 - 1
        smp = F.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
        out = out + (smp * attn[:, :, :, l].permute(0, 2, 1, 3).reshape(N * H, 1, Lq, P)).sum(-1)
    return out.view(N, H, D, Lq).permute(0, 3, 1, 2).reshape(N, Lq, H * D)


def timeit(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_msda.py needs a GPU")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    MSDA = ref_op()
    results = {"gpu": smi, "reference_op": MSDA is not None, "shapes": {}}
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (Lq, H, shapes, P, L_ref) in SHAPES.items():
        L = len(shapes)
        S_in = sum(h * w for h, w in shapes)
        starts = [sum(h * w for h, w in shapes[:i]) for i in range(L)]
        HD, n_proj = H * 32, 3 * H * L * P
        value = torch.randn(S_in, HD, device="cuda", generator=g).to(torch.bfloat16)
        proj = torch.randn(Lq, n_proj, device="cuda", generator=g)
        proj[:, :2 * H * L * P] *= 2.0
        ref = torch.rand(Lq, L_ref, 2, device="cuda", generator=g)
        d_out = torch.randn(Lq, HD, device="cuda", generator=g).to(torch.bfloat16)
        v32 = value.float().view(1, S_in, H, 32).contiguous()
        sp = torch.tensor(shapes, dtype=torch.long, device="cuda")
        st = torch.tensor(starts, dtype=torch.long, device="cuda")
        dv = torch.zeros(S_in, HD, device="cuda")
        dp = torch.empty_like(proj)
        g32 = d_out.float().view(1, Lq, HD).contiguous()

        def ours_f():
            K.ms_deform_attn_fwd(value, proj, ref, shapes, starts, 1, Lq, H, P)

        def ours_fb():
            K.ms_deform_attn_fwd(value, proj, ref, shapes, starts, 1, Lq, H, P)
            dv.zero_()
            K.ms_deform_attn_bwd(value, proj, ref, d_out, shapes, starts, 1, Lq, H, P, d_value=dv, d_proj=dp)

        def ref_f():
            loc, attn = locations(proj, ref, shapes, Lq, H, P)
            MSDA.ms_deform_attn_forward(v32, sp, st, loc, attn, 64)

        def ref_fb():
            loc, attn = locations(proj, ref, shapes, Lq, H, P)
            MSDA.ms_deform_attn_forward(v32, sp, st, loc, attn, 64)
            MSDA.ms_deform_attn_backward(v32, sp, st, loc, attn, g32, 64)

        pv = proj.clone().requires_grad_(True)
        vv = v32.clone().requires_grad_(True)

        def torch_f():
            with torch.no_grad():
                loc, attn = locations(proj, ref, shapes, Lq, H, P)
                torch_core(v32, loc, attn, shapes, starts)

        def torch_fb():
            pv.grad = vv.grad = None
            loc, attn = locations(pv, ref, shapes, Lq, H, P)
            torch_core(vv, loc, attn, shapes, starts).backward(g32)

        variants = {"ours": (ours_f, ours_fb), "torch_grid_sample": (torch_f, torch_fb)}
        if MSDA is not None:
            variants["reference_op"] = (ref_f, ref_fb)
        times = {k: {"fwd": [], "fwd_bwd": []} for k in variants}
        for _ in range(args.rounds):
            for k, (f, fb) in variants.items():
                times[k]["fwd"].append(timeit(f, args.iters))
                times[k]["fwd_bwd"].append(timeit(fb, args.iters))
        out_b = 2 * Lq * HD
        fwd_bytes = {"ours": 2 * S_in * HD + 4 * Lq * (n_proj + 2 * L_ref) + out_b}
        fwd_bytes["fp32"] = 4 * S_in * HD + 4 * Lq * (n_proj + 2 * L_ref) + 4 * Lq * HD
        bwd_extra = 2 * Lq * HD + 2 * 4 * S_in * HD + 4 * Lq * n_proj
        row = {}
        for k, t in times.items():
            fb_bytes = fwd_bytes["ours" if k == "ours" else "fp32"]
            tf, tfb = min(t["fwd"]), min(t["fwd_bwd"])
            row[k] = {"fwd_us": round(tf, 1), "fwd_bwd_us": round(tfb, 1), "fwd_us_all": [round(x, 1) for x in t["fwd"]],
                      "fwd_bwd_us_all": [round(x, 1) for x in t["fwd_bwd"]], "fwd_bytes": fb_bytes,
                      "fwd_hbm_share": round(fb_bytes / HBM / (tf * 1e-6), 3),
                      "fwd_bwd_bytes": 2 * fb_bytes + bwd_extra,
                      "fwd_bwd_hbm_share": round((2 * fb_bytes + bwd_extra) / HBM / (tfb * 1e-6), 3)}
        results["shapes"][name] = row
        print(name, json.dumps(row))
        del value, proj, ref, d_out, v32, dv, dp, g32, pv, vv
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
