"""Detection backbone (one_peace_b200.vision.det.OnePeace, production config) at 1280^2 with random weights on one GPU.

Prints one JSON line: the card name and power limit read in the same run; images/s and ms per image at B = 1 and 2;
the decomposed attention alone at S = 6400 (B = 1) and S = 256 (B = 25) in us per launch and TFLOP/s; the projection kernel
against its HBM floor; and a torch eager bf16 restatement (oracle/restated_det.py with SDPA taking the bias and the
decomposed terms as a float mask), timed alternately with this path in the same process.

FLOP counts (per image): GEMMs 2 (4 d^2 + 3 d F) per token per layer = 8 d^2 + 6 d F; attention 4 S_seq * 64 per query row
and head (q.k and P.v), over 6400-token sequences in the 10 global layers and 256-token windows in the 30 window layers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

D, F_, H, L, SIDE, WIN = 1536, 6144, 24, 40, 80, 16
N_GLOBAL = 10
HBM = 3.35e12


def flops_per_image():
    tok = SIDE * SIDE
    gemm = L * tok * (8 * D * D + 6 * D * F_)
    glob = N_GLOBAL * H * tok * 4 * tok * 64
    win = (L - N_GLOBAL) * H * tok * 4 * WIN * WIN * 64
    return gemm, glob, win


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_det.py needs a CUDA device")
    import restated_det
    import synth_det as sd_
    from one_peace_b200 import kernels as K
    from one_peace_b200.vision.det import OnePeace
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    lin = torch.linspace
    torch.linspace = lambda *a, **k: lin(*a, **{**k, "device": "cpu"})
    try:
        with torch.device("meta"):
            m = OnePeace(**sd_.PRODUCTION)
    finally:
        torch.linspace = lin
    m = m.to_empty(device="cuda")
    bufs = {"image_adapter.rp_bucket": restated_det.make_image_bucket_position(80, 159 * 159 + 3)[1:, 1:].contiguous(),
            "image_adapter.rp_bucket_window": restated_det.make_image_bucket_position(16, 31 * 31 + 3)[1:, 1:].contiguous()}
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    sd = sd_.det_state_dict(shapes, {k: v.cuda() for k, v in bufs.items()}, device="cuda")
    m.load_state_dict(sd, strict=True)
    m.eval().requires_grad_(False)
    res = dict(card=smi, flops_per_image=dict(zip(("gemm", "global_attn", "window_attn"), flops_per_image())))
    gemm, glob, win = flops_per_image()
    with torch.no_grad():
        for B in (1, 2):
            img = sd_.det_images(80, batch=B).cuda()
            m(img)
            ms = timed(lambda: m(img), args.iters)
            res[f"B{B}"] = dict(ms_per_image=ms / B, images_per_s=1000.0 * B / ms,
                                tflops=(gemm + glob + win) * B / (ms * 1e-3) / 1e12)
        # torch eager bf16 restatement, alternated with this path at B = 1
        sd16 = {k: (v.to(torch.bfloat16) if v.is_floating_point() else v) for k, v in sd.items()}
        img = sd_.det_images(80, batch=1).cuda()
        eager = lambda: restated_det.forward(sd16, img, H, L, SIDE, WIN, sd_.PRODUCTION["window_block_indexes"],
                                             dtype=torch.bfloat16, sdpa=True)
        eager()
        ours, theirs = [], []
        for _ in range(3):
            ours.append(timed(lambda: m(img), 2))
            theirs.append(timed(eager, 2))
        res["alternating_B1_ms"] = dict(this=min(ours), torch_eager_bf16_sdpa=min(theirs))
        # the two kernels alone
        for name, B, side in (("global_S6400_B1", 1, SIDE), ("window_S256_B25", 25, WIN)):
            S = side * side
            g = torch.Generator(device="cuda").manual_seed(0)
            qkv = (torch.randn(B * S, 3 * H * 64, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
            rph = 0.1 * torch.randn(2 * side - 1, 64, device="cuda", generator=g)
            yy = torch.arange(S, device="cuda") // side
            py, px = yy.int().contiguous(), (torch.arange(S, device="cuda") % side).int().contiguous()
            code = yy * (2 * side - 1) + torch.arange(S, device="cuda") % side
            maxc = (side - 1) * 2 * side
            rp = K.RelPosBias(lut=0.1 * torch.randn(H, (2 * side - 1) ** 2, device="cuda", generator=g),
                              code_row=(code + maxc).int().contiguous(), code_col=code.int().contiguous())
            rh, rw = K.relpos_decomp_proj(qkv, rph, rph, py, px, B, S, H, side, side)
            out = torch.empty(B * S, H * 64, dtype=torch.bfloat16, device="cuda")
            st = torch.empty(H * B * S * 2, device="cuda")
            n = 20
            t_proj = timed(lambda: K.relpos_decomp_proj(qkv, rph, rph, py, px, B, S, H, side, side, rel_h=rh, rel_w=rw), n)
            t_att = timed(lambda: K.attention_decomp(qkv, rp, rh, rw, py, px, B, S, H, side, side, out=out, ln_stats=st), n)
            proj_bytes = B * H * S * 2 * side * 4 + B * S * H * 64 * 2
            att_flops = B * H * S * S * 4 * 64
            res[name] = dict(attention_us=t_att * 1e3, attention_tflops=att_flops / (t_att * 1e-3) / 1e12,
                             proj_us=t_proj * 1e3, proj_hbm_floor_us=proj_bytes / HBM * 1e6,
                             proj_share_of_floor=(proj_bytes / HBM) / (t_proj * 1e-3))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
