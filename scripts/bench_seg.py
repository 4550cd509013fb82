"""Segmentation backbone (vision/seg.py, OnePeaceAdapter) at 896^2 on one GPU: ms per crop at B = 1 and 2 with TFLOP/s
from the shape count, alternated in one process with the eager bf16 torch restatement (oracle/restated_seg.py); the
per-part split of the forward (CUDA events at the part boundaries: SPM, stem, injectors, layers, extractors, output maps);
one layer's attention at S = 3137 in LUT form against the
dense table (its build included), and the two csrc/seg.cu kernels against their HBM floors.  Prints one JSON line with
the card's name and power limit read in the same run.

    python scripts/bench_seg.py [--steps 10] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

import restated_seg as RS  # noqa: E402
import synth_seg as ss  # noqa: E402
from one_peace_b200 import kernels as K  # noqa: E402
from one_peace_b200.vision.seg import OnePeaceAdapter, make_image_bucket_position  # noqa: E402

D, H, F, L, SIDE = 1536, 24, 6144, 40, 56


def flops_per_crop():
    """Shapes only: the 40 layers (GEMMs + attention), injectors, extractors with ConvFFN, transposed conv."""
    S, T, P = SIDE * SIDE + 1, 21 * (SIDE // 2) ** 2, SIDE * SIDE
    layer = 2 * S * D * (3 * D + D + 2 * F) + 2 * S * F * D + 4 * S * S * D
    msda = lambda q, v, lvl: 2 * v * D * D // 2 + 2 * q * D * (3 * H * lvl * 4) + 2 * q * D // 2 * D
    inj = 4 * msda(P, T, 3)
    ext = 6 * (msda(T, P, 1) + 2 * T * D * 384 * 2)
    convt = 2 * (2 * SIDE) ** 2 * D * 4 * D
    return L * layer + inj + ext + convt


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = "cuda"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    torch.manual_seed(0)
    with torch.device("meta"):
        m = OnePeaceAdapter(**ss.PRODUCTION)
    m = m.to_empty(device=dev)
    bucket = m.encoder.layers[0].rp_bucket                  # one tensor under every layer's name
    bucket.copy_(make_image_bucket_position(SIDE, (2 * SIDE - 1) ** 2 + 3))
    m.load_state_dict(ss.seg_state_dict(m, device=dev), strict=True)
    m.eval().requires_grad_(False)
    res = dict(gpu=smi, flop_per_crop=flops_per_crop())
    sd16 = {k: (v.to(torch.bfloat16) if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    cfg = ss.PRODUCTION
    eager = lambda x: RS.forward(sd16, x, cfg["attention_heads"], cfg["deform_num_heads"], cfg["n_points"],
                                 cfg["interaction_indexes"])
    with torch.no_grad():
        for B in (1, 2):
            x = ss.seg_images(B, SIDE, device=dev)
            x16 = x.to(torch.bfloat16)
            ours, base = [], []
            for _ in range(args.rounds):                     # alternated: both see the same clocks and neighbours
                ours.append(timed(lambda: m(x), args.steps))
                base.append(timed(lambda: eager(x16), args.steps))
            ms, ms_eager = sorted(ours)[len(ours) // 2], sorted(base)[len(base) // 2]
            m.part_events = []
            m(x)
            torch.cuda.synchronize()
            parts, prev = {}, m.part_events[0][1]
            for name, ev in m.part_events[1:]:
                parts[name] = parts.get(name, 0.0) + prev.elapsed_time(ev)
                prev = ev
            m.part_events = None
            res[f"b{B}"] = dict(ms_per_crop=ms / B, tflops=flops_per_crop() * B / ms / 1e9, eager_bf16_ms_per_crop=ms_eager / B,
                                speedup_over_eager=ms_eager / ms, rounds_ms=ours, eager_rounds_ms=base,
                                parts_ms={k: round(v, 3) for k, v in parts.items()})
        # one layer's attention at S = 3137: LUT form against the dense table, the table's build included
        S = SIDE * SIDE + 1
        qkv = (0.5 * torch.randn(S, 3 * D, device=dev)).to(torch.bfloat16)
        layer = m.encoder.layers[0]
        lut = m.encoder.biases()[0]
        table = layer.rel_pos_table.weight.float().contiguous()
        res["attention_lut_ms"] = timed(lambda: K.attention_tc(qkv, lut, None, 1, S, H), args.steps)
        res["attention_dense_ms"] = timed(lambda: K.attention(qkv, K.relpos_bias_build(table, bucket, S, H), None, 1, S, H),
                                          args.steps)
        res["lut_len"] = int(lut.lut.shape[1])
        # the two new kernels against their HBM floors (3.35 TB/s data-sheet bandwidth)
        shapes = [(112, 112), (56, 56), (28, 28)]
        T = sum(h * w for h, w in shapes)
        h = torch.randn(T, 384, device=dev).to(torch.bfloat16)
        w9, bb = torch.randn(9, 384, device=dev), torch.randn(384, device=dev)
        ms = timed(lambda: K.seg_dwconv_gelu(h, w9, bb, shapes, 1), 50)
        res["dwconv_gelu"] = dict(us=1e3 * ms, hbm_floor_us=1e6 * 2 * h.numel() * 2 / 3.35e12)
        c = torch.randn(T, D, device=dev)
        xv = torch.randn(S, D, device=dev)
        sc, sh = torch.ones(D, device=dev), torch.zeros(D, device=dev)
        c1 = torch.randn(224 * 224, D, device=dev)
        up = torch.randn(112 * 112, 4 * D, device=dev)
        ms = timed(lambda: K.seg_out_map(c1, 224 * 224, 0, xv, S, 1, SIDE, sc, sh, 1, 224, 224, extra=up), 20)
        byt = 4 * (c1.numel() * 2 + up.numel() + SIDE * SIDE * D)
        res["out_map_c1"] = dict(us=1e3 * ms, hbm_floor_us=1e6 * byt / 3.35e12)
        ms = timed(lambda: K.seg_out_map(c, T, 0, xv, S, 1, SIDE, sc, sh, 1, 112, 112), 20)
        byt = 4 * (2 * 112 * 112 * D + SIDE * SIDE * D)
        res["out_map_c2"] = dict(us=1e3 * ms, hbm_floor_us=1e6 * byt / 3.35e12)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
