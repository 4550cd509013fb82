"""TEST INFRASTRUCTURE.  Generates tests/golden/msda.pt by executing the reference's OWN multi-scale deformable attention
module (one_peace_vision/seg/ops/modules/ms_deform_attn.py) in fp64 on the CPU.  It needs the reference source tree:

    python oracle/make_golden_msda.py

The compiled ``MultiScaleDeformableAttention`` import is stubbed (it is only called through MSDeformAttnFunction), and
``MSDeformAttnFunction.apply`` is routed to the reference's own ``ms_deform_attn_core_pytorch`` (grid_sample), so torch
autograd gives every gradient.

Stored per case: the config, the level layout, the fp32 inputs and parameters the case runs on, the fixed cotangent, and in
fp64 the output and the gradients of query, input_flatten and the eight parameters.  Also stored: the freshly initialised
state of each case's config (torch.manual_seed(0) before construction) and its key / shape list.
"""
import importlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402

SEG = os.path.join(ref_stub.REF_ROOT, "one_peace_vision", "seg")
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "msda.pt")

# name -> (module config, level shapes, N, Lq, L_ref, offset scale in pixels).  Every case has 32 channels per head.
CASES = {
    # the injector's form: three non-square levels, one reference point per query shared by the levels, ratio 0.5,
    # 3 * H * L * P = 36 projection columns (not a multiple of 8)
    "injector": (dict(d_model=64, n_levels=3, n_heads=1, n_points=4, ratio=0.5), [(6, 5), (3, 4), (2, 3)], 1, 7, 1, 2.5),
    # the extractor's form: one level
    "extractor": (dict(d_model=32, n_levels=1, n_heads=1, n_points=4, ratio=1.0), [(5, 6)], 1, 9, 1, 2.5),
    # per-level reference points, two samples, two heads
    "per_level_n2": (dict(d_model=64, n_levels=2, n_heads=2, n_points=3, ratio=1.0), [(4, 4), (2, 3)], 2, 5, 2, 4.0),
}


def load_reference():
    """The reference's ops package with the extension stubbed and the CUDA function routed to the torch core."""
    ref_stub._mod("MultiScaleDeformableAttention")
    sys.path.insert(0, SEG)
    func = importlib.import_module("ops.functions.ms_deform_attn_func")
    mod = importlib.import_module("ops.modules.ms_deform_attn")

    def apply(value, shapes, start_index, locations, weights, im2col_step):
        return func.ms_deform_attn_core_pytorch(value, shapes, locations, weights)
    func.MSDeformAttnFunction.apply = staticmethod(apply)
    return mod


def case_inputs(name, m, shapes, N, Lq, L_ref, off_scale):
    """Seeded parameters (the init perturbed: offsets of a few pixels, so some taps fall partly or wholly outside, and
    non-uniform soft-max weights) and inputs, all fp32."""
    g = torch.Generator().manual_seed(sorted(CASES).index(name) + 11)
    d = m.d_model
    state = {}
    for k, v in m.state_dict().items():
        noise = torch.randn(v.shape, generator=g)
        if k == "sampling_offsets.weight":
            v = noise * (off_scale / d ** 0.5) / 4
        elif k == "sampling_offsets.bias":
            v = v * off_scale / 2 + noise
        elif k == "attention_weights.weight":
            v = noise / d ** 0.5
        else:
            v = v + 0.1 * noise if k.endswith("bias") else v
        state[k] = v.float().contiguous()
    len_in = sum(h * w for h, w in shapes)
    query = torch.randn(N, Lq, d, generator=g)
    feat = torch.randn(N, len_in, d, generator=g)
    ref = torch.rand(N, Lq, L_ref, 2, generator=g) * 0.9 + 0.05
    cot = torch.randn(N, Lq, d, generator=g)
    return state, query, feat, ref, cot


def main():
    mod = load_reference()
    torch.set_num_threads(8)
    out = {"cases": {}, "init": {}}
    for name, (cfg, shapes, N, Lq, L_ref, off_scale) in CASES.items():
        torch.manual_seed(0)
        m = mod.MSDeformAttn(**cfg)
        out["init"][name] = {k: v.clone() for k, v in m.state_dict().items()}
        out["keys"] = out.get("keys", {})
        out["keys"][name] = [(k, tuple(p.shape)) for k, p in m.named_parameters()]
        state, query, feat, ref, cot = case_inputs(name, m, shapes, N, Lq, L_ref, off_scale)
        m = m.double()
        m.load_state_dict({k: v.double() for k, v in state.items()})
        q = query.double().requires_grad_(True)
        x = feat.double().requires_grad_(True)
        sp = torch.tensor(shapes, dtype=torch.long)
        start = torch.cat([sp.new_zeros(1), (sp[:, 0] * sp[:, 1]).cumsum(0)[:-1]])
        y = m(q, ref.double(), x, sp, start)
        (y * cot.double()).sum().backward()
        out["cases"][name] = dict(
            config=cfg, shapes=shapes, starts=start.tolist(), state=state, query=query, input_flatten=feat,
            reference_points=ref, cotangent=cot, output=y.detach(), d_query=q.grad, d_input_flatten=x.grad,
            grads={k: p.grad.clone() for k, p in m.named_parameters()})
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
