"""TEST INFRASTRUCTURE.  Generates tests/golden/adan.pt by executing the reference's OWN optim/adan.py (the python ``Adan``,
via oracle/ref_stub.py) on the CPU, on seeded parameters and gradients:

    python oracle/make_golden_adan.py

adan.py imports omegaconf (absent here) at module scope for FairseqAdan's config; the same shell make_golden.py uses for
adam.py is installed.  Only the ``Adan`` class is run.

Every case has three parameters in two param groups (lr, wd) = (1e-2, 0.05) and (5e-3, 0.0):
  a  [16, 16] in group 0, a gradient at every step;
  b  [37]     in group 0, its first gradient at step 3 (the group is at step 3 then: diff = 0, bias correction of t = 3);
  c  [96]     in group 1, no gradient (grad None) at step 2: skipped, its state (pre_grad included) kept.
Cases: fp32 and bf16 parameters (and gradients of the same dtype), no_prox both ways; ``scaled``: fp32, gradients
multiplied by SCALE before each step, as fairseq's memory-efficient wrapper does in place before ``FairseqAdan.step`` (the
fixture stores the unscaled gradients and the factor); ``resume``: the state_dict of the fp32 proximal run after 2 steps.
Each case stores the initial parameters, the gradients per step (None where absent), the parameters after every step and
the final optimizer state of each parameter (exp_avg, exp_avg_diff, exp_avg_sq, pre_grad) and of each group (step).
"""
import copy
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "adan.pt")
STEPS = 5
SHAPES = {"a": (16, 16), "b": (37,), "c": (96,)}
GROUPS = [dict(names=("a", "b"), lr=1e-2, weight_decay=0.05), dict(names=("c",), lr=5e-3, weight_decay=0.0)]
BETAS, EPS = (0.98, 0.92, 0.99), 1e-8
SCALE = 1.0 / 3.7
RESUME_AFTER = 2


def inputs(seed=0):
    """fp32 initial parameters and gradients [step][name] (None: no gradient at that step)"""
    g = torch.Generator().manual_seed(seed)
    p0 = {k: torch.randn(s, generator=g) for k, s in SHAPES.items()}
    grads = []
    for t in range(1, STEPS + 1):
        row = {k: torch.randn(s, generator=g) * (0.05 + 0.3 * t) for k, s in SHAPES.items()}
        if t < 3:
            row["b"] = None
        if t == 2:
            row["c"] = None
        grads.append(row)
    return p0, grads


def run(Adan, dtype, no_prox, scale=None, resume_after=None):
    p0, grads = inputs()
    params = {k: torch.nn.Parameter(v.clone().to(dtype)) for k, v in p0.items()}
    opt = Adan([dict(params=[params[k] for k in gr["names"]], lr=gr["lr"], weight_decay=gr["weight_decay"])
                for gr in GROUPS], betas=BETAS, eps=EPS, no_prox=no_prox)
    traj, saved = [], None
    for t, row in enumerate(grads, start=1):
        for k, q in params.items():
            gk = row[k]
            if gk is None:
                q.grad = None
            else:
                q.grad = gk.clone().to(dtype)
                if scale is not None:
                    q.grad.mul_(scale)          # fairseq multiplies the gradients in place before FairseqAdan.step
        opt.step()
        traj.append({k: q.detach().clone() for k, q in params.items()})
        if resume_after == t:
            saved = copy.deepcopy(opt.state_dict())
    state = {k: {n: opt.state[q][n].clone() for n in ("exp_avg", "exp_avg_diff", "exp_avg_sq", "pre_grad")}
             for k, q in params.items()}
    out = dict(dtype=dtype, no_prox=no_prox, scale=scale, p0={k: v.to(dtype) for k, v in p0.items()},
               grads=[{k: (None if v is None else v.to(dtype)) for k, v in row.items()} for row in grads],
               traj=traj, state=state, group_steps=[gr["step"] for gr in opt.param_groups])
    if saved is not None:
        out["resume_after"], out["state_dict"] = resume_after, saved
    return out


def main():
    om = types.ModuleType("omegaconf")
    om.II = lambda x: None
    om.OmegaConf = object
    sys.modules.setdefault("omegaconf", om)
    Adan = ref_stub.ref_module("one_peace.optim.adan").Adan
    torch.set_num_threads(1)
    cases = {
        "fp32_prox": run(Adan, torch.float32, False),
        "fp32_noprox": run(Adan, torch.float32, True),
        "bf16_prox": run(Adan, torch.bfloat16, False),
        "bf16_noprox": run(Adan, torch.bfloat16, True),
        "scaled": run(Adan, torch.float32, False, scale=SCALE),
        "resume": run(Adan, torch.float32, False, resume_after=RESUME_AFTER),
    }
    torch.save(dict(shapes=SHAPES, groups=GROUPS, betas=BETAS, eps=EPS, steps=STEPS, cases=cases), OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
