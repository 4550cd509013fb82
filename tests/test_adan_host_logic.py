"""CPU: the Adan optimizer's host side (optim/adan.py) and its error contract (tests/adan_ref.py).

* ``oracle/restated_adan.py`` ``adan_step`` reproduces tests/golden/adan.pt, made by the reference's own optim/adan.py.
* An fp32 emulation of ``adan_math`` (csrc/adam.cu), every operation rounded on its own, stays within ``adan_ref``'s
  bounds, and each planted mistake exceeds some bound at least 100-fold.
* ``FairseqAdan``'s config plumbing, its registration under ``adan`` and the YAML swap; the C ABI refuses bad arguments
  before any CUDA call.
"""
import ctypes
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import adan_ref as A
import restated_adan as restated

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adan.pt")
F = np.float32


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLDEN, weights_only=False)


def replay(fx, case, upto=None, start=None):
    """restated.adan_step over the fixture's steps; -> (params after each step, final state per name, group steps).
    ``start``: (step count, {name: state dict}, {name: p}) to continue from."""
    c = fx["cases"][case]
    groups = fx["groups"]
    dt = c["dtype"]
    if start is None:
        params = {k: v.float().clone() for k, v in c["p0"].items()}
        state, steps, t0 = {}, [0] * len(groups), 0
    else:
        t0, state, params = start
        steps = [t0] * len(groups)
    traj = []
    for t in range(t0 + 1, (upto or fx["steps"]) + 1):
        row = c["grads"][t - 1]
        for gi, gr in enumerate(groups):
            steps[gi] += 1
            for k in gr["names"]:
                if row[k] is None:
                    continue
                g = row[k].float()
                if c["scale"] is not None:
                    g = g * c["scale"]
                st = state.setdefault(k, {})
                if not st:
                    st.update(exp_avg=torch.zeros_like(g), exp_avg_diff=torch.zeros_like(g), exp_avg_sq=torch.zeros_like(g))
                p32 = params[k].to(dt).float() if dt != torch.float32 else params[k]
                st["pre_grad"] = restated.adan_step(p32, g, st["exp_avg"], st["exp_avg_diff"], st["exp_avg_sq"],
                                                    st.get("pre_grad"), steps[gi], gr["lr"], fx["betas"], fx["eps"],
                                                    gr["weight_decay"], c["no_prox"])
                params[k] = p32.to(dt).float() if dt != torch.float32 else p32
        traj.append({k: v.to(dt).clone() for k, v in params.items()})
    return traj, state, steps


def close(got, want, what):
    if want.dtype == torch.bfloat16:         # an fp32 difference of an ulp may move the rounding by one bf16 ulp
        torch.testing.assert_close(got.float(), want.float(), rtol=2 ** -7, atol=1e-30, msg=what)
    else:
        torch.testing.assert_close(got.float(), want.float(), rtol=1e-5, atol=1e-7, msg=what)


@pytest.mark.parametrize("case", ["fp32_prox", "fp32_noprox", "bf16_prox", "bf16_noprox", "scaled", "resume"])
def test_restatement_reproduces_golden(fixture, case):
    c = fixture["cases"][case]
    traj, state, steps = replay(fixture, case)
    assert steps == c["group_steps"]
    for t, (got, want) in enumerate(zip(traj, c["traj"]), start=1):
        for k in want:
            close(got[k], want[k], f"{case} step {t} {k}")
    for k, st in c["state"].items():
        for name, want in st.items():
            close(state[k][name], want, f"{case} {k} {name}")


def test_golden_pins_the_reference_rules(fixture):
    """b's first gradient comes at group step 3 (diff = 0 there, bias correction of t = 3); c keeps its pre_grad over the
    step without a gradient; the group steps count every call."""
    c = fixture["cases"]["fp32_prox"]
    assert c["group_steps"] == [5, 5]
    assert all(torch.equal(c["traj"][i]["b"], c["p0"]["b"]) for i in range(2))
    assert torch.equal(c["traj"][1]["c"], c["traj"][0]["c"])
    sd = fixture["cases"]["resume"]["state_dict"]
    assert [g["step"] for g in sd["param_groups"]] == [2, 2] and 1 not in sd["state"]
    assert set(sd["state"][0]) == {"exp_avg", "exp_avg_sq", "exp_avg_diff", "pre_grad"}


# ---- the kernel's arithmetic in fp32, with planted mistakes ----
def emulate(o, *, first, t, lr, wd, no_prox, betas=A.BETAS, eps=A.EPS, s=None, mistake=None):
    """``adan_math`` in numpy fp32 (each operation rounded on its own).  -> dict p, m, n, v, pre (float32 arrays)"""
    b1, b2, b3 = (F(b) for b in betas)
    if mistake == "swap_b2_b3":
        b2, b3 = b3, b2
    c1, c2, c3 = F(1) - b1, F(1) - b2, F(1) - b3
    tt = 1 if mistake == "param_step" else t
    bc1, bc2, sb3 = (F(x) for x in A.group_coefs(tt, betas))
    lr32, wd32, eps32 = F(lr), F(wd), F(eps)
    p, g, m, n, v, pre = (o[k].numpy().astype(F) for k in ("p", "g", "m", "n", "v", "pre"))
    x = g * F(1 if s is None else s)
    fst = np.broadcast_to(np.asarray(first), x.shape)
    d = np.where(fst & (mistake != "late_diff"), x - x, x - pre).astype(F)
    u = x + (c2 if mistake == "one_minus_b2_in_u" else b2) * d
    m = m * b1 + x * c1
    n = n * b2 + d * c2
    v = v * b3 + (c3 * u) * u
    if mistake == "eps_before_div":
        den = (np.sqrt(v) + eps32) / sb3
    else:
        den = np.sqrt(v) / sb3 + eps32
    upd = (m / (bc2 if mistake == "bc2_on_m" else bc1) + (b2 * n) / bc2) / den
    lw = lr32 * wd32
    if no_prox:
        p = p * (F(1) - lw) + (-lr32) * upd
    elif mistake == "prox_before_update":
        p = p / (F(1) + lw) + (-lr32) * upd
    else:
        p = (p + (-lr32) * upd) / (F(1) + lw)
    pre = g if mistake == "pre_unscaled" else x
    return {k: torch.from_numpy(np.ascontiguousarray(val, dtype=F)) for k, val in
            dict(p=p, m=m, n=n, v=v, pre=pre).items()}


def worst_share(o, got, r):
    worst = 0.0
    for k in ("p", "m", "n", "v", "pre"):
        err = (got[k].double() - getattr(r, k)).abs()
        tol = getattr(r, k + "_err")
        ratio = torch.where(err == 0, torch.zeros_like(err), err / tol)
        worst = max(worst, float(torch.nan_to_num(ratio, nan=float("inf")).max()))
    return worst


CONFIGS = [  # (t, lr, wd, no_prox, grad scale, share of first-step elements)
    (1, 1e-2, 0.05, False, None, 1.0),
    (2, 1e-2, 0.05, True, None, 0.0),
    (3, 2e-2, 0.3, False, 1 / 3.7, 0.5),
    (10, 5e-3, 0.0, False, 0.25, 0.0),
    (1000, 1e-3, 0.05, True, None, 0.0),
]


def operands(t, first_share, seed):
    o = A.sample_operands(4096, t, seed)
    first = (torch.arange(4096) % 8) < int(8 * first_share)
    return o, first


@pytest.mark.parametrize("cfg", CONFIGS, ids=[f"t{c[0]}" for c in CONFIGS])
def test_fp32_emulation_within_bounds(cfg):
    t, lr, wd, no_prox, s, fs = cfg
    o, first = operands(t, fs, seed=t)
    got = emulate(o, first=first.numpy(), t=t, lr=lr, wd=wd, no_prox=no_prox, s=s)
    r = A.adan_ref(o["p"], o["g"], o["m"], o["n"], o["v"], o["pre"], first=first, t=t, lr=lr, wd=wd, no_prox=no_prox,
                   grad_scale=s)
    for k in ("p", "m", "n", "v", "pre"):
        A.assert_within(got[k], getattr(r, k), getattr(r, k + "_err"), 1.0, torch.float32, what=k)
    # the bf16 rule: a bf16 parameter written from the emulated fp32 p' passes the bf16 check
    A.bf16_param_check(got["p"].bfloat16(), r.p, r.p_err)


MISTAKES = {  # mistake -> (t, lr, wd, no_prox, grad scale, share of first-step elements)
    "late_diff": (3, 1e-2, 0.05, False, None, 0.5),
    "param_step": (3, 1e-2, 0.05, False, None, 0.5),
    "swap_b2_b3": (2, 1e-2, 0.05, False, None, 0.0),
    "bc2_on_m": (2, 1e-2, 0.05, False, None, 0.0),
    "eps_before_div": (1, 1e-2, 0.05, False, None, 0.0),
    "prox_before_update": (2, 2e-2, 0.3, False, None, 0.0),
    "pre_unscaled": (2, 1e-2, 0.05, False, 1 / 3.7, 0.0),
    "one_minus_b2_in_u": (2, 1e-2, 0.05, False, None, 0.0),
}


@pytest.mark.parametrize("mistake", list(MISTAKES))
def test_planted_mistakes_exceed_a_bound_100_fold(mistake):
    t, lr, wd, no_prox, s, fs = MISTAKES[mistake]
    o, first = operands(t, fs, seed=7)
    if mistake in ("late_diff", "param_step"):        # a late parameter: its pre_grad was just allocated
        o["pre"] = torch.where(first, torch.zeros_like(o["pre"]), o["pre"])
    r = A.adan_ref(o["p"], o["g"], o["m"], o["n"], o["v"], o["pre"], first=first, t=t, lr=lr, wd=wd, no_prox=no_prox,
                   grad_scale=s)
    good = worst_share(o, emulate(o, first=first.numpy(), t=t, lr=lr, wd=wd, no_prox=no_prox, s=s), r)
    assert good <= 1.0
    if mistake == "param_step":                        # the per-parameter count differs from the group's only where late
        bad = emulate(o, first=first.numpy(), t=t, lr=lr, wd=wd, no_prox=no_prox, s=s, mistake=mistake)
        right = emulate(o, first=first.numpy(), t=t, lr=lr, wd=wd, no_prox=no_prox, s=s)
        bad = {k: torch.where(first, bad[k], right[k]) for k in bad}
    else:
        bad = emulate(o, first=first.numpy(), t=t, lr=lr, wd=wd, no_prox=no_prox, s=s, mistake=mistake)
    factor = worst_share(o, bad, r)
    print(f"{mistake}: {factor:.3g} x bound")
    assert factor >= 100, (mistake, factor)


# ---- FairseqAdan ----
def _cfg(**kw):
    base = dict(lr=[3e-4], adan_betas="(0.98,0.92,0.99)", adan_eps=1e-8, weight_decay=0.05, no_prox=False,
                fp16_adan_stats=False, tpu=False)
    base.update(kw)
    return SimpleNamespace(**base)


def _params():
    return [torch.nn.Parameter(torch.zeros(4)), torch.nn.Parameter(torch.zeros(3))]


def test_fairseq_adan_config():
    from one_peace_b200.optim import FairseqAdan
    ps = _params()
    opt = FairseqAdan(_cfg(), [{"params": ps[:1], "lr_scale": 0.5, "weight_decay": 0.05},
                               {"params": ps[1:], "lr_scale": 0.25, "weight_decay": 0.0}])
    assert opt.optimizer_config == {"lr": 3e-4, "betas": (0.98, 0.92, 0.99), "eps": 1e-8, "weight_decay": 0.05}
    g = opt.param_groups
    assert [x["betas"] for x in g] == [(0.98, 0.92, 0.99)] * 2 and [x["weight_decay"] for x in g] == [0.05, 0.0]
    assert all(x["no_prox"] is False for x in g)
    opt.set_lr(1e-3)                   # FairseqOptimizer.set_lr: lr_scale is ignored, as in the reference
    assert [x["lr"] for x in g] == [1e-3, 1e-3] and opt.get_lr() == 1e-3
    # sequence betas, scalar lr; no_prox in the config is not passed on (adan.py:89-98)
    opt2 = FairseqAdan(_cfg(lr=2e-4, adan_betas=[0.9, 0.9, 0.95], no_prox=True), _params())
    assert opt2.optimizer_config["betas"] == (0.9, 0.9, 0.95) and opt2.optimizer_config["lr"] == 2e-4
    assert opt2.param_groups[0]["no_prox"] is False and "no_prox" not in opt2.optimizer_config
    with pytest.raises(NotImplementedError):
        FairseqAdan(_cfg(fp16_adan_stats=True), _params())
    assert opt.optimizer.supports_memory_efficient_fp16 and opt.optimizer.supports_flat_params
    from one_peace_b200.optim import MemoryEfficientBF16Optimizer
    MemoryEfficientBF16Optimizer(opt)            # accepted as the wrapped optimizer


def test_registered_as_adan_and_the_yaml_swap():
    """`optimizer: {_name: adan, ...}` with user_dir = this package: fairseq looks the name up in its registry, fills the
    registered dataclass with the YAML's fields (lr interpolated from optimization.lr) and calls cls(cfg, params)."""
    import dataclasses

    from one_peace_b200 import fairseq_compat
    import one_peace_b200.user_module  # noqa: F401
    from one_peace_b200.optim.adan import FairseqAdan, FairseqAdanConfig
    if fairseq_compat.HAVE_FAIRSEQ:                                    # pragma: no cover
        from fairseq.optim import OPTIMIZER_REGISTRY as reg
    else:
        reg = fairseq_compat.REGISTRY
    assert reg["adan"] is FairseqAdan and reg["adjust_adam"].__name__ == "AdjustAdam"
    yaml = {"_name": "adan", "adan_betas": "(0.98,0.92,0.99)", "adan_eps": 1e-8, "weight_decay": 0.02}
    names = {f.name for f in dataclasses.fields(FairseqAdanConfig)}
    assert {"adan_betas", "adan_eps", "weight_decay", "no_prox", "fp16_adan_stats", "tpu", "lr"} <= names
    cfg = FairseqAdanConfig(**{k: v for k, v in yaml.items() if k != "_name"})
    cfg.lr, cfg.tpu = [5e-5], False                                    # optimization.lr / common.tpu
    opt = reg[yaml["_name"]](cfg, _params())
    g = opt.param_groups[0]
    assert g["lr"] == 5e-5 and g["betas"] == (0.98, 0.92, 0.99) and g["weight_decay"] == 0.02 and g["eps"] == 1e-8


def test_adan_refuses_cpu_parameters_and_mixed_betas():
    from one_peace_b200.optim import Adan
    p = torch.nn.Parameter(torch.zeros(3))
    p.grad = torch.ones(3)
    opt = Adan([p])
    with pytest.raises(RuntimeError):
        opt.step()
    assert "step" not in opt.param_groups[0]          # a refused step does not advance the group's count
    q = torch.nn.Parameter(torch.zeros(3))
    opt = Adan([{"params": [p]}, {"params": [q], "betas": (0.9, 0.9, 0.9)}])
    with pytest.raises(NotImplementedError):
        opt.step()


def test_adan_abi_refuses_bad_arguments_without_a_gpu():
    from one_peace_b200 import _lib
    lib = _lib.load()
    one = (ctypes.c_float * 1)(1.0)
    flag = (ctypes.c_int32 * 1)(0)
    fp = ctypes.cast(one, ctypes.c_void_p)
    ip = ctypes.cast(flag, ctypes.c_void_p)
    dummy = ctypes.c_void_p(16)            # never dereferenced: the checks run before any CUDA call

    def call(tensors=dummy, ct=dummy, co=dummy, lr=fp, wd=fp, np_=ip, b1=fp, b2=fp, b3=fp, n_groups=1):
        return lib.opb_adan_multi_step(tensors, ct, co, 1, lr, wd, np_, b1, b2, b3, n_groups, 0.98, 0.92, 0.99, 1e-8,
                                       None, None)
    for kw in ("tensors", "ct", "co", "lr", "wd", "np_", "b1", "b2", "b3"):
        assert call(**{kw: None}) == 1, kw                               # OPB_ERR_INVALID
    assert call(n_groups=0) == 3 and call(n_groups=129) == 3           # OPB_ERR_UNSUPPORTED
