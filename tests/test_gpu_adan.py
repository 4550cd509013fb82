"""GPU: the contract of the fused Adan step (``opb_adan_multi_step``, csrc/adam.cu) and of the optimizers built on it
(optim/adan.py), element by element against the fp64 reference of tests/adan_ref.py, and against tests/golden/adan.pt made
by the reference's own optim/adan.py.

Kernel-level tests build the table with ``optim.adam._Table(ADAN_LAYOUT)`` as ``Adan.step`` does.  Every operand (p, g, m,
n, v, pre_grad, the master copy) is a view into its own NaN-filled buffer at an element offset (0 or 4 / 8 keep 16-byte
alignment, 1, 2 or 1, 4 do not), so both the vector path and the scalar path run and a write outside a tensor shows up.
Under ``first`` pre_grad is NaN-filled: the kernel must not read it.  Data: adan_ref.sample_operands (a band of gradients
with sqrt(v) comparable to eps, zeros, moments preset as t - 1 steps leave them).  Run with -s for the largest share of
each bound."""
import ctypes
import os

import numpy as np
import pytest
import torch

import adan_ref as A
import restated_adan as restated

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
CHUNK = 8192
OPS = ("p", "g", "m", "n", "v", "pre", "master")
OFFS = {F32: [0, 1, 2, 4], BF16: [0, 1, 4, 8]}
SIZES = [1, 3, 4, 5, 8191, 8192, 8193, 3 * 8192 + 7]
GROUPS = [(1e-2, 0.05, 0), (5e-3, 0.0, 0), (2e-2, 0.3, 1), (1e-3, 0.05, 1)]     # (lr, wd, no_prox)
STEPS = [1, 2, 10, 1000]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adan.pt")


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def ratios():
    seen = {}
    yield seen
    print(f"\nAdan bound used on {torch.cuda.get_device_name()}:")
    for k in sorted(seen):
        print(f"bound used: {k:<44s} {seen[k]:.3g}")


def note(ratios, key, r):
    ratios[key] = max(ratios.get(key, 0.0), r)


def bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def op_dtype(s, op):
    return s["p"] if op == "p" else s["g"] if op == "g" else F32


class Tensors:
    """One Adan tensor record: every operand a view into its own NaN-filled buffer at offset ``off[op]``."""

    def __init__(self, s, seed, t):
        self.s = s
        o = A.sample_operands(s["n"], t, seed, device="cuda")
        self.bufs, self.views = {}, {}
        for k, op in enumerate(OPS):
            if op == "master" and not s["master"]:
                continue
            dt = op_dtype(s, op)
            off = OFFS[dt][(s["j"] + k) % 4] if s["j"] % 2 else (0 if (s["j"] // 2 + k) % 2 == 0 else OFFS[dt][3])
            buf = torch.full((off + s["n"] + 37,), float("nan"), dtype=dt, device="cuda")
            view = buf[off:off + s["n"]]
            src = o["p"] if op == "master" else o[op]
            if not (op == "pre" and s["first"]):
                view.copy_(src.to(dt))
            self.bufs[op], self.views[op] = buf, view
        if s["master"]:      # the bf16 parameter is the rounded master, as Adan keeps them
            self.views["p"].copy_(self.views["master"].to(s["p"]))
        self.init = {op: b.clone() for op, b in self.bufs.items()}

    def entry(self, gi):
        v = self.views
        return (v["p"], v["g"], v["m"], v["n"], v["v"], v["pre"], v.get("master"), gi, self.s["first"])

    def read(self, op):
        """fp64 values the kernel read (the initial contents)"""
        b = self.init[op]
        return b[self.views[op].storage_offset() - self.bufs[op].storage_offset():][:self.s["n"]].double()


def spec(n, p=F32, g=F32, master=False, group=0, first=False, j=0):
    return dict(n=n, p=p, g=g, master=master, group=group, first=first, j=j)


def launch(lib, tens, groups_t, grad_scale=None):
    """groups_t: [(lr, wd, no_prox, t)] per kernel group"""
    from one_peace_b200.optim.adam import _Table
    from one_peace_b200.optim.adan import ADAN_LAYOUT
    tab = _Table(ADAN_LAYOUT)
    tab.build([x.entry(x.s["group"]) for x in tens], torch.device("cuda"))
    n = len(groups_t)
    coefs = [A.group_coefs(t, A.BETAS) for *_, t in groups_t]
    f = lambda vals: ctypes.cast((ctypes.c_float * n)(*vals), ctypes.c_void_p)
    npx = ctypes.cast((ctypes.c_int32 * n)(*[g[2] for g in groups_t]), ctypes.c_void_p)
    st = lib.opb_adan_multi_step(tab.tensors.data_ptr(), tab.chunk_tensor.data_ptr(), tab.chunk_off.data_ptr(), tab.n_chunks,
                                 f([g[0] for g in groups_t]), f([g[1] for g in groups_t]), npx, f([c[0] for c in coefs]),
                                 f([c[1] for c in coefs]), f([c[2] for c in coefs]), n, *A.BETAS, A.EPS,
                                 0 if grad_scale is None else grad_scale.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == 0
    torch.cuda.synchronize()
    return tab


def check(tens, groups_t, ratios, label, gs=None, dgs=0.0, finite_only=False):
    """every output element against adan_ref on the operands the kernel read; canaries intact; gradients unwritten"""
    for x in tens:
        s = x.s
        lr, wd, no_prox, t = groups_t[s["group"]]
        pread = x.read("master") if s["master"] else x.read("p")
        pre = torch.zeros_like(pread) if s["first"] else x.read("pre")
        r = A.adan_ref(pread, x.read("g"), x.read("m"), x.read("n"), x.read("v"), pre, first=s["first"], t=t, lr=lr, wd=wd,
                       no_prox=bool(no_prox), grad_scale=gs, grad_scale_err=dgs)
        sel = torch.isfinite(r.p) if finite_only else slice(None)
        for op in ("m", "n", "v", "pre"):
            got = x.views[op]
            note(ratios, f"{label} {op}", A.assert_within(got[sel], getattr(r, op)[sel], getattr(r, op + "_err")[sel], 1.0,
                                                          F32, what=f"{label} {op}"))
        if s["master"]:
            note(ratios, f"{label} master", A.assert_within(x.views["master"][sel], r.p[sel], r.p_err[sel], 1.0, F32,
                                                            what=f"{label} master"))
            assert torch.equal(bits(x.views["p"]), bits(x.views["master"].to(s["p"]))), "p != bf16_rn(master)"
        elif s["p"] == BF16:
            amb = A.bf16_param_check(x.views["p"][sel], r.p[sel], r.p_err[sel], what=f"{label} bf16 p")
            note(ratios, f"{label} bf16 p: share with two allowed values", amb / max(s["n"], 1))
        else:
            note(ratios, f"{label} fp32 p", A.assert_within(x.views["p"][sel], r.p[sel], r.p_err[sel], 1.0, F32,
                                                            what=f"{label} fp32 p"))
        for op, buf in x.bufs.items():
            lo = x.views[op].storage_offset() - buf.storage_offset()
            outside = torch.ones(buf.numel(), dtype=torch.bool, device="cuda")
            outside[lo:lo + s["n"]] = False
            if op == "g":
                assert torch.equal(bits(buf), bits(x.init[op])), "the gradient was written"
            else:
                assert torch.equal(bits(buf)[outside], bits(x.init[op])[outside]), f"{op}: written outside the tensor"
                if not finite_only:
                    assert torch.isfinite(x.views[op]).all(), f"{op}: an element was not written"


PAIRS = [(F32, F32, False), (F32, BF16, False), (BF16, BF16, False), (BF16, BF16, True), (BF16, F32, False),
         (BF16, F32, True)]
PAIR_IDS = ["p32-g32", "p32-g16", "p16-g16", "p16-g16-master", "p16-g32", "p16-g32-master"]


def size_specs(p, g, master):
    """every size twice (aligned, misaligned), spread over the groups; every third tensor on its first step"""
    return [spec(SIZES[j // 2], p, g, master, group=j % len(GROUPS), first=j % 3 == 0, j=j) for j in range(2 * len(SIZES))]


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("t", STEPS)
@pytest.mark.parametrize("gs", [None, 0.37, 1 / 3.7])
def test_adan_kernel_contract(lib, ratios, pair, t, gs):
    specs = size_specs(*pair)
    tens = [Tensors(s, seed=100 * t + i, t=t) for i, s in enumerate(specs)]
    groups_t = [g + (t,) for g in GROUPS]
    scale = None if gs is None else torch.full((1,), gs, dtype=F32, device="cuda")
    launch(lib, tens, groups_t, scale)
    check(tens, groups_t, ratios, f"kernel {'-'.join(str(x) for x in pair)}", gs=gs)


def test_adan_kernel_mixed_table_and_repeat(lib, ratios):
    """all pairs in one table, with groups at different step counts; two launches on identical tables agree bit for bit"""
    specs = [spec(n, p, g, ms, group=k % 4, first=k % 5 == 0, j=k) for k, (n, (p, g, ms)) in
             enumerate(zip([7, 8192, 9000, 1, 16385, 333, 4096, 12], PAIRS + PAIRS[:2]))]
    groups_t = [GROUPS[0] + (3,), GROUPS[1] + (1,), GROUPS[2] + (10,), GROUPS[3] + (1000,)]
    runs = []
    for _ in range(2):
        tens = [Tensors(s, seed=7 + i, t=groups_t[s["group"]][3]) for i, s in enumerate(specs)]
        launch(lib, tens, groups_t)
        runs.append(tens)
    check(runs[0], groups_t, ratios, "mixed")
    for a, b in zip(*runs):
        for op in a.bufs:
            assert torch.equal(bits(a.bufs[op]), bits(b.bufs[op])), f"{op}: two launches differ"


def test_adan_kernel_large_tables(lib, ratios):
    """one tensor over 1000 chunks, and 1200 tiny tensors (1 to 40 elements) in 128 groups"""
    big = [Tensors(spec(1000 * CHUNK + 5, BF16, BF16, True, j=1), seed=1, t=2)]
    launch(lib, big, [GROUPS[0] + (2,)])
    check(big, [GROUPS[0] + (2,)], ratios, "1000 chunks")
    del big
    groups_t = [(1e-3 * (1 + i % 5), 0.05 * (i % 2), i % 3 == 0, 1 + i % 4) for i in range(128)]
    tiny = [Tensors(spec(1 + i % 40, PAIRS[i % 6][0], PAIRS[i % 6][1], PAIRS[i % 6][2], group=i % 128, first=i % 7 == 0,
                         j=i), seed=i, t=groups_t[i % 128][3]) for i in range(1200)]
    launch(lib, tiny, groups_t)
    check(tiny, groups_t, ratios, "1200 tiny")


@pytest.mark.parametrize("what", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("first", [False, True])
def test_adan_kernel_non_finite(lib, what, first):
    """a non-finite gradient poisons its own element as in the reference's torch arithmetic (a first step computes g - g);
    every other element stays within its bound"""
    s = spec(3 * CHUNK + 5, F32, F32, False, first=first, j=0)
    x = Tensors(s, seed=3, t=2)
    bad = [5, CHUNK + 3, 3 * CHUNK + 4]
    x.views["g"][bad] = float(what)
    x.init["g"].copy_(x.bufs["g"])
    groups_t = [GROUPS[0] + (2,)]
    launch(lib, [x], groups_t)
    check([x], groups_t, {}, "non-finite", finite_only=True)
    g = x.read("g")[bad]
    pre = g if first else x.read("pre")[bad]
    d = g - pre
    for op in ("m", "n", "v", "p", "pre"):
        got = x.views[op][bad].double()
        ref = {"m": 0.98 * x.read("m")[bad] + 0.02 * g, "n": 0.92 * x.read("n")[bad] + 0.08 * d,
               "pre": g}.get(op)
        if op == "v":                                          # +inf, or NaN where diff is
            assert (~torch.isfinite(got)).all(), (op, got)
            continue
        if op == "p":                                          # (+-inf) / inf or NaN
            assert torch.isnan(got).all(), (op, got)
            continue
        assert torch.equal(torch.isnan(got), torch.isnan(ref)) and torch.equal(got[~torch.isnan(got)], ref[~torch.isnan(ref)]), \
            (op, got, ref)


# ---------------------------------------------------------------------------------------------------------------------
# optimizers
# ---------------------------------------------------------------------------------------------------------------------
def golden():
    return torch.load(GOLDEN, weights_only=False)


def build(fx, case, cls="Adan", master=False):
    from one_peace_b200.optim import Adan, FairseqAdan
    c = fx["cases"][case]
    params = {k: torch.nn.Parameter(v.clone().cuda()) for k, v in c["p0"].items()}
    groups = [dict(params=[params[k] for k in gr["names"]], lr=gr["lr"], weight_decay=gr["weight_decay"])
              for gr in fx["groups"]]
    if cls == "Adan":
        opt = Adan(groups, betas=fx["betas"], eps=fx["eps"], no_prox=c["no_prox"], master_weights=master)
        return params, opt, opt
    from types import SimpleNamespace
    cfg = SimpleNamespace(lr=[fx["groups"][0]["lr"]], adan_betas=str(fx["betas"]), adan_eps=fx["eps"], weight_decay=0.05,
                          no_prox=False, fp16_adan_stats=False, tpu=False)
    fo = FairseqAdan(cfg, groups)
    return params, fo, fo.optimizer


def feed(params, c, t):
    for k, q in params.items():
        gk = c["grads"][t - 1][k]
        q.grad = None if gk is None else gk.clone().cuda()


def close(got, want, what):
    got, want = got.detach().cpu(), want.detach().cpu()
    if want.dtype == BF16:
        torch.testing.assert_close(got.float(), want.float(), rtol=2 ** -7, atol=1e-30, msg=what)
    else:
        torch.testing.assert_close(got, want, rtol=2e-5, atol=1e-6, msg=what)


@pytest.mark.parametrize("case", ["fp32_prox", "fp32_noprox", "bf16_prox", "bf16_noprox", "scaled"])
@pytest.mark.parametrize("cls", ["Adan", "FairseqAdan"])
def test_golden_trajectories(lib, case, cls):
    fx = golden()
    c = fx["cases"][case]
    if cls == "FairseqAdan" and c["no_prox"]:
        pytest.skip("FairseqAdan never passes no_prox (the reference's optimizer_config)")
    params, outer, opt = build(fx, case, cls)
    for t in range(1, fx["steps"] + 1):
        feed(params, c, t)
        if c["scale"] is None:
            outer.step()
        elif cls == "Adan":
            opt.step(grad_scale=torch.full((1,), c["scale"], dtype=F32, device="cuda"))
        else:
            outer.step(scale=1.0 / c["scale"])
        for k, q in params.items():
            close(q, c["traj"][t - 1][k], f"{case} {cls} step {t} {k}")
    assert [g["step"] for g in opt.param_groups] == c["group_steps"]
    for k, st in c["state"].items():
        for name, want in st.items():
            close(opt.state[params[k]][name], want, f"{case} {cls} {k} {name}")


def test_reference_state_dict_loads_and_training_continues(lib):
    fx = golden()
    c = fx["cases"]["resume"]
    params, _, opt = build(fx, "resume")
    with torch.no_grad():
        for k, q in params.items():
            q.copy_(c["traj"][c["resume_after"] - 1][k].cuda())
    opt.load_state_dict(c["state_dict"])
    assert [g["step"] for g in opt.param_groups] == [c["resume_after"]] * 2
    for st in opt.state.values():
        assert all(st[n].dtype == F32 and st[n].is_cuda for n in ("exp_avg", "exp_avg_diff", "exp_avg_sq", "pre_grad"))
    for t in range(c["resume_after"] + 1, fx["steps"] + 1):
        feed(params, c, t)
        opt.step()
        for k, q in params.items():
            close(q, c["traj"][t - 1][k], f"resume step {t} {k}")
    sd = opt.state_dict()                  # and our own state dict round-trips
    params2, _, opt2 = build(fx, "resume")
    opt2.load_state_dict(sd)
    assert opt2.param_groups[0]["step"] == fx["steps"]


def test_bf16_optimizer_with_clipping(lib, ratios):
    """MemoryEfficientBF16Optimizer(FairseqAdan): multiply_grads and clip_grad_norm fold into one device grad_scale; every
    state element against adan_ref with that scale, bf16 parameters with master weights (p16 == bf16_rn(master))"""
    from types import SimpleNamespace

    import kernel_ref as R
    from one_peace_b200.optim import FairseqAdan, MemoryEfficientBF16Optimizer
    gen = torch.Generator(device="cuda").manual_seed(0)
    shapes = [(1536, 384), (77,), (3, 5, 7), (8193,), (1,)]
    params = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=gen).bfloat16()) for s in shapes]
    cfg = SimpleNamespace(lr=[1e-2], adan_betas=(0.98, 0.92, 0.99), adan_eps=1e-8, weight_decay=0.05, no_prox=False,
                          fp16_adan_stats=False, tpu=False, master_weights=True)
    fo = FairseqAdan(cfg, [dict(params=params[:2], weight_decay=0.05), dict(params=params[2:], weight_decay=0.0)])
    opt = MemoryEfficientBF16Optimizer(fo)
    wd_of = lambda p: 0.05 if any(p is q for q in params[:2]) else 0.0
    for t, max_norm in enumerate((1.0, 1.0, 1e6), start=1):
        for p in params:
            p.grad = (torch.randn(p.shape, device="cuda", generator=gen) * 0.3).bfloat16()
        opt.multiply_grads(0.5)
        opt.clip_grad_norm(max_norm)
        ref = R.grad_norm_ref([p.grad for p in params], 0.5, max_norm)
        before = {}
        for p in params:
            st = fo.optimizer.state[p]
            z = torch.zeros(p.shape, dtype=torch.float64, device="cuda")
            before[p] = dict(p=(st["master"] if "master" in st else p.detach()).double().clone(), g=p.grad.double().clone(),
                             **{k: st[k].double().clone() if k in st else z for k in ("exp_avg", "exp_avg_diff",
                                                                                   "exp_avg_sq", "pre_grad")})
        opt.step()
        for p, b in before.items():
            r = A.adan_ref(b["p"], b["g"], b["exp_avg"], b["exp_avg_diff"], b["exp_avg_sq"], b["pre_grad"], first=t == 1, t=t,
                           lr=1e-2, wd=wd_of(p), no_prox=False, grad_scale=ref.scale, grad_scale_err=ref.scale_err)
            st = fo.optimizer.state[p]
            for name, op in (("exp_avg", "m"), ("exp_avg_diff", "n"), ("exp_avg_sq", "v"), ("pre_grad", "pre"), ("master", "p")):
                note(ratios, f"BF16Optimizer {op}", A.assert_within(st[name], getattr(r, op), getattr(r, op + "_err"), 1.0, F32,
                                                                    what=f"BF16Optimizer {name}"))
            assert torch.equal(bits(p.detach()), bits(st["master"].bfloat16()))


def test_classify_fine_tuning_through_adan(lib):
    """a tiny one_peace_classify, three steps through the registered `adan`: the parameters match restated.adan_step applied
    to the same gradients (fp32 model, so the gradients are the ones the kernel read)"""
    import synth
    import synth_classify as sc
    from one_peace_b200 import fairseq_compat
    from one_peace_b200.criterions import ClassifyCriterion
    from one_peace_b200.one_peace.hub_interface import from_pretrained
    from types import SimpleNamespace
    T = sc.CLASSIFY_TINY
    sd = synth.make_state_dict(**T, modalities=("text",), seed=4)
    hub = from_pretrained(model_type="one_peace_classify", state_dict=sd, head_type="text", layers=T["layers"],
                          embed_dim=T["embed_dim"], ffn_embed_dim=T["ffn"], attention_heads=T["heads"], patch_image_size=224,
                          device="cuda", dtype="float32", num_classes=2, use_two_images=False, use_pooler=False,
                          use_image_features=False)
    m = hub.model
    m.train()
    for p in m.parameters():
        p.requires_grad_(True)
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(4, 50000, (8, 12), generator=g)
    sample = {"net_input": {"src_tokens": tok.cuda()}, "target": (torch.arange(8) % 2).cuda(), "nsentences": 8}
    named = [(n, p) for n, p in m.named_parameters()]
    groups = [dict(params=[p for n, p in named if p.ndim > 1], weight_decay=0.05),
              dict(params=[p for n, p in named if p.ndim <= 1], weight_decay=0.0)]
    cfg = SimpleNamespace(lr=[1e-3], adan_betas="(0.98,0.92,0.99)", adan_eps=1e-8, weight_decay=0.05, no_prox=False,
                          fp16_adan_stats=False, tpu=False)
    reg = fairseq_compat.REGISTRY if not fairseq_compat.HAVE_FAIRSEQ else __import__("fairseq.optim").optim.OPTIMIZER_REGISTRY
    opt = reg["adan"](cfg, groups)
    crit = ClassifyCriterion(task=None)
    shadow = {id(p): dict(p=p.detach().float().cpu().clone(), m=None) for _, p in named}
    for t in range(1, 4):
        m.zero_grad(set_to_none=True)
        loss, n, _ = crit(m, sample)
        (loss / n).backward()
        for gi, gr in enumerate(groups):
            wd = gr["weight_decay"]
            for p in gr["params"]:
                if p.grad is None:
                    continue
                s = shadow[id(p)]
                gg = p.grad.detach().float().cpu().clone()
                if s["m"] is None:
                    s.update(m=torch.zeros_like(gg), n=torch.zeros_like(gg), v=torch.zeros_like(gg), pre=None)
                s["pre"] = restated.adan_step(s["p"], gg, s["m"], s["n"], s["v"], s["pre"], t, 1e-3, (0.98, 0.92, 0.99),
                                              1e-8, wd)
        opt.step()
        assert torch.isfinite(loss)
    worst = 0.0
    for name, p in named:
        want = shadow[id(p)]["p"]
        err = (p.detach().cpu() - want).abs().max().item()
        worst = max(worst, err)
        torch.testing.assert_close(p.detach().cpu(), want, rtol=1e-5, atol=2e-6, msg=name)
    print(f"\nclassify through adan: worst parameter difference to the restatement {worst:.3g}")
