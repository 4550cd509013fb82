"""GPU: the contract of the fused Adam step and the gradient norm (csrc/adam.cu) and of the optimizers built on them
(optim/adam.py, optim/distributed_adam.py, optim/fp16_optimizer_memory_efficent.py), element by element against the fp64
references of tests/kernel_ref.py (module docstring, "Optimizer").

Kernel-level tests build the tables with ``optim.adam._Table`` and call ``opb_adam_multi_step`` / ``opb_grad_norm_clip``
as ``adam.py`` does.  Every operand (p, g, m, v, the master copy) is a view into a NaN-filled buffer at its own element
offset (0, 1, 2, 4 for fp32; 0, 1, 4, 8 for bf16), so both the 16-byte vector path and the scalar path run, and a write
outside a tensor shows up.  Data: N(0, 0.3) gradients with every 4th in a band 1e-9 <= |g| <= 1e-6 (sqrt(v) comparable to
eps), every 16th gradient and state zero, m and v preset as t - 1 steps leave them (t = 1, 2, 10, 1000)."""
import ctypes
import math

import numpy as np
import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
CHUNK = R.ADAM_CHUNK
OFFS = {F32: [0, 1, 2, 4], BF16: [0, 1, 4, 8]}          # element offsets; 0 and 4 / 8 keep 16-byte alignment
ALIGNED = {F32: [0, 4], BF16: [0, 8]}
SIZES = [1, 3, 4, 5, 8191, 8192, 8193, 3 * 8192 + 7]
STEPS = [1, 2, 10, 1000]
GROUPS = [(1e-2, 0.05), (0.5 * 1e-3, 0.05), (1e-3, 0.0)]   # (lr * lr_scale, weight decay): layer-decayed, no-decay groups
EPS = 1e-8
OPERANDS = ("p", "g", "m", "v", "master")


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def ratios():
    """largest fraction of the bound used, per output (printed at the end of the module; run with -s)"""
    seen = {}
    yield seen
    print(f"\nbound used on {torch.cuda.get_device_name()}:")
    for k in sorted(seen):
        print(f"bound used: {k:<40s} {seen[k]:.3g}")


def note(ratios, family, r):
    ratios[family] = max(ratios.get(family, 0.0), r)


def bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def spec(n, p=F32, g=F32, master=False, group=0, t=1, off=None):
    return dict(n=n, p=p, g=g, master=master, group=group, t=t, off=off or {})


def offsets_for(j, s):
    """even j: every operand 16-byte aligned (vector path); odd j: offsets from the full list, some misaligned"""
    out = {}
    for k, op in enumerate(OPERANDS):
        dt = s["p"] if op == "p" else s["g"] if op == "g" else F32
        out[op] = ALIGNED[dt][(j // 2 + k) % 2] if j % 2 == 0 else OFFS[dt][(j + k) % 4]
    return out


def size_table(p, g, master):
    """every size twice (aligned, misaligned), spread over the three groups and the four step counts"""
    specs = []
    for j in range(2 * len(SIZES)):
        s = spec(SIZES[j // 2], p, g, master, group=j % 3, t=STEPS[(j // 2 + j) % 4])
        s["off"] = offsets_for(j, s)
        specs.append(s)
    return specs


class Table:
    """The tensors of ``specs`` as views into one NaN-filled buffer per (operand, dtype), each at its element offset with
    NaN gaps between them, filled from ``seed``.  ``lead`` moves every tensor by that many elements (a multiple of 64 keeps
    the alignment)."""

    def __init__(self, specs, betas, seed, lead=64, with_state=True):
        self.specs, self.betas = specs, betas
        cursor, self.pos = {}, []
        for s in specs:
            d = {}
            for op in OPERANDS:
                if op == "master" and not s["master"]:
                    continue
                if op != "g" and not with_state:
                    continue
                dt = s["p"] if op == "p" else s["g"] if op == "g" else F32
                c = cursor.get((op, dt), lead)
                start = c + s["off"].get(op, 0)
                d[op] = ((op, dt), start)
                cursor[(op, dt)] = (start + s["n"] + 64 + 63) // 64 * 64
            self.pos.append(d)
        n_log = sum(s["n"] for s in specs)
        self.lstart = np.cumsum([0] + [s["n"] for s in specs])
        dev = "cuda"
        # logical (concatenated) per-element attributes
        e = torch.from_numpy(np.concatenate([np.arange(s["n"]) for s in specs])).to(dev)
        tt = torch.from_numpy(np.concatenate([np.full(s["n"], s["t"]) for s in specs])).to(dev)
        self.tensor_of = torch.from_numpy(np.concatenate([np.full(s["n"], i) for i, s in enumerate(specs)])).to(dev)
        gen = torch.Generator(device=dev).manual_seed(seed)
        band, zero = e % 4 == 1, e % 16 == 3
        g = torch.randn(n_log, device=dev, generator=gen) * 0.3
        small = 10.0 ** (-9 + 3 * torch.rand(n_log, device=dev, generator=gen))
        g = torch.where(band, torch.sign(g) * small, g)
        b1, b2 = betas
        sc = torch.where(band, 1e-7, 0.3)
        h1 = torch.randn(n_log, device=dev, generator=gen) * sc
        h2 = torch.randn(n_log, device=dev, generator=gen) * sc
        ttd = tt.double()
        m = ((1 - b1 ** (ttd - 1)) * h1).float()
        v = ((1 - b2 ** (ttd - 1)) * h2 * h2).float()
        g, m, v = (torch.where(zero, 0.0, x) for x in (g, m, v))
        pv = torch.randn(n_log, device=dev, generator=gen)
        logical = {"g": g, "m": m, "v": v, "master": pv, "p": pv}
        self.bufs, self.idx = {}, {}
        for key, size in cursor.items():
            op, dt = key
            pos = [(start, i) for i, d in enumerate(self.pos) for o, (k, start) in d.items() if k == key]
            bi = np.concatenate([np.arange(st, st + specs[i]["n"]) for st, i in pos])
            li = np.concatenate([np.arange(self.lstart[i], self.lstart[i] + specs[i]["n"]) for _, i in pos])
            bi, li = torch.from_numpy(bi).to(dev), torch.from_numpy(li).to(dev)
            buf = torch.full((size + 64,), float("nan"), dtype=dt, device=dev)
            buf[bi] = logical[op][li].to(dt)
            self.bufs[key], self.idx[key] = buf, (bi, li)
        self.init = {k: b.clone() for k, b in self.bufs.items()}
        self.n_log = n_log

    def view(self, i, op):
        (key, start) = self.pos[i][op]
        return self.bufs[key][start:start + self.specs[i]["n"]]

    def logical(self, op, init=False):
        """fp64 values of operand ``op`` over all tensors that have it, in logical order (NaN where absent)"""
        out = torch.full((self.n_log,), float("nan"), dtype=torch.float64, device="cuda")
        for (o, _), (bi, li) in self.idx.items():
            if o == op:
                out[li] = (self.init if init else self.bufs)[(o, _)][bi].double()
        return out

    def vgroups(self):
        keys = list(dict.fromkeys((s["group"], s["t"]) for s in self.specs))
        return keys, [keys.index((s["group"], s["t"])) for s in self.specs]

    def entries(self):
        _, vg = self.vgroups()
        return [(self.view(i, "p"), self.view(i, "g"), self.view(i, "m"), self.view(i, "v"),
                 self.view(i, "master") if s["master"] else None, vg[i]) for i, s in enumerate(self.specs)]

    def grad_entries(self):
        return [(self.view(i, "g"),) * 4 + (None, 0) for i in range(len(self.specs))]


def adam_launch(lib, tab, eps=EPS, grad_scale=None):
    from one_peace_b200.optim.adam import _Table
    keys, _ = tab.vgroups()
    groups = [(GROUPS[gi][0], GROUPS[gi][1], R.bias_correction(t, tab.betas)) for gi, t in keys]
    tt = _Table()
    tt.build(tab.entries(), torch.device("cuda"))
    n = len(groups)
    arr = lambda k: ctypes.cast((ctypes.c_float * n)(*[x[k] for x in groups]), ctypes.c_void_p)
    st = lib.opb_adam_multi_step(tt.tensors.data_ptr(), tt.chunk_tensor.data_ptr(), tt.chunk_off.data_ptr(), tt.n_chunks,
                                 arr(0), arr(1), arr(2), n, tab.betas[0], tab.betas[1], eps,
                                 0 if grad_scale is None else grad_scale.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == 0
    torch.cuda.synchronize()


def norm_launch(lib, tab, mf, max_norm):
    from one_peace_b200.optim.adam import _Table
    tt = _Table()
    tt.build(tab.grad_entries(), torch.device("cuda"))
    out = torch.full((2,), float("nan"), device="cuda")
    st = lib.opb_grad_norm_clip(tt.tensors.data_ptr(), tt.chunk_tensor.data_ptr(), tt.chunk_off.data_ptr(), tt.n_chunks,
                                tt.partial.data_ptr(), float(mf), float(max_norm), out.data_ptr(),
                                torch.cuda.current_stream().cuda_stream)
    assert st == 0
    torch.cuda.synchronize()
    return out


def check_canaries(tab):
    """gradients untouched; outside the tensors every buffer still holds its NaN fill; inside, every state element finite"""
    for key, buf in tab.bufs.items():
        op, dt = key
        if op == "g":
            assert torch.equal(bits(buf), bits(tab.init[key])), "the gradients were written"
            continue
        bi, _ = tab.idx[key]
        inside = torch.zeros(buf.numel(), dtype=torch.bool, device="cuda")
        inside[bi] = True
        assert torch.equal(bits(buf)[~inside], bits(tab.init[key])[~inside]), f"{op} {dt}: written outside the tensors"
        assert torch.isfinite(buf[inside]).all(), f"{op} {dt}: an element was not written"


def check_step(tab, ratios, label, grad_scale=None, grad_scale_err=0.0):
    """every output element against adam_ref on the operands the kernel read"""
    keys, vg = tab.vgroups()
    vg_log = torch.tensor(vg, device="cuda")[tab.tensor_of]
    g0, m0, v0 = tab.logical("g", True), tab.logical("m", True), tab.logical("v", True)
    master0, p0 = tab.logical("master", True), tab.logical("p", True)
    has_master = torch.tensor([s["master"] for s in tab.specs], device="cuda")[tab.tensor_of]
    p_bf16 = torch.tensor([s["p"] == BF16 for s in tab.specs], device="cuda")[tab.tensor_of]
    pread = torch.where(has_master, master0, p0)
    ref = {k: torch.empty(tab.n_log, dtype=torch.float64, device="cuda") for k in ("m", "m_err", "v", "v_err", "p", "p_err")}
    for k, (gi, t) in enumerate(keys):
        sel = vg_log == k
        r = R.adam_ref(pread[sel], g0[sel], m0[sel], v0[sel], t=t, lr=GROUPS[gi][0], wd=GROUPS[gi][1], betas=tab.betas,
                       eps=EPS, grad_scale=grad_scale, grad_scale_err=grad_scale_err)
        for name in ref:
            ref[name][sel] = getattr(r, name)
    for op in ("m", "v"):
        note(ratios, f"{label} {op}", R.assert_within(tab.logical(op), ref[op], ref[op + "_err"], 1.0, F32, what=op))
    p32 = ~p_bf16
    if p32.any():
        note(ratios, f"{label} fp32 p", R.assert_within(tab.logical("p")[p32], ref["p"][p32], ref["p_err"][p32], 1.0, F32,
                                                        what="fp32 p"))
    if has_master.any():
        mst = tab.logical("master")
        note(ratios, f"{label} master", R.assert_within(mst[has_master], ref["p"][has_master], ref["p_err"][has_master], 1.0,
                                                        F32, what="master"))
        for i, s in enumerate(tab.specs):
            if s["master"]:
                assert torch.equal(bits(tab.view(i, "p")), bits(tab.view(i, "master").bfloat16())), "p16 != bf16(master)"
    nm = p_bf16 & ~has_master
    if nm.any():
        amb = R.bf16_param_check(tab.logical("p")[nm], ref["p"][nm], ref["p_err"][nm])
        note(ratios, f"{label} bf16 p: share with two allowed values", amb / int(nm.sum()))
    check_canaries(tab)


def run_twice(specs, betas, seed, launch):
    """two identical tables, one launch each: every buffer must match bit for bit"""
    a, b = Table(specs, betas, seed), Table(specs, betas, seed)
    launch(a)
    launch(b)
    for key in a.bufs:
        assert torch.equal(bits(a.bufs[key]), bits(b.bufs[key])), f"{key}: two launches differ"
    return a


PAIRS = [(F32, F32, False), (F32, BF16, False), (BF16, BF16, True), (BF16, BF16, False), (BF16, F32, True),
         (BF16, F32, False)]
PAIR_IDS = ["p32-g32", "p32-g16", "p16-g16-master", "p16-g16", "p16-g32-master", "p16-g32"]
BETAS = [(0.9, 0.98), (0.9, 0.999)]


def scale_for(lib, mode, specs, betas, seed):
    """-> (grad_scale device tensor or None, its value for the reference, norm check or None)"""
    if mode == "none":
        return None, None
    if mode == "clip":          # out[1] of opb_grad_norm_clip over the same gradients, clipping to 0.3 of the norm
        tab = Table(specs, betas, seed)
        grads = [tab.view(i, "g") for i in range(len(specs))]
        ref = R.grad_norm_ref(grads, 0.5)
        out = norm_launch(lib, tab, 0.5, 0.3 * ref.norm)
        full = R.grad_norm_ref(grads, 0.5, 0.3 * ref.norm)
        R.assert_within(out[1:].double().cpu(), torch.tensor([full.scale]), torch.tensor([full.scale_err]), 1.0, F32,
                        what="clip scale")
        return out[1:2].clone(), float(out[1])
    v = float(mode)
    return torch.full((1,), v, device="cuda"), v


@pytest.mark.parametrize("gs_mode", ["none", "1.0", "0.37", "clip"])
@pytest.mark.parametrize("betas", BETAS, ids=["b2=0.98", "b2=0.999"])
@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
def test_adam_kernel_contract(lib, ratios, pair, betas, gs_mode):
    specs = size_table(*pair)
    seed = 1000 * PAIRS.index(pair) + 10 * BETAS.index(betas)
    gs, gsv = scale_for(lib, gs_mode, specs, betas, seed)
    tab = run_twice(specs, betas, seed, lambda t: adam_launch(lib, t, grad_scale=gs))
    check_step(tab, ratios, PAIR_IDS[PAIRS.index(pair)], grad_scale=gsv)


def test_adam_kernel_mixed_table(lib, ratios):
    """all four (p, g) dtype pairs, with and without a master copy, in one table"""
    specs = []
    for k, pair in enumerate(PAIRS):
        for j in range(4):
            s = spec(SIZES[(2 * k + j) % len(SIZES)], *pair, group=(k + j) % 3, t=STEPS[(k + 2 * j) % 4])
            s["off"] = offsets_for(k + j, s)
            specs.append(s)
    gs = torch.full((1,), 0.37, device="cuda")
    tab = run_twice(specs, (0.9, 0.98), 77, lambda t: adam_launch(lib, t, grad_scale=gs))
    check_step(tab, ratios, "mixed", grad_scale=0.37)


def test_adam_kernel_large_tables(lib, ratios):
    """a 1100-chunk bf16 tensor with a master copy (vector path), then 1200 tiny tensors at misaligned offsets (scalar path)"""
    big = [spec(1100 * CHUNK, BF16, BF16, True, group=0, t=10)]
    tab = run_twice(big, (0.9, 0.98), 5, lambda t: adam_launch(lib, t))
    check_step(tab, ratios, "1100 chunks")
    del tab
    tiny = []
    for j in range(1200):
        s = spec(1 + j % 17, (F32, BF16)[j % 2], (F32, BF16)[(j // 2) % 2], j % 4 == 1, group=j % 3, t=STEPS[j % 4])
        s["off"] = offsets_for(2 * j + 1, s)
        tiny.append(s)
    gs = torch.full((1,), 0.37, device="cuda")
    tab = run_twice(tiny, (0.9, 0.999), 6, lambda t: adam_launch(lib, t, grad_scale=gs))
    check_step(tab, ratios, "1200 tiny", grad_scale=0.37)


# ---------------------------------------------------------------------------------------------------------------------
# gradient norm
# ---------------------------------------------------------------------------------------------------------------------
def check_norm(lib, ratios, specs, label, seed):
    tab = Table(specs, (0.9, 0.98), seed, with_state=False)
    grads = [tab.view(i, "g") for i in range(len(specs))]
    n0 = R.grad_norm_ref(grads, 1.0).norm
    # a second copy of the same gradients at other 16-byte-aligned addresses
    moved = Table(specs, (0.9, 0.98), seed, lead=64 * 37, with_state=False)
    for (key, b) in tab.bufs.items():
        bi, li = tab.idx[key]
        bm, lm = moved.idx[key]
        assert torch.equal(li, lm)
        moved.bufs[key][bm] = b[bi]
    for mf, mn in ((1.0, 0.0), (0.37, 0.0), (0.37, 0.5 * 0.37 * n0), (2.5, 2 * 2.5 * n0), (0.37, 0.37 * n0)):
        ref = R.grad_norm_ref(grads, mf, mn)
        out = norm_launch(lib, tab, mf, mn)
        d = lambda x: torch.tensor([x], dtype=torch.float64)
        note(ratios, "grad norm out[0]", R.assert_within(out[0:1].cpu(), d(ref.norm), d(ref.norm_err), 1.0, F32,
                                                         what=f"{label} norm"))
        note(ratios, "grad norm out[1]", R.assert_within(out[1:2].cpu(), d(ref.scale), d(ref.scale_err), 1.0, F32,
                                                         what=f"{label} grad_scale"))
        assert torch.equal(bits(out), bits(norm_launch(lib, tab, mf, mn))), f"{label}: repeated call differs"
        assert torch.equal(bits(out), bits(norm_launch(lib, moved, mf, mn))), f"{label}: moved gradients differ"
    assert all(torch.equal(bits(b), bits(tab.init[k])) for k, b in tab.bufs.items()), "the gradients were written"
    return ref


@pytest.mark.parametrize("dt", [F32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n_chunks", [1, 1055, 1056, 1057, 2113])
def test_grad_norm_chunk_counts(lib, ratios, n_chunks, dt):
    """one tensor whose last chunk is a 4000-element tail: CTAs own one chunk up to 1056 chunks, two past it"""
    n = 5000 if n_chunks == 1 else (n_chunks - 1) * CHUNK + 4000
    ref = check_norm(lib, ratios, [spec(n, dt, dt)], f"{n_chunks} chunks", n_chunks)
    assert ref.n_chunks == n_chunks and ref.grid == min(n_chunks, 1056)


def test_grad_norm_large_and_mixed_tables(lib, ratios):
    check_norm(lib, ratios, [spec(1100 * CHUNK, F32, F32)], "1100 chunks", 1)
    tiny = [spec(1 + j % 17, F32, (F32, BF16)[j % 2], off={"g": OFFS[(F32, BF16)[j % 2]][j % 4]}) for j in range(1200)]
    ref = check_norm(lib, ratios, tiny, "1200 tiny", 2)
    assert ref.n_chunks == 1200 and ref.grid == 1056
    mixed = [spec(n, g=(F32, BF16)[k % 2], off={"g": OFFS[(F32, BF16)[k % 2]][k % 4]}) for k, n in enumerate(SIZES * 2)]
    check_norm(lib, ratios, mixed, "mixed dtypes", 3)


@pytest.mark.parametrize("what", ["nan", "inf", "-inf", "nan+inf"])
def test_grad_norm_non_finite(lib, what):
    """NaN anywhere -> out[0] NaN and, with max_norm > 0, out[1] NaN (clamp(max=1) keeps it, as the reference and
    DistributedAdam do); +-inf and no NaN -> out[0] = +inf, out[1] = 0.  The bad values sit in a CTA's second chunk and in
    a bf16 tail."""
    specs = [spec(1057 * CHUNK, F32, F32), spec(CHUNK + 9, BF16, BF16, off={"g": 1})]
    tab = Table(specs, (0.9, 0.98), 9, with_state=False)
    big, small = tab.view(0, "g"), tab.view(1, "g")
    if what in ("nan", "nan+inf"):
        big[1056 * CHUNK + 77] = float("nan")
    if what in ("inf", "nan+inf"):
        small[CHUNK + 3] = float("inf")
    if what == "-inf":
        big[5] = float("-inf")
    for mf, mn in ((1.0, 1.0), (0.5, 0.0)):
        out = norm_launch(lib, tab, mf, mn).cpu()
        if "nan" in what:
            assert math.isnan(out[0]), out
            assert math.isnan(out[1]) if mn > 0 else out[1] == mf, out
        else:
            assert out[0] == float("inf"), out
            assert out[1] == 0.0 if mn > 0 else out[1] == mf, out


# ---------------------------------------------------------------------------------------------------------------------
# optimizers
# ---------------------------------------------------------------------------------------------------------------------
def snapshot(opt, params):
    """the operands the next step's kernel reads, per parameter with a gradient"""
    out = {}
    for p in params:
        if p.grad is None:
            continue
        st = opt.state[p]
        z = torch.zeros(p.shape, dtype=torch.float64, device=p.device)
        out[p] = dict(p=(st["master"] if "master" in st else p.detach()).double().clone(), g=p.grad.double().clone(),
                      m=st["exp_avg"].double().clone() if "exp_avg" in st else z,
                      v=st["exp_avg_sq"].double().clone() if "exp_avg_sq" in st else z, t=st.get("step", 0) + 1)
    return out


def check_module_step(ratios, label, opt, before, hyper, betas, gs=None, dgs=0.0):
    """hyper: p -> (lr, wd).  State and parameters after one step against adam_ref on the snapshot ``before``."""
    for p, b in before.items():
        lr, wd = hyper(p)
        r = R.adam_ref(b["p"], b["g"], b["m"], b["v"], t=b["t"], lr=lr, wd=wd, betas=betas, eps=EPS, grad_scale=gs,
                       grad_scale_err=dgs)
        st = opt.state[p]
        assert st["step"] == b["t"]
        note(ratios, f"{label} m", R.assert_within(st["exp_avg"], r.m, r.m_err, 1.0, F32, what=f"{label} m"))
        note(ratios, f"{label} v", R.assert_within(st["exp_avg_sq"], r.v, r.v_err, 1.0, F32, what=f"{label} v"))
        if "master" in st:
            note(ratios, f"{label} master", R.assert_within(st["master"], r.p, r.p_err, 1.0, F32, what=f"{label} master"))
            assert torch.equal(bits(p.detach()), bits(st["master"].bfloat16()))
        elif p.dtype == BF16:
            R.bf16_param_check(p.detach(), r.p, r.p_err, what=f"{label} bf16 p")
        else:
            note(ratios, f"{label} p", R.assert_within(p.detach(), r.p, r.p_err, 1.0, F32, what=f"{label} p"))


def test_adam_per_parameter_step_counts(lib, ratios):
    """a parameter that gets its first gradient later than its group-mates keeps its own bias correction (the reference
    tracks `step` per parameter, optim/adam.py:207-213); three steps, fp32 and bf16 parameters, against adam_ref"""
    from one_peace_b200.optim import Adam
    g = torch.Generator(device="cuda").manual_seed(4)
    for dt in (F32, BF16):
        pa = torch.nn.Parameter(torch.randn(300, device="cuda", generator=g).to(dt))
        pb = torch.nn.Parameter(torch.randn(37, 5, device="cuda", generator=g).to(dt))
        opt = Adam([pa, pb], lr=1e-2, betas=(0.9, 0.98), eps=EPS, weight_decay=0.05)
        for t in range(3):
            pa.grad = torch.randn(pa.shape, device="cuda", generator=g).to(dt)
            pb.grad = None if t == 0 else torch.randn(pb.shape, device="cuda", generator=g).to(dt)
            before = snapshot(opt, [pa, pb])
            opt.step()
            check_module_step(ratios, "Adam", opt, before, lambda p: (1e-2, 0.05), (0.9, 0.98))
        assert opt.state[pa]["step"] == 3 and opt.state[pb]["step"] == 2


def test_adam_virtual_group_limit(lib, ratios):
    """128 (param group, step count) combinations run; a 129th raises NotImplementedError before anything changes"""
    from one_peace_b200.optim import Adam
    g = torch.Generator(device="cuda").manual_seed(8)
    ps = [torch.nn.Parameter(torch.randn(5 + i % 7, device="cuda", generator=g)) for i in range(129)]
    opt = Adam([dict(params=[p], lr=1e-3 * (1 + i % 5), weight_decay=0.05 * (i % 2)) for i, p in enumerate(ps)],
               betas=(0.9, 0.999), eps=EPS)
    hyper = {p: (1e-3 * (1 + i % 5), 0.05 * (i % 2)) for i, p in enumerate(ps)}
    for i, p in enumerate(ps):
        p.grad = None if i == 128 else torch.randn(p.shape, device="cuda", generator=g)
    before = snapshot(opt, ps)
    opt.step()                                                  # 128 groups at t = 1
    check_module_step(ratios, "Adam", opt, before, hyper.get, (0.9, 0.999))
    for p in ps:
        p.grad = torch.randn(p.shape, device="cuda", generator=g)
    old = [p.detach().clone() for p in ps]
    with pytest.raises(NotImplementedError):
        opt.step()                                              # 128 groups at t = 2 and one at t = 1
    assert all(torch.equal(bits(p.detach()), bits(o)) for p, o in zip(ps, old))
    assert [opt.state[p].get("step", 0) for p in ps] == [1] * 128 + [0]


def test_adjust_adam_step_scale(lib, ratios):
    """AdjustAdam.step(scale=s) divides the gradients inside the kernel: grad_scale = fp32(1 / s)"""
    from one_peace_b200.optim import AdjustAdam
    g = torch.Generator(device="cuda").manual_seed(9)
    ps = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g)) for s in [(64, 33), (8193,), (1,)]]

    class Cfg:
        lr = [2e-3]; adam_betas = "(0.9, 0.98)"; adam_eps = EPS; weight_decay = 0.05
    fo = AdjustAdam(Cfg, [dict(params=ps[:2], weight_decay=0.05, lr_scale=0.5), dict(params=ps[2:], weight_decay=0.0)])
    fo.set_lr(2e-3)
    hyper = lambda p: (1e-3, 0.05) if any(p is q for q in ps[:2]) else (2e-3, 0.0)
    for scale in (3.0, 1.0, 0.7):
        for p in ps:
            p.grad = torch.randn(p.shape, device="cuda", generator=g)
        before = snapshot(fo.optimizer, ps)
        fo.step(scale=scale)
        s = 1.0 / scale
        check_module_step(ratios, "AdjustAdam", fo.optimizer, before, hyper, (0.9, 0.98), gs=s, dgs=abs(float(np.float32(s)) - s))


def test_adam_multi_tensor_groups_clip_and_master(lib, ratios):
    """bf16 parameters with fp32 master weights behind MemoryEfficientBF16Optimizer: multiply_grads and clip_grad_norm fold
    into one device grad_scale (two groups with lr_scale / no decay as utils/layer_decay.py builds them).  The norm and the
    scale against grad_norm_ref, every state element against adam_ref, p16 == bf16(master), a bit-identical norm on
    repeat."""
    from one_peace_b200.optim import AdjustAdam, MemoryEfficientBF16Optimizer
    g = torch.Generator(device="cuda").manual_seed(0)
    shapes = [(1536, 384), (1536,), (77,), (3, 5, 7), (8193,), (1,), (50000,)]
    params = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g).bfloat16()) for s in shapes]

    class Cfg:
        lr = [1e-2]; adam_betas = "(0.9, 0.98)"; adam_eps = EPS; weight_decay = 0.05; master_weights = True
    fo = AdjustAdam(Cfg, [dict(params=params[:3], weight_decay=0.05, lr_scale=0.5),
                          dict(params=params[3:], weight_decay=0.0, lr_scale=1.0)])
    fo.set_lr(1e-2)
    opt = MemoryEfficientBF16Optimizer(fo)
    hyper = lambda p: (5e-3, 0.05) if any(p is q for q in params[:3]) else (1e-2, 0.0)
    for max_norm in (1.0, 1.0, 1e6):                       # clipping, then a norm under the limit
        for p in params:
            p.grad = (torch.randn(p.shape, device="cuda", generator=g) * 0.3).bfloat16()
        opt.multiply_grads(0.5)
        norm = opt.clip_grad_norm(max_norm)
        ref = R.grad_norm_ref([p.grad for p in params], 0.5, max_norm)
        d = lambda x: torch.tensor([x], dtype=torch.float64)
        R.assert_within(norm.reshape(1).cpu(), d(ref.norm), d(ref.norm_err), 1.0, F32, what="norm")
        R.assert_within(opt._grad_scale.cpu(), d(ref.scale), d(ref.scale_err), 1.0, F32, what="grad_scale")
        before = snapshot(opt.optimizer, params)
        opt.step()
        check_module_step(ratios, "BF16Optimizer", opt.optimizer, before, hyper, (0.9, 0.98), gs=ref.scale, dgs=ref.scale_err)
    n1 = opt.optimizer.grad_norm_and_scale(1.0, 0.0)
    n2 = opt.optimizer.grad_norm_and_scale(1.0, 0.0)
    assert torch.equal(bits(n1), bits(n2))


def _dist_pair(dt, seed, sizes=((1536, 40), (77,), (8193,), (3, 5, 7), (1,))):
    from one_peace_b200.optim import Adam
    from one_peace_b200.optim.distributed_adam import DistributedAdam
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = [torch.randn(s, device="cuda", generator=g).to(dt) for s in sizes]
    pa = [torch.nn.Parameter(b.clone()) for b in base]
    pb = [torch.nn.Parameter(b.clone()) for b in base]
    groups = lambda ps: [dict(params=ps[:2], weight_decay=0.05, lr=5e-3), dict(params=ps[2:], weight_decay=0.0)]
    return (DistributedAdam(groups(pa), lr=1e-2, betas=(0.9, 0.98), eps=EPS), pa,
            Adam(groups(pb), lr=1e-2, betas=(0.9, 0.98), eps=EPS, master_weights=True), pb, g)


def _dist_state(da, i):
    off, n = da.offsets[i], da._plist[i][1].numel()
    sl = slice(off, off + n)
    out = dict(exp_avg=da.exp_avg[sl], exp_avg_sq=da.exp_avg_sq[sl])
    if da.master is not None:
        out["master"] = da.master[sl]
    return out


def _assert_flat_padding_untouched(da):
    """parameters are views into one flat buffer: the padding between them and the state there stay zero"""
    used = torch.zeros(da.total, dtype=torch.bool, device="cuda")
    for (_, p), off in zip(da._plist, da.offsets):
        used[off:off + p.numel()] = True
    for name, buf in (("flat_param", da.flat_param), ("exp_avg", da.exp_avg), ("exp_avg_sq", da.exp_avg_sq)):
        assert not buf[~used].any(), f"DistributedAdam wrote the padding of {name}"


@pytest.mark.parametrize("dt", [F32, BF16], ids=["fp32", "bf16"])
def test_distributed_adam_world1_matches_adam(lib, dt):
    """world size 1, no process group, no clipping: the same kernel on the same operands as Adam(master_weights=True), so
    parameters and state are bit-identical; the second parameter gets its first gradient at step 2"""
    da, pa, ad, pb, g = _dist_pair(dt, 21)
    for step in range(3):
        for i, (p, q) in enumerate(zip(pa, pb)):
            gr = None if (i == 1 and step == 0) else torch.randn(p.shape, device="cuda", generator=g).to(dt)
            p.grad = q.grad = gr
        da.step()
        ad.step()
        for i, (p, q) in enumerate(zip(pa, pb)):
            assert torch.equal(bits(p.detach()), bits(q.detach())), f"param {i} step {step}"
            for k, v in _dist_state(da, i).items():
                if k in ad.state[q]:
                    assert torch.equal(bits(v), bits(ad.state[q][k].reshape(-1))), f"{k} of param {i} step {step}"
                elif k != "master":         # no gradient yet: Adam has no state, the shard's moments are still zero
                    assert not v.any(), f"{k} of param {i} step {step}"
        _assert_flat_padding_untouched(da)
    assert da.steps == [3, 2, 3, 3, 3] and [ad.state[q]["step"] for q in pb] == [3, 2, 3, 3, 3]


def test_distributed_adam_late_gradient_bias_correction(lib, ratios):
    """a parameter whose first gradient comes at step 2 gets bias_corr(1) then bias_corr(2), as python Adam's per-parameter
    step count gives it (with one global count its first step was 0.74 of the correct size at betas (0.9, 0.98))"""
    from one_peace_b200.optim.distributed_adam import DistributedAdam
    g = torch.Generator(device="cuda").manual_seed(22)
    pa = torch.nn.Parameter(torch.randn(1000, device="cuda", generator=g))
    pb = torch.nn.Parameter(torch.randn(300, device="cuda", generator=g))
    da = DistributedAdam([pa, pb], lr=1e-2, betas=(0.9, 0.98), eps=EPS, weight_decay=0.05)
    st = {p: dict(m=torch.zeros(p.numel(), dtype=torch.float64, device="cuda"),
                  v=torch.zeros(p.numel(), dtype=torch.float64, device="cuda"), t=0) for p in (pa, pb)}
    for step in range(3):
        pa.grad = torch.randn(pa.shape, device="cuda", generator=g)
        pb.grad = None if step == 0 else torch.randn(pb.shape, device="cuda", generator=g)
        before = {p: (p.detach().double().clone(), p.grad.double().clone()) for p in (pa, pb) if p.grad is not None}
        da.step()
        for i, p in enumerate((pa, pb)):
            if p not in before:
                continue
            s = st[p]
            s["t"] += 1
            x, gr = before[p]
            r = R.adam_ref(x, gr, s["m"], s["v"], t=s["t"], lr=1e-2, wd=0.05, betas=(0.9, 0.98), eps=EPS, grad_scale=1.0)
            ds = _dist_state(da, i)
            note(ratios, "DistributedAdam p", R.assert_within(p.detach(), r.p, r.p_err, 1.0, F32, what=f"param {i} step {step}"))
            R.assert_within(ds["exp_avg"], r.m, r.m_err, 1.0, F32, what="m")
            R.assert_within(ds["exp_avg_sq"], r.v, r.v_err, 1.0, F32, what="v")
            s["m"], s["v"] = ds["exp_avg"].double().clone(), ds["exp_avg_sq"].double().clone()
    assert da.steps == [3, 2]


def test_distributed_adam_world1_clipping(lib, ratios):
    """with clipping, DistributedAdam's scale comes from fp32 torch ops on the kernel's norm (squared and rooted again, then
    max_norm * reciprocal): three fp32 roundings between the norm and the coefficient, two more on the norm"""
    for dt in (F32, BF16):
        da, pa, _, _, g = _dist_pair(dt, 23)
        for step in range(3):
            for p in pa:
                p.grad = (torch.randn(p.shape, device="cuda", generator=g) * 0.3).to(dt)
            before = {}
            for i, p in enumerate(pa):
                ds = _dist_state(da, i)
                before[p] = dict(p=(ds["master"] if "master" in ds else p.detach().reshape(-1)).double().clone(),
                                 g=p.grad.double().reshape(-1).clone(), m=ds["exp_avg"].double().clone(),
                                 v=ds["exp_avg_sq"].double().clone())
            r0 = R.grad_norm_ref([p.grad for p in pa], 1.0)
            norm_err = r0.norm_err + r0.norm * 1.5 * R.U32
            max_norm = 1.0 if step < 2 else 1e6
            gs, dgs = R.clip_scale_ref(r0.norm, norm_err, 1.0, max_norm, roundings=3)
            norm = da.step(max_norm=max_norm)
            d = lambda x: torch.tensor([x], dtype=torch.float64)
            R.assert_within(norm.reshape(1).cpu(), d(r0.norm), d(norm_err), 1.0, F32, what="norm")
            for i, p in enumerate(pa):
                b = before[p]
                lr, wd = (5e-3, 0.05) if i < 2 else (1e-2, 0.0)
                r = R.adam_ref(b["p"], b["g"], b["m"], b["v"], t=step + 1, lr=lr, wd=wd, betas=(0.9, 0.98), eps=EPS,
                               grad_scale=gs, grad_scale_err=dgs)
                ds = _dist_state(da, i)
                R.assert_within(ds["exp_avg"], r.m, r.m_err, 1.0, F32, what="m")
                R.assert_within(ds["exp_avg_sq"], r.v, r.v_err, 1.0, F32, what="v")
                if dt == BF16:
                    note(ratios, "DistributedAdam clipped master",
                         R.assert_within(ds["master"], r.p, r.p_err, 1.0, F32, what="master"))
                    assert torch.equal(bits(p.detach().reshape(-1)), bits(ds["master"].bfloat16()))
                else:
                    note(ratios, "DistributedAdam clipped p",
                         R.assert_within(p.detach().reshape(-1), r.p, r.p_err, 1.0, F32, what="p"))
            _assert_flat_padding_untouched(da)


@pytest.mark.parametrize("dt", [F32, BF16], ids=["fp32", "bf16"])
def test_distributed_adam_state_dict_round_trip(lib, dt):
    """state_dict after two steps (one parameter one step behind) into a fresh optimizer over the same parameter values,
    then one more step on both: bit-identical.  A checkpoint with the single `step` of earlier versions still loads."""
    from one_peace_b200.optim.distributed_adam import DistributedAdam
    da, pa, _, _, g = _dist_pair(dt, 24)
    grads = [[None if (i == 1 and s == 0) else torch.randn(p.shape, device="cuda", generator=g).to(dt)
              for i, p in enumerate(pa)] for s in range(3)]
    for s in range(2):
        for p, gr in zip(pa, grads[s]):
            p.grad = gr
        da.step()
    sd = da.state_dict()
    assert sd["distributed_adam"]["steps"] == [2, 1, 2, 2, 2]
    pc = [torch.nn.Parameter(p.detach().clone()) for p in pa]
    db = DistributedAdam([dict(params=pc[:2], weight_decay=0.05, lr=5e-3), dict(params=pc[2:], weight_decay=0.0)],
                         lr=1e-2, betas=(0.9, 0.98), eps=EPS)
    db.load_state_dict(sd)
    assert db.steps == da.steps
    for p, q, gr in zip(pa, pc, grads[2]):
        p.grad = gr.clone()
        q.grad = gr.clone()
    da.step()
    db.step()
    for name in ("flat_param", "exp_avg", "exp_avg_sq") + (("master",) if dt == BF16 else ()):
        assert torch.equal(bits(getattr(da, name)), bits(getattr(db, name))), name
    legacy = {"distributed_adam": {k: v for k, v in sd["distributed_adam"].items() if k != "steps"}, "param_groups": sd["param_groups"]}
    legacy["distributed_adam"]["step"] = 2
    db.load_state_dict(legacy)
    assert db.steps == [2] * 5
