"""Multi-scale deformable attention on the GPU: the kernels' contract against the fp64 reference (tests/msda_ref.py), the
module against the reference module's fixture, the kernels against the reference's own compiled op (when
oracle/_ref/ holds it), and the module at the recipe shapes against an fp32 torch restatement."""
import ctypes
import glob
import importlib.machinery
import importlib.util
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import msda_ref as R  # noqa: E402
from kernel_ref import assert_within  # noqa: E402

pytestmark = pytest.mark.gpu

# name -> (N, Lq, H, level shapes, P, L_ref, offset scale in pixels)
TINY = {
    "one_level": (1, 5, 1, [(3, 4)], 4, 1, 2.0),
    "three_levels_shared_ref": (2, 9, 2, [(6, 5), (3, 4), (2, 3)], 4, 1, 3.0),
    "per_level_ref": (1, 7, 3, [(4, 4), (2, 2)], 8, 2, 3.0),
    "four_levels_p1": (1, 33, 1, [(5, 7), (3, 3), (2, 1), (1, 1)], 1, 4, 1.5),
}
RECIPE = {   # 896^2, N = 1
    "injector": (1, 3136, 24, [(112, 112), (56, 56), (28, 28)], 4, 1, 2.0),
    "extractor": (1, 16464, 24, [(56, 56)], 4, 1, 2.0),
    "pixel_decoder": (1, 16464, 32, [(112, 112), (56, 56), (28, 28)], 4, 3, 2.0),
}
CHUNK = 1024


def _K():
    from one_peace_b200 import kernels as K
    return K


def _canary(rows, cols, dtype):
    buf = torch.full((rows + 2, cols), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[1:-1]


def _run(c):
    K = _K()
    N, Lq, H, P = c["N"], c["Lq"], c["H"], c["P"]
    value, proj, ref, d_out = c["value"], c["proj"], c["ref"], c["d_out"]
    obuf, out = _canary(N * Lq, H * 32, torch.bfloat16)
    K.ms_deform_attn_fwd(value, proj, ref, c["shapes"], c["starts"], N, Lq, H, P, out=out)
    vbuf = torch.full((value.shape[0] + 2, H * 32), float("nan"), dtype=torch.float32, device="cuda")
    vbuf[1:-1].zero_()
    pbuf, dp = _canary(proj.shape[0], proj.shape[1], torch.float32)
    K.ms_deform_attn_bwd(value, proj, ref, d_out, c["shapes"], c["starts"], N, Lq, H, P, d_value=vbuf[1:-1], d_proj=dp)
    torch.cuda.synchronize()
    for buf, what in ((obuf, "out"), (vbuf, "d_value"), (pbuf, "d_proj")):
        assert torch.isnan(buf[0]).all() and torch.isnan(buf[-1]).all(), f"{what}: canary row overwritten"
        assert not torch.isnan(buf[1:-1]).any(), f"{what}: element not written"
    return out.clone(), vbuf[1:-1].clone(), dp.clone()


def _check_contract(name, c):
    out, dv, dp = _run(c)
    out2, _, dp2 = _run(c)
    assert torch.equal(out, out2), "forward repeats differ"
    assert torch.equal(dp, dp2), "d_proj repeats differ"
    N, Lq, H, P = c["N"], c["Lq"], c["H"], c["P"]
    shares = {"out": 0.0, "d_proj": 0.0}
    if N == 1 and Lq > CHUNK:
        acc = {}
        for r0 in range(0, Lq, CHUNK):
            r1 = min(Lq, r0 + CHUNK)
            sl = slice(r0, r1)
            want, b = R.forward(c["value"], c["proj"][sl], c["ref"][sl], c["shapes"], c["starts"], 1, r1 - r0, H, P,
                                with_bound=True)
            shares["out"] = max(shares["out"], assert_within(out[sl], want, b, 1.0, torch.bfloat16, what=f"{name} out"))
            res = R.backward(c["value"], c["proj"][sl], c["ref"][sl], c["d_out"][sl], c["shapes"], c["starts"], 1, r1 - r0,
                             H, P, with_bound=True, acc=acc)
            shares["d_proj"] = max(shares["d_proj"], assert_within(dp[sl], res[1], res[3], 1.0, torch.float32,
                                                                   what=f"{name} d_proj"))
            del want, b
        want_dv, b_dv = res[0], res[2]
    else:
        want, b = R.forward(c["value"], c["proj"], c["ref"], c["shapes"], c["starts"], N, Lq, H, P, with_bound=True)
        shares["out"] = assert_within(out, want, b, 1.0, torch.bfloat16, what=f"{name} out")
        want_dv, want_dp, b_dv, b_dp = R.backward(c["value"], c["proj"], c["ref"], c["d_out"], c["shapes"], c["starts"], N,
                                                  Lq, H, P, with_bound=True)
        shares["d_proj"] = assert_within(dp, want_dp, b_dp, 1.0, torch.float32, what=f"{name} d_proj")
    shares["d_value"] = assert_within(dv, want_dv, b_dv, 1.0, torch.float32, what=f"{name} d_value")
    print(f"{name}: largest share of the bound: " + ", ".join(f"{k} {v:.3f}" for k, v in shares.items()))


@pytest.mark.parametrize("name", sorted(TINY))
def test_kernel_contract_tiny(name):
    N, Lq, H, shapes, P, L_ref, off = TINY[name]
    _check_contract(name, R.contract_case(N, Lq, H, shapes, P, L_ref, off, seed=len(name), device="cuda"))


@pytest.mark.parametrize("name", sorted(RECIPE))
def test_kernel_contract_recipe_shapes(name):
    N, Lq, H, shapes, P, L_ref, off = RECIPE[name]
    _check_contract(name, R.contract_case(N, Lq, H, shapes, P, L_ref, off, seed=len(name), device="cuda"))
    torch.cuda.empty_cache()


def test_at_a_cell_crossing():
    """Samples exactly on integer pixel coordinates: the forward within its bound, each offset gradient equal to one of
    the two one-sided derivatives."""
    shapes, N, Lq, H, P = [(4, 8)], 1, 6, 1, 4
    c = R.contract_case(N, Lq, H, shapes, P, 1, 0.0, seed=3, device="cuda")
    # off = 0 and ref = (k + 0.5) / W: px = k exactly in fp32 (W, H powers of two)
    k = torch.arange(Lq * 2, device="cuda").view(Lq, 1, 2).float() % 3
    c["ref"] = ((k + 0.5) / torch.tensor([8.0, 4.0], device="cuda")).contiguous()
    c["proj"][:, :2 * H * P] = 0.0
    out, dv, dp = _run(c)
    want, b = R.forward(c["value"], c["proj"], c["ref"], shapes, c["starts"], N, Lq, H, P, with_bound=True)
    assert_within(out, want, b, 1.0, torch.bfloat16, what="out at crossings")
    _, right, _, b_r = R.backward(c["value"], c["proj"], c["ref"], c["d_out"], shapes, c["starts"], N, Lq, H, P,
                                  with_bound=True)
    _, left, _, b_l = R.backward(c["value"], c["proj"], c["ref"], c["d_out"], shapes, c["starts"], N, Lq, H, P, left=True,
                                 with_bound=True)
    n_off = 2 * H * P
    g = dp[:, :n_off].double()
    ok = ((g - right[:, :n_off]).abs() <= b_r[:, :n_off]) | ((g - left[:, :n_off]).abs() <= b_l[:, :n_off])
    assert ok.all(), "an offset gradient at a crossing matches neither one-sided derivative"


def test_invalid_arguments():
    from one_peace_b200 import _lib
    lib = _lib.load()
    c = R.contract_case(1, 4, 1, [(2, 3)], 4, 1, 1.0, seed=0, device="cuda")
    out = torch.empty(4, 32, dtype=torch.bfloat16, device="cuda")
    dv = torch.zeros(6, 32, device="cuda")
    dp = torch.empty_like(c["proj"])
    hw = (ctypes.c_int32 * 2)(2, 3)
    st = (ctypes.c_int32 * 1)(0)
    s = torch.cuda.current_stream().cuda_stream
    v, p, r, g = c["value"].data_ptr(), c["proj"].data_ptr(), c["ref"].data_ptr(), c["d_out"].data_ptr()

    def fwd(D=32, L=1, P=4, v=v, o=out.data_ptr(), hw=hw):
        return lib.opb_ms_deform_attn_fwd(v, p, r, o, 1, 6, 4, 1, D, L, P, 1, hw, st, s)

    def bwd(D=32, L=1, P=4, v=v, d=dv.data_ptr()):
        return lib.opb_ms_deform_attn_bwd(v, p, r, g, d, dp.data_ptr(), 1, 6, 4, 1, D, L, P, 1, hw, st, s)
    assert fwd() == 0 and bwd() == 0
    for kw in (dict(D=16), dict(D=64), dict(L=0), dict(L=5), dict(P=0), dict(P=9), dict(v=0), dict(v=v + 2),
               dict(o=0), dict(o=out.data_ptr() + 8), dict(hw=None)):
        assert fwd(**kw) == 1, kw
    for kw in (dict(D=16), dict(L=5), dict(P=9), dict(v=0), dict(v=v + 2), dict(d=0), dict(d=dv.data_ptr() + 4)):
        assert bwd(**kw) == 1, kw
    big = (ctypes.c_int32 * 2)(3, 3)      # a level larger than S_in
    assert fwd(hw=big) == 1
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the module
# ---------------------------------------------------------------------------------------------------------------------
def _cos(a, b):
    return F.cosine_similarity(a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten(), dim=0).item()


@pytest.mark.parametrize("case", ["extractor", "injector", "per_level_n2"])
def test_module_matches_reference_fixture(case):
    from one_peace_b200.vision.ms_deform_attn import MSDeformAttn
    c = torch.load(os.path.join(HERE, "golden", "msda.pt"))["cases"][case]
    m = MSDeformAttn(**c["config"]).cuda()
    m.load_state_dict(c["state"])
    q = c["query"].cuda().requires_grad_(True)
    x = c["input_flatten"].cuda().requires_grad_(True)
    sp = torch.tensor(c["shapes"], device="cuda")
    y = m(q, c["reference_points"].cuda(), x, sp, torch.tensor(c["starts"], device="cuda"))
    (y * c["cotangent"].cuda()).sum().backward()
    cos = {"output": _cos(y, c["output"]), "d_query": _cos(q.grad, c["d_query"]),
           "d_input_flatten": _cos(x.grad, c["d_input_flatten"])}
    for k, p in m.named_parameters():
        cos[k] = _cos(p.grad, c["grads"][k])
    print(case, " ".join(f"{k} {v:.5f}" for k, v in cos.items()))
    assert y.dtype == torch.float32
    assert cos["output"] > 0.9995
    assert min(cos.values()) > 0.995, cos


def _ref_op():
    hits = sorted(glob.glob(os.path.join(ROOT, "oracle", "_ref", "MultiScaleDeformableAttention*.so")))
    if not hits:
        pytest.skip("oracle/_ref/MultiScaleDeformableAttention*.so is absent (built by oracle/build_ref_msda.py)")
    loader = importlib.machinery.ExtensionFileLoader("MultiScaleDeformableAttention", hits[0])
    spec = importlib.util.spec_from_loader("MultiScaleDeformableAttention", loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("name", ["three_levels_shared_ref", "per_level_ref", "injector"])
def test_against_reference_compiled_op(name):
    MSDA = _ref_op()
    N, Lq, H, shapes, P, L_ref, off = {**TINY, **RECIPE}[name]
    c = R.contract_case(N, Lq, H, shapes, P, L_ref, off, seed=7, device="cuda")
    L = len(shapes)
    S_in = c["value"].shape[0] // N
    out, dv, dp = _run(c)
    # the same locations and weights, formed in fp32 as the reference module forms them
    pr = c["proj"].view(N, Lq, -1)
    offs = pr[..., :2 * H * L * P].reshape(N, Lq, H, L, P, 2)
    attn = torch.softmax(pr[..., 2 * H * L * P:].reshape(N, Lq, H, L * P), -1).view(N, Lq, H, L, P)
    sp = torch.tensor(shapes, dtype=torch.long, device="cuda")
    norm = torch.stack([sp[:, 1], sp[:, 0]], -1)
    r = c["ref"].view(N, Lq, L_ref, 2)
    loc = (r[:, :, None, :, None, :] + offs / norm[None, None, None, :, None, :]).contiguous()
    start = torch.tensor(c["starts"], dtype=torch.long, device="cuda")
    value = c["value"].float().view(N, S_in, H, 32).contiguous()
    ref_out = MSDA.ms_deform_attn_forward(value, sp, start, loc, attn.contiguous(), 64)
    g = c["d_out"].float().view(N, Lq, H * 32).contiguous()
    ref_dv, ref_dloc, ref_dattn = MSDA.ms_deform_attn_backward(value, sp, start, loc, attn.contiguous(), g, 64)
    want, b = R.forward(c["value"], c["proj"], c["ref"], shapes, c["starts"], N, Lq, H, P, with_bound=True)
    _, _, b_dv, b_dp = R.backward(c["value"], c["proj"], c["ref"], c["d_out"], shapes, c["starts"], N, Lq, H, P,
                                  with_bound=True)
    ro = ref_out.view(N * Lq, H * 32).double()
    s_out = assert_within(out, ro, 2 * b, 1.0, torch.bfloat16, what=f"{name} out vs reference op")
    s_dv = assert_within(dv, ref_dv.view(N * S_in, H * 32), 2 * b_dv, 1.0, torch.float32, what=f"{name} d_value vs reference op")
    Wn = norm.double().view(1, 1, 1, L, 1, 2)
    ref_doff = (ref_dloc.double() / Wn).reshape(N * Lq, -1)
    a = attn.double()
    ref_dlogit = (a * (ref_dattn.double() - (a * ref_dattn.double()).sum((3, 4), keepdim=True))).reshape(N * Lq, -1)
    n_off = 2 * H * L * P
    s_off = assert_within(dp[:, :n_off], ref_doff, 2 * b_dp[:, :n_off], 1.0, torch.float32, what=f"{name} d_off vs reference op")
    s_lg = assert_within(dp[:, n_off:], ref_dlogit, 2 * b_dp[:, n_off:] + 8 * R.U32 * (a * ref_dattn.double().abs()).reshape(
        N * Lq, -1), 1.0, torch.float32, what=f"{name} d_logit vs reference op")
    print(f"{name} vs the reference's op, largest share of the bound: out {s_out:.3f} d_value {s_dv:.3f} d_off {s_off:.3f} "
          f"d_logit {s_lg:.3f}")


def _torch_msda(value, loc, attn, shapes, starts):
    """fp32 restatement: value [N, S_in, H, 32], loc [N, Lq, H, L, P, 2] in [0, 1], attn [N, Lq, H, L, P]."""
    N, S_in, H, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    out = 0
    for l, ((h, w), s0) in enumerate(zip(shapes, starts)):
        img = value[:, s0:s0 + h * w].permute(0, 2, 3, 1).reshape(N * H, D, h, w)
        grid = loc[:, :, :, l].permute(0, 2, 1, 3, 4).reshape(N * H, Lq, P, 2) * 2 - 1
        smp = F.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=False)   # [N*H, D, Lq, P]
        wl = attn[:, :, :, l].permute(0, 2, 1, 3).reshape(N * H, 1, Lq, P)
        out = out + (smp * wl).sum(-1)
    return out.view(N, H, D, Lq).permute(0, 3, 1, 2).reshape(N, Lq, H * D)


def _torch_module(st, q, r, x, shapes, starts, H, L, P):
    N, Lq, d = q.shape
    value = F.linear(x, st["value_proj.weight"], st["value_proj.bias"]).view(N, x.shape[1], H, -1)
    off = F.linear(q, st["sampling_offsets.weight"], st["sampling_offsets.bias"]).view(N, Lq, H, L, P, 2)
    attn = torch.softmax(F.linear(q, st["attention_weights.weight"], st["attention_weights.bias"]).view(N, Lq, H, L * P), -1)
    wh = torch.tensor([[w, h] for h, w in shapes], dtype=q.dtype, device=q.device)
    loc = r[:, :, None, :, None, :] + off / wh[None, None, None, :, None, :]
    core = _torch_msda(value, loc, attn.view(N, Lq, H, L, P), shapes, starts)
    return F.linear(core, st["output_proj.weight"], st["output_proj.bias"])


# name -> (module config, N, Lq, level shapes, L_ref)
RECIPE_MODULE = {
    "injector": (dict(d_model=1536, n_levels=3, n_heads=24, n_points=4, ratio=0.5), 3136, [(112, 112), (56, 56), (28, 28)], 1),
    "extractor": (dict(d_model=1536, n_levels=1, n_heads=24, n_points=4, ratio=0.5), 16464, [(56, 56)], 1),
    "pixel_decoder": (dict(d_model=1024, n_levels=3, n_heads=32, n_points=4, ratio=1.0), 16464,
                      [(112, 112), (56, 56), (28, 28)], 3),
}


@pytest.mark.parametrize("name", sorted(RECIPE_MODULE))
def test_module_recipe_shapes_against_torch(name):
    from one_peace_b200.vision.ms_deform_attn import MSDeformAttn
    cfg, Lq, shapes, L_ref = RECIPE_MODULE[name]
    torch.manual_seed(0)
    m = MSDeformAttn(**cfg).cuda()
    d = cfg["d_model"]
    with torch.no_grad():      # offsets of a few pixels and non-uniform weights, as a trained module has
        m.sampling_offsets.weight.normal_(0, 0.5 / d ** 0.5)
        m.attention_weights.weight.normal_(0, 1 / d ** 0.5)
        m.value_proj.bias.normal_(0, 0.1)
    S_in = sum(h * w for h, w in shapes)
    starts = [sum(h * w for h, w in shapes[:i]) for i in range(len(shapes))]
    q = torch.randn(1, Lq, d, device="cuda", requires_grad=True)
    x = torch.randn(1, S_in, d, device="cuda", requires_grad=True)
    r = torch.rand(1, Lq, L_ref, 2, device="cuda")
    cot = torch.randn(1, Lq, d, device="cuda")
    y = m(q, r, x, torch.tensor(shapes, device="cuda"), torch.tensor(starts, device="cuda"))
    (y * cot).sum().backward()
    st = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    q2 = q.detach().clone().requires_grad_(True)
    x2 = x.detach().clone().requires_grad_(True)
    y2 = _torch_module(st, q2, r, x2, shapes, starts, cfg["n_heads"], cfg["n_levels"], cfg["n_points"])
    (y2 * cot).sum().backward()
    cos = {"output": _cos(y, y2), "d_query": _cos(q.grad, q2.grad), "d_input_flatten": _cos(x.grad, x2.grad)}
    for k, p in m.named_parameters():
        cos[k] = _cos(p.grad, st[k].grad)
    print(name, " ".join(f"{k} {v:.5f}" for k, v in cos.items()))
    assert cos["output"] > 0.999
    assert min(cos.values()) > 0.99, cos
