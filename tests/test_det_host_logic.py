"""CPU: the detection backbone's host logic.  oracle/restated_det.py against tests/golden/det.pt (the reference's own
onepeace.py); the production key / shape / dtype list and lr-decay rates; the ``pretrained=`` path for .pth and .pkl; the
refusals and the C ABI rejecting bad arguments; the window-major layout, LUT codes and decomposed-term indexing restated
on the CPU in fp64 against the restatement, with planted mistakes that must exceed the bound 100-fold; and the fp32
emulation of the projection kernel within its bound."""
import json
import os
import pickle
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import det_ref as D
import restated_det as RD
import synth_det as sd_
from one_peace_b200 import relpos


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "det.pt"), weights_only=False)


def _tiny(case, **kw):
    from one_peace_b200.vision.det import OnePeace
    bucket, window, pretrain, wbi = sd_.DET_CASES[case]
    torch.manual_seed(0)
    return OnePeace(bucket_size=bucket, window_size=window, pretrain_bucket_size=pretrain, window_block_indexes=wbi,
                    **sd_.DET_TINY, **kw)


def _state(m):
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    return sd_.det_state_dict(shapes, dict(m.named_buffers()))


@pytest.mark.parametrize("case", list(sd_.DET_CASES))
def test_restatement_matches_reference(case, golden_dir):
    g = _gold(golden_dir)["cases"][case]
    m = _tiny(case)
    assert [(k, tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()] == [tuple(x) for x in g["keys"]]
    bucket, window, pretrain, wbi = sd_.DET_CASES[case]
    out = RD.forward(_state(m), sd_.det_images(bucket), 4, 4, bucket, window, wbi)
    torch.testing.assert_close(out, g["last_feat"], rtol=1e-4, atol=1e-4)


def test_production_keys_and_lr_decay(golden_dir):
    from one_peace_b200.vision.det import OnePeace, get_onepeace_lr_decay_rate
    prod = json.loads(zlib.decompress(_gold(golden_dir)["production_z"]))
    lin = torch.linspace
    torch.linspace = lambda *a, **k: lin(*a, **{**k, "device": "cpu"})
    try:
        with torch.device("meta"):
            m = OnePeace(**sd_.PRODUCTION)
    finally:
        torch.linspace = lin
    assert [(k, tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()] == [tuple(x[:1]) + (tuple(x[1]), x[2])
                                                                                      for x in prod["keys"]]
    rates = {n: get_onepeace_lr_decay_rate("backbone.net." + n, 0.9, 40) for n, _ in m.named_parameters()}
    assert rates == prod["rates"]
    assert m._out_feature_strides == {"last_feat": 16} and m._out_feature_channels == {"last_feat": 1536}


@pytest.mark.parametrize("ext", ["pth", "pkl"])
def test_pretrained_loading(ext, golden_dir, tmp_path):
    g = _gold(golden_dir)["pretrained"]
    path = tmp_path / f"ckpt.{ext}"
    ckpt = {"model": {k: v.clone() for k, v in g["ckpt"].items()}}
    if ext == "pth":
        torch.save(ckpt, path)
    else:
        with open(path, "wb") as f:
            pickle.dump(ckpt, f)
    st = _tiny("win4", pretrained=str(path)).state_dict()
    for k, v in g["loaded"].items():
        torch.testing.assert_close(st[k], v, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("kw,exc", [(dict(dropout=0.1), NotImplementedError), (dict(rp_bias=True), NotImplementedError),
                                    (dict(shared_rp_bias=False), NotImplementedError),
                                    (dict(use_decomposed_rel_pos=False), NotImplementedError),
                                    (dict(window_size=3), NotImplementedError)])
def test_constructor_refusals(kw, exc):
    from one_peace_b200.vision.det import OnePeace
    args = dict(sd_.DET_TINY, bucket_size=8, window_size=4, window_block_indexes=(0, 1, 2))
    args.update(kw)
    with pytest.raises(exc):
        OnePeace(**args)


def test_abi_rejects_bad_arguments():
    from one_peace_b200 import _lib
    lib = _lib.load()
    p = 16        # any non-null pointer: every check below fails before a launch
    INVALID = 1
    proj = lambda **o: lib.opb_relpos_decomp_proj(*[o.get(n, v) for n, v in [
        ("qkv", p), ("h", p), ("w", p), ("py", p), ("px", p), ("qu", 8.0), ("rh", p), ("rw", p), ("B", 1), ("S", 256),
        ("H", 2), ("kh", 16), ("kw", 16), ("st", None)]])
    for bad in (dict(qkv=None), dict(rh=None), dict(S=255), dict(kh=0), dict(kh=512, kw=1, S=512), dict(B=0),
                dict(qu=float("nan"))):
        assert proj(**bad) != 0, bad
    att = lambda **o: lib.opb_attention_decomp_fwd(*[o.get(n, v) for n, v in [
        ("qkv", p), ("lut", p), ("L", 961), ("cr", p), ("cc", p), ("rh", p), ("rw", p), ("ky", p), ("kx", p), ("kh", 16),
        ("kw", 16), ("out", p), ("lse", None), ("st", None), ("B", 1), ("S", 256), ("H", 2), ("s", None)]])
    for bad in (dict(out=None), dict(ky=None), dict(S=250), dict(kw=0), dict(L=0), dict(H=0)):
        assert att(**bad) != 0, bad


# ---------------------------------------------------------------------------------------------------------------------
# The kernel path's layout restated in fp64 on the CPU (window-major rows, LUT codes, grid positions, decomposed terms
# indexed by key coordinates) against the restatement in fp64.
# ---------------------------------------------------------------------------------------------------------------------
LAYOUT_TOL = 1e-9          # relative; fp64 reorderings only


def emulate_forward(sd, img, heads, layers, side, win, wbi, mistake=None):
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    from one_peace_b200.vision.det import resize_table
    B = img.shape[0]
    d = sd["image_adapter.pos_embed"].shape[1]
    pos = sd["image_adapter.pos_embed"]
    x = RD.stem({**sd, "image_adapter.pos_embed": pos if mistake != "pos_embed_0" else torch.cat([pos[:-1][:1], pos[:-1]])},
                img.double()).reshape(B, side * side, d)
    order, y, xx, ly, lx = relpos.window_major_order(side, win)
    x = x[:, torch.from_numpy(order)]
    table = sd["image_adapter.rel_pos_table.weight"]
    glob_set = [i for i in range(layers) if i not in wbi]
    if mistake == "sets_swapped":
        wbi = tuple(glob_set)
    for i in range(layers):
        p = f"encoder.layers.{i}."
        windowed = i in wbi
        s_ = win if windowed else side
        t = resize_table(table, 31, 2 * s_ - 1) if mistake != "no_interp" else table[:(2 * s_ - 1) ** 2 + 3]
        if windowed:
            _, cr, cc = relpos.grid_lut_index(win)
            py, px = ly, lx
        else:
            _, cr, cc = relpos.grid_lut_index(side, order)
            py, px = y, xx
            if mistake == "window_codes_global":
                _, cr, cc = relpos.grid_lut_index(win, None)
                cr = np.resize(cr, side * side); cc = np.resize(cc, side * side)
        n = side * side // (s_ * s_)
        S = s_ * s_
        cr, cc = torch.from_numpy(cr[:S].astype(np.int64)), torch.from_numpy(cc[:S].astype(np.int64))
        bias = t[:, :][cr[:, None] - cc[None, :]].permute(2, 0, 1)          # [H, S, S]
        py_t, px_t = torch.from_numpy(py[:S]), torch.from_numpy(px[:S])       # every window has the same local grid
        ln = lambda name, v, k=d: F.layer_norm(v, (k,), sd[p + name + ".weight"], sd[p + name + ".bias"])
        h = ln("self_attn_layer_norm", x).reshape(B * n, S, d)
        lin = lambda name, v: F.linear(v, sd[p + "self_attn." + name + ".weight"], sd.get(p + "self_attn." + name + ".bias"))
        sp = lambda v: v.reshape(B * n, S, heads, 64).permute(0, 2, 1, 3)
        q, k, v = sp(lin("q_proj", h)), sp(lin("k_proj", h)), sp(lin("v_proj", h))
        qd = q * 0.125 if mistake == "scaled_q" else q
        sgn = -1 if mistake == "ky_minus_qy" else 1
        rh_tab, rw_tab = sd[p + "self_attn.rel_pos_h"], sd[p + "self_attn.rel_pos_w"]
        if mistake == "swap_hw":
            py_t, px_t = px_t, py_t
        ar = torch.arange(s_)
        rel_h = torch.einsum("bhsc,skc->bhsk", qd, rh_tab[sgn * (py_t[:, None] - ar[None, :]) + s_ - 1])
        rel_w = torch.einsum("bhsc,skc->bhsk", qd, rw_tab[sgn * (px_t[:, None] - ar[None, :]) + s_ - 1])
        logits = (q * 0.125) @ k.transpose(-1, -2) + bias[None] + rel_h[..., py_t] + rel_w[..., px_t]
        o = logits.softmax(-1) @ v
        o = o.permute(0, 2, 1, 3).reshape(B, side * side, d)
        o = F.layer_norm(o, (d,), sd[p + "self_attn.ln.weight"], sd[p + "self_attn.ln.bias"])
        x = x + sd[p + "gamma_1"] * lin("out_proj", o)
        f = p + "image_ffn."
        y2 = ln("final_layer_norm", x)
        u = F.gelu(F.linear(y2, sd[f + "0.wi_0.weight"])) * F.linear(y2, sd[f + "0.wi_1.weight"])
        u = F.layer_norm(u, (u.shape[-1],), sd[f + "2.weight"], sd[f + "2.bias"])
        x = x + sd[p + "gamma_2"] * F.linear(u, sd[f + "3.weight"], sd[f + "3.bias"])
    if mistake != "window_major_output":
        inv = np.argsort(order)
        x = x[:, torch.from_numpy(inv)]
    return x.reshape(B, side, side, d).permute(0, 3, 1, 2)


MISTAKES = ["scaled_q", "ky_minus_qy", "swap_hw", "window_codes_global", "no_interp", "pos_embed_0", "sets_swapped",
            "window_major_output"]


@pytest.fixture(scope="module")
def layout_case():
    m = _tiny("win4")
    sd = _state(m)
    img = sd_.det_images(8, batch=1)
    ref = RD.forward({k: v.double() if v.is_floating_point() else v for k, v in sd.items()}, img, 4, 4, 8, 4, (0, 1, 2),
                     dtype=torch.float64)
    return sd, img, ref


def test_layout_emulation_within_bound(layout_case):
    sd, img, ref = layout_case
    got = emulate_forward(sd, img, 4, 4, 8, 4, (0, 1, 2))
    err = ((got - ref).abs().max() / ref.abs().max()).item()
    assert err <= LAYOUT_TOL, err


@pytest.mark.parametrize("mistake", MISTAKES)
def test_layout_planted_mistakes_exceed_bound(layout_case, mistake):
    sd, img, ref = layout_case
    try:
        got = emulate_forward(sd, img, 4, 4, 8, 4, (0, 1, 2), mistake=mistake)
        err = ((got - ref).abs().max() / ref.abs().max()).item()
    except IndexError:          # swapped layer sets: a layer's rel_pos_h is too short for its grid
        err = float("inf")
    assert err > 100 * LAYOUT_TOL, (mistake, err)


def test_projection_fp32_emulation_within_bound():
    g = torch.Generator().manual_seed(5)
    H, kh, kw, B = 2, 8, 6, 1
    S = kh * kw
    qkv = (torch.randn(B * S, 3 * H * 64, generator=g) * 0.2).to(torch.bfloat16)
    rph, rpw = torch.randn(2 * kh - 1, 64, generator=g), torch.randn(2 * kw - 1, 64, generator=g)
    order = torch.randperm(S, generator=g)
    py, px = (order // kw).int(), (order % kw).int()
    rh, eh, rw, ew = D.proj_ref(qkv, rph, rpw, py, px, B, S, H, kh, kw)
    for h in range(H):
        q = qkv[:, h * 64:(h + 1) * 64]
        got_h = D.proj_emulate_fp32(q, rph, py, kh)
        assert ((got_h.double() - rh[0, h]).abs() <= eh[0, h]).all()
        # planted: the scaled q (no unscale) is far outside the bound
        bad = D.proj_emulate_fp32(q, rph, py, kh) / 8
        assert ((bad.double() - rh[0, h]).abs() > 100 * eh[0, h]).any()
        got_w = D.proj_emulate_fp32(q, rpw, px, kw)
        assert ((got_w.double() - rw[0, h]).abs() <= ew[0, h]).all()
