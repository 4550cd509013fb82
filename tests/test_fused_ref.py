"""CPU: the bounds of tests/fused_ref.py against the fused-LayerNorm layer loop of inference
(``TransformerEncoder.run_fused``, ``TransformerEncoderLayer.forward_rows_fused``; the detection backbone's
``OnePeace.forward``, its row gathers around ``DetEncoder.run_fused`` with ``DetAttention``; the video backbone's
``VideoLayer.forward_video``) run on the fp64 kernel emulation ``Emu`` of tests/test_stem_ref.py, at
d = 128, H = 2, F = 256 (the fold needs F % 128 == 0, the GeGLU tiles 2F % 256 == 0) and two layers.

Each case runs the loop with its kernels behind ``Snapshots`` (``fused_ref.route``) and checks every recorded stage, the
records, xb == bf16(x) and the stack output.  Every case must stay within its bounds, and each planted mistake (a
one-line change of the loop's source) must exceed a bound at least MISS-fold.  The mistakes read buffers the loop has
written, never an uninitialised workspace, so each fails the same way every run.
tests/test_gpu_fused_contract.py runs the same case builders on the kernels at model width."""
from types import SimpleNamespace as NS

import pytest
import torch

import fused_ref as FR
import kernel_ref as R
import stem_ref as SR
from test_layer_ref import Snapshots, build_encoder, init_params, key_pad_of, lut_bias
from test_stem_ref import MISS, Emu

F32 = torch.float32
SMALL = dict(d=128, H=2, F=256)


def fused_case(kernels, form, edit=None, L=2, d=128, H=2, F=256, B=None, S=None, p_dtype=F32, seed=0, dev="cpu"):
    """one run_fused.  form: 'text' (mixed key padding, one sample with one live key, one shared LUT-form table),
    'image' (one LUT-form table per layer), 'audio' (the audio FFN, padded frames), 'long' (the dense table: ``attention``
    with records).  Returns NS(shares, exempt, got, ...)."""
    from one_peace_b200 import kernels as KM
    dev = torch.device(dev)
    g = torch.Generator().manual_seed(seed + 2000)
    enc = build_encoder(L, d, H, F, p_dtype, dev, seed).eval()
    B = B or {"text": 8, "image": 3, "audio": 2, "long": 2}[form]
    S = S or {"text": 17, "image": 197, "audio": 120, "long": 257}[form]
    modality = {"long": "text"}.get(form, form)
    valid = {"text": [S, S - 1, 1, S // 2, 2, S - 3, S, 5][:B], "image": None, "audio": [S, S - 37][:B],
             "long": [S, S - 100][:B]}[form]
    key_pad = key_pad_of(B, S, valid, dev) if valid else None
    tbs = [lut_bias(KM, S, H, g, dev) for _ in range(L if form == "image" else 1)]
    dense = [t[0].detach()[..., :S] for t in tbs]
    fast = [KM.RelPosBias(dense=t[0].detach()) if form == "long" else t[1] for t in tbs]
    return _run(kernels, enc, edit, fast, dense, key_pad, B, S, modality, d, g, dev)


def _vision_cfg(d, F, L, H):
    from one_peace_b200.unify_model_config import AdjustEncDecConfig
    return AdjustEncDecConfig(embed_dim=d, ffn_embed_dim=F, layers=L, attention_heads=H, drop_path_rate=0.0, dropout=0.0,
                              attention_dropout=0.0, activation_dropout=0.0, magneto_scale_attn=True, scale_attn=False,
                              scale_fc=True, scale_heads=False, use_text_moe=False, use_image_moe=True, use_audio_moe=False,
                              use_layer_scale=True, layer_scale_init_value=1e-2)


def det_case(kernels, edit=None, L=2, d=128, H=2, F=256, B=2, bucket=16, window=8, seed=0, dev="cpu"):
    """one detection backbone forward (``OnePeace.forward``) whose stem gives random grid-order rows: the window-major
    gather, layer 0 within the window x window windows of the bucket x bucket grid (B (bucket / window)^2 sequences),
    layer 1 over the whole grid (B sequences), random decomposed rel_pos_h / rel_pos_w and shared table, and the gather
    back to grid order"""
    from one_peace_b200.vision.det import OnePeace
    dev = torch.device(dev)
    g = torch.Generator().manual_seed(seed + 3000)
    model = OnePeace(attention_heads=H, bucket_size=bucket, embed_dim=d, ffn_embed_dim=F, layers=L,
                     use_decomposed_rel_pos=True, window_size=window, window_block_indexes=(0,))
    init_params(model.encoder, seed)
    with torch.no_grad():
        model.image_adapter.rel_pos_table.weight.copy_(torch.randn(model.image_adapter.rel_pos_table.weight.shape, generator=g))
    model = model.to(dev).eval()
    S = bucket * bucket
    x0 = torch.randn(B * S, d, generator=g).to(dev)
    model.image_adapter.stem = lambda img: x0.clone()          # the stem has its own tests; the loop starts from x0
    with FR.route(Snapshots(kernels), edit) as rec, torch.no_grad():
        out = model(torch.zeros(B, 3, 16 * bucket, 16 * bucket, device=dev))["last_feat"]
    chk, got, grid = FR.det_checks(model, x0, B, rec.log)
    chk["y"] = (grid.double(), torch.zeros_like(grid, dtype=torch.float64), F32)
    got["y"] = out.permute(0, 2, 3, 1).reshape(B * S, d)
    n = 3 + 1 + 3 + 1 + sum(11 + 2 for _ in model.encoder.layers)
    return _result(chk, got, rec.log, n)


def video_case(kernels, edit=None, L=2, d=128, H=2, F=256, Bv=2, T=5, N=17, seed=0, dev="cpu"):
    """one video backbone layer loop (``TransformerEncoder.run`` of vision/video.py) over Bv clips of T frames of N tokens,
    frame-major rows, the shared table in LUT form for the spatial pass"""
    from one_peace_b200 import kernels as KM
    from one_peace_b200.vision.video import TransformerEncoder as VideoEncoder
    dev = torch.device(dev)
    g = torch.Generator().manual_seed(seed + 4000)
    enc = init_params(VideoEncoder(_vision_cfg(d, F, L, H), T, 0.5), seed).to(dev).eval()
    dense, fast = lut_bias(KM, N, H, g, dev)
    x0 = torch.randn(Bv * T * N, d, generator=g).to(dev)
    rows = x0.clone()
    with FR.route(Snapshots(kernels), edit) as rec, torch.no_grad():
        enc.run(rows, fast, Bv, T, N)
    chk, got, xs = FR.video_checks(enc, x0, dense.detach()[..., :N], Bv, T, N, rec.log)
    chk["y"] = (xs[-1].double(), torch.zeros_like(xs[-1], dtype=torch.float64), F32)
    got["y"] = rows
    return _result(chk, got, rec.log, 3 + 1 + 24 * L)


def _run(kernels, enc, edit, fast, refs, key_pad, B, S, modality, d, g, dev):
    x0 = torch.randn(B * S, d, generator=g).to(dev)
    rows = x0.clone()
    with FR.route(Snapshots(kernels), edit) as rec, torch.no_grad():
        enc.run_fused(rows, fast, key_pad, B, S, modality)
    chk, got, xs = FR.encoder_checks(enc, x0, refs, key_pad, B, S, modality, rec.log)
    chk["y"] = (xs[-1].double(), torch.zeros_like(xs[-1], dtype=torch.float64), F32)
    got["y"] = rows
    return _result(chk, got, rec.log, 3 + 1 + 11 * len(enc.layers))


def _result(chk, got, log, n):
    sh = SR.shares(got, chk)
    return NS(shares=sh, exempt={k for k in sh if FR.is_exempt(k)}, got=got, log=log, n_checks=n)


CASES = {
    "text": dict(form="text"),
    "image": dict(form="image"),
    "audio": dict(form="audio"),
    "long": dict(form="long"),
    "det": dict(form="det"),
    "video": dict(form="video"),
}


def run(kernels, form, **kw):
    return {"det": det_case, "video": video_case}.get(form, lambda k, **a: fused_case(k, form, **a))(kernels, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulation_within_bounds(name):
    r = run(Emu(), **{**SMALL, **CASES[name]})
    assert len(r.shares) == r.n_checks
    bad = {k: v for k, v in r.shares.items() if not v <= 1.0}
    assert not bad, f"{name}: outside the bound: {bad}"


# name -> (case, (old, new) in the loop's source)
MISTAKES = {
    "FFN-LN records counted without the zero records": ("text", (
        "n_rec = 2 * ((2 * F_) // 256)   ", "n_rec = (2 * F_) // 256   ")),
    "out_proj without the bf16 copy (GeGLU reads a stale xb)": ("text", (
        'stats_out=ws["part_b"], out_bf16=xb,', 'stats_out=ws["part_b"],')),
    "next layer's LN1 from part_b": ("text", (
        'return dict(ln_partial=(ws["part_d"], n_t, d, self.self_attn_layer_norm.eps))',
        'return dict(ln_partial=(ws["part_b"], n_t, d, self.self_attn_layer_norm.eps))')),
    "out_proj without LayerScale": ("image", ('gamma=a["g1"], resid=x', "gamma=None, resid=x")),
    "QKV without the q scaling": ("text", ('colscale=a["qscale"],\n' + ' ' * 14 + 'workspace=ws["tail"]',
                                           '\n' + ' ' * 14 + 'workspace=ws["tail"]')),
    "image FFN for an audio pass": ("audio", ("f = self._fused_ffn_pack(modality)", 'f = self._fused_ffn_pack("image")')),
    "detection: decomposed terms of the scaled q": ("det", ("q_unscale=Q_UNSCALE)", "q_unscale=1.0)")),
    "detection: grid order restored with perm": ("det", ("K.row_gather(rows, inv)", "K.row_gather(rows, perm)")),
    "video: S-adapter fc2 residual from x": ("video", ('gamma=a["g1"], resid=ws["y"],', 'gamma=a["g1"], resid=x,')),
    "video: MLP adapter without scale": ("video", ('gamma=ad["scale"], resid=x,', "gamma=None, resid=x,")),
    "video: temporal attention with T and N swapped": ("video", (
        'K.attention_temporal(ws["qkv"], Bv, T, N, H,', 'K.attention_temporal(ws["qkv"], Bv, N, T, H,')),
}


@pytest.mark.parametrize("name", sorted(MISTAKES))
def test_planted_mistake_exceeds_bound(name):
    form, edit = MISTAKES[name]
    r = run(Emu(), edit=edit, **{**SMALL, **CASES[form]})
    # a bounded stage must see it: the bit-exact copies of a stage's own output (xb, y) alone do not count; a misplaced
    # row gather can only show in its exact check
    sh = {k: v for k, v in r.shares.items() if k.split(".")[-1] not in ("xb", "xb0", "y")}
    worst = max(sh, key=sh.get)
    assert sh[worst] >= MISS, f"{name}: largest share of a bound only {sh[worst]:.3g} ({worst})"


def test_route_restores():
    """the loop's kernels and methods are the package's again after a routed, edited run"""
    from one_peace_b200 import kernels as KM
    from one_peace_b200.transformer import multihead_attention as MHA
    from one_peace_b200.transformer import transformer_encoder as TE
    from one_peace_b200.transformer import transformer_layer as TL
    before = TL.TransformerEncoderLayer.__dict__["forward_rows_fused"]
    run(Emu(), edit=MISTAKES["FFN-LN records counted without the zero records"][1], **{**SMALL, **CASES["text"]})
    assert TL.K is KM and TE.K is KM and MHA.K is KM
    assert TL.TransformerEncoderLayer.__dict__["forward_rows_fused"] is before
