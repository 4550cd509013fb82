"""CPU: the bounds of tests/layer_ref.py against the encoder stack of the training path (``EncoderStackFn``,
``layer_forward``, ``layer_backward`` of one_peace_b200/autograd.py) run on the fp64 kernel emulation ``Emu`` of
tests/test_stem_ref.py, at d = 128, H = 2, F = 192 and two or three layers.

Each case runs the stack through a fresh copy of the autograd module whose kernels sit behind ``Snapshots`` (a
``Recorder`` that keeps copies of every argument before the call and of every output after it), takes the upstream
gradient on every row (padded rows included), and checks every recorded stage, every parameter's ``.grad`` in its dtype,
``dx0`` and the bias-table gradients.  Every case must stay within its bounds under both activation policies (and the
single-modality ones, at F = 256, after the fused-LayerNorm forward, whose own stages tests/fused_ref.py checks), and each
planted mistake (a one-line change of the module's source, or the ``dbias_t_overwrite`` flag of ``Emu``) must exceed a
bound at least MISS-fold.  Where the reference is exactly zero the bound is zero: dk / dv of padded keys, the bias
gradient under -inf canvas entries and past S, the other modality's FFN (no ``.grad`` at all).
tests/test_gpu_layer_contract.py runs the same case builders on the kernels at model width."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import fused_ref as FR
import kernel_ref as R
import layer_ref as LR
import stem_ref as SR
from test_stem_ref import MISS, Emu, Recorder, functions

BF, F32 = torch.bfloat16, torch.float32
SMALL = dict(d=128, H=2, F=192)


def _copy(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, (list, tuple)):
        return type(v)(_copy(t) for t in v)
    return v


class Snapshots(Recorder):
    """``Recorder`` whose log entries hold copies: the arguments as they were before the call (``a``), the keyword
    arguments and the result as they are after it (``kw``, ``r``).  The stack updates its gradient buffer and its
    bias-gradient tables in place, so a reference to them would show only their final values.  Kernels that write into
    positional arguments and return nothing of them (``POST``) also keep those arguments as they are after the call
    (``post``)."""
    POST = ("row_stats_cast", "ln_fold")

    def __getattr__(self, name):
        f = getattr(self.kernels, name)
        if not callable(f) or isinstance(f, type):
            return f

        def call(*a, **kw):
            before = _copy(a)
            r = f(*a, **kw)
            self.log.append(NS(name=name, a=before, kw={k: _copy(v) for k, v in kw.items()}, r=_copy(r),
                               post=_copy(a) if name in self.POST else None))
            return r
        return call


# ----------------------------------------------------------------------------------------------------------------------
# the model, the biases, the case
# ----------------------------------------------------------------------------------------------------------------------
def build_encoder(L, d, H, F, p_dtype, dev, seed, decoder=False):
    """L layers with random parameters: weights N(0, 1 / fan_in), LayerNorm weights 1 + N(0, 0.2^2), biases
    N(0, 0.1^2), LayerScale gammas of either sign with magnitudes in [0.1, 1]"""
    from one_peace_b200.transformer.transformer_encoder import TransformerEncoder
    from one_peace_b200.unify_model_config import one_peace_4b_decoder_config, one_peace_4b_encoder_config
    mk = one_peace_4b_decoder_config if decoder else one_peace_4b_encoder_config
    enc = TransformerEncoder(mk(layers=L, embed_dim=d, ffn_embed_dim=F, attention_heads=H), None, True, True, True)
    return init_params(enc, seed).to(dev, p_dtype).train()


def init_params(enc, seed):
    """the random parameters of ``build_encoder``"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in enc.named_parameters():
            if "gamma" in name:
                sign = torch.where(torch.rand(p.shape, generator=g) < 0.5, -1.0, 1.0)
                p.copy_(sign * (0.1 + 0.9 * torch.rand(p.shape, generator=g)))
            elif p.dim() == 2:
                p.copy_(torch.randn(p.shape, generator=g) * p.shape[1] ** -0.5)
            elif name.endswith("weight"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    return enc


def lut_bias(kernels, S, H, g, dev):
    """dense fp32 (H,S,S_pad) leaf and the same values as a LUT-form kernels.RelPosBias (image codes for S = w^2 + 1, text
    codes otherwise), as the adapters build them for a training forward"""
    import restated
    from one_peace_b200 import relpos
    w = int(round((S - 1) ** 0.5))
    if w * w + 1 == S and S > 2:
        bucket, codes, ntab = restated.make_image_bucket_position(w), relpos.image_codes(S, w), (2 * w - 1) ** 2 + 3
    else:
        bucket, codes, ntab = restated.make_token_bucket_position(256)[:S, :S], relpos.text_codes(S), 514
    table = torch.randn(ntab, H, generator=g).to(dev)
    idx, crow, ccol = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in relpos.build_lut_index(bucket.numpy(), codes))
    fast = kernels.RelPosBias(lut=R.relpos_lut_ref(table, idx).contiguous(), code_row=crow, code_col=ccol)
    dense = torch.zeros(H, S, (S + 7) // 8 * 8, device=dev)
    dense[..., :S] = table[bucket.to(dev)].permute(2, 0, 1)
    assert torch.equal(fast.lut[:, (crow[:S, None] - ccol[None, :S]).long()], dense[..., :S])
    return dense.requires_grad_(), fast


def key_pad_of(B, S, valid, dev):
    kp = torch.zeros(B, S, dtype=torch.uint8)
    for b, n in enumerate(valid):
        kp[b, n:] = 1
    return kp.to(dev)


def canvas(shape, S_pad, key_pad, g, dev):
    """dense fp32 (Bb,H,S,S_pad) canvas: N(0, 1) over the S logical columns, -inf on padded keys of a per-sample canvas,
    zero padding columns"""
    Bb, H, S = shape
    c = torch.zeros(Bb, H, S, S_pad)
    c[..., :S] = torch.randn(Bb, H, S, S, generator=g)
    if Bb > 1 and key_pad is not None:
        c[..., :S] = c[..., :S].masked_fill(key_pad.cpu().bool().view(Bb, 1, 1, S), float("-inf"))
    return c.to(dev).requires_grad_()


def _drop_path_seed(layers, B, dev):
    """a torch seed under which every drop-path draw of the stack drops at least one sample and keeps at least one"""
    for s in range(1000):
        torch.manual_seed(s)
        ok = True
        for layer in layers:
            if layer.drop_path_prob > 0:
                keep = torch.rand(B, device=dev) < 1 - layer.drop_path_prob
                ok = ok and bool(keep.any()) and not bool(keep.all())
        if ok:
            return s
    raise AssertionError("no seed drops and keeps")


def stack_case(kernels, form, policy="keep", edit=None, L=2, d=128, H=2, F=192, B=None, S=None, parts=None,
               p_dtype=F32, drop_path=0.0, seed=0, dev="cpu"):
    """one EncoderStackFn forward and backward.  form: 'text' (one shared LUT-form table, mixed key padding), 'image'
    (one table per layer), 'long' (S > BIAS_T_Q, shared table: dense backward), 'vl' (two parts, one per-sample canvas
    per layer with -inf padded keys), 'al' (two parts, one (1,H,S,S_pad) canvas), 'decoder' (two parts, no LayerScale, no
    bias).  policy: 'keep', 'recompute' (the forward layer by layer; single-modality passes then attend with the dense
    tables), or 'fused' (recompute after the fused-LayerNorm forward, LUT-form biases).
    Returns NS(shares, exempt, ...) with the logs, the layout and the inputs for the exact-zero checks."""
    dev = torch.device(dev)
    g = torch.Generator().manual_seed(seed + 1000)
    fns = functions(kernels, edit, recorder=Snapshots)
    decoder = form == "decoder"
    enc = build_encoder(L, d, H, F, p_dtype, dev, seed, decoder=decoder)
    for layer in enc.layers:
        layer.drop_path_prob = drop_path
    from one_peace_b200 import kernels as KM
    if form in ("text", "image", "long"):
        B = B or {"text": 8, "image": 3, "long": 2}[form]
        S = S or {"text": 17, "image": 197, "long": 257}[form]
        parts = [(form if form != "long" else "text", S)]
        valid = {"text": [S, S - 1, 1, S // 2, 2, S - 3, S, 5][:B], "image": None, "long": [S, S - 100][:B]}[form]
        key_pad = key_pad_of(B, S, valid, dev) if valid else None
        tbs = [lut_bias(KM, S, H, g, dev) for _ in range(L if form == "image" else 1)]
        biases = [t[0] for t in tbs]
        # un-fused recompute: without a LUT form the forward runs layer by layer on the dense tables
        bias_list = [fns.TrainBias(dn, None if policy == "recompute" else fast) for dn, fast in tbs]
    else:
        B = B or 2
        parts = parts or ([("text", 17), ("image", 50)] if form in ("vl", "decoder") else [("text", 17), ("audio", 40)])
        S = sum(s for _, s in parts)
        S1 = parts[0][1]
        pads = [torch.zeros(B, s, dtype=torch.uint8) for _, s in parts]
        pads[0][1, S1 - 3:] = 1                                     # sample 1: the last three text tokens padded
        if form == "al":
            pads[1][0, parts[1][1] // 2:] = 1                       # sample 0: half of its audio frames padded
        key_pad = torch.cat(pads, 1).to(dev) if form != "decoder" else None
        S_pad = (S + 7) // 8 * 8
        if form == "vl":
            biases = [canvas((B, H, S), S_pad, key_pad, g, dev) for _ in range(L)]
        elif form == "al":
            biases = [canvas((1, H, S), S_pad, None, g, dev)]
        else:
            biases = []
    lay = LR.layout(B, parts, dev)
    x0 = torch.randn(lay.M, d, generator=g).to(dev).requires_grad_()
    dy = torch.randn(lay.M, d, generator=g).to(dev)
    if drop_path:
        torch.manual_seed(_drop_path_seed(enc.layers, B, dev))
    rng = torch.cuda.get_rng_state(dev) if dev.type == "cuda" else torch.get_rng_state()
    old = os.environ.get("OPB_ACTIVATIONS")
    os.environ["OPB_ACTIVATIONS"] = "keep" if policy == "keep" else "recompute"
    try:
        with FR.route(fns.K):                  # the fused forward (TransformerEncoder.run_fused) logs to the same recorder
            if len(parts) == 1:
                y = fns.run_encoder_stack(enc, x0.view(B, S, d), bias_list, key_pad, parts[0][0])
            else:
                y = fns.run_general_stack(enc, x0, fns.SeqLayout(B, parts, dev), key_pad, biases, True)
        node = y.grad_fn
        while not hasattr(node, "xs"):
            node = node.next_functions[0][0]
        kept = [t.clone() for t in node.xs]
        fwd_log = list(fns.K.log)
        fns.K.log.clear()
        y.backward(dy.view(y.shape))
    finally:
        if old is None:
            del os.environ["OPB_ACTIVATIONS"]
        else:
            os.environ["OPB_ACTIVATIONS"] = old
    bwd_log = fns.K.log
    fused = policy == "fused"
    assert fused == (not LR.segments(fwd_log, lay)), "the forward ran fused exactly when the fused policy was asked"
    rs = LR.row_scales(enc.layers, lay, rng, dev)
    chk, got = LR.stack_checks(enc, lay, x0, dy, y, biases, key_pad, rs, fwd_log, bwd_log, shared_tables=len(parts) == 1,
                               kept_inputs=kept if fused else None)
    sh = SR.shares(got, chk)
    exempt = {k for k in sh if LR.is_exact(k) or LR.is_reduction(k) or FR.is_exempt(k)}
    return NS(shares=sh, exempt=exempt, got=got, enc=enc, lay=lay, parts=parts, key_pad=key_pad, biases=biases, x0=x0, rs=rs,
              fwd_log=fwd_log, bwd_log=bwd_log, L=L, d=d)


CASES = {
    "text": dict(form="text"),
    "image": dict(form="image"),
    "long": dict(form="long"),
    "vl": dict(form="vl", L=3),
    "al": dict(form="al"),
    "decoder": dict(form="decoder"),
    "drop_path": dict(form="text", drop_path=0.5, L=3, seed=5),
    "text_bf16": dict(form="text", p_dtype=BF, seed=7),
}


FUSED = ("text", "image", "long")          # single-modality, every bias with a LUT form, no drop-path


@pytest.mark.parametrize("policy", ["keep", "recompute", "fused"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_emulation_within_bounds(case, policy):
    if policy == "fused" and case not in FUSED:
        pytest.skip("the fused forward runs single-modality passes without drop-path")
    # the fused forward folds its LayerNorms into GEMMs whose tiles need F % 128 == 0
    r = stack_case(Emu(), policy=policy, **{**SMALL, **CASES[case], **(dict(F=256) if policy == "fused" else {})})
    bad = {k: v for k, v in r.shares.items() if not v <= 1.0}
    assert not bad, f"{case} / {policy}: outside the bound: {bad}"


# name -> (case, policy, source edit or kernel flags)
MISTAKES = {
    "v bias gradient from the k slot": ("text", "keep", dict(edit=("dbqkv[2 * d:], dWo", "dbqkv[d:2 * d], dWo"))),
    "fc2 bias summed over every part": ("vl", "keep", dict(edit=("K.colsum(dfp, g(d))", "K.colsum(df, g(d))"))),
    "GeGLU weight halves swapped": ("text", "keep", dict(edit=("ffn_grads += [dW01[:F_], dW01[F_:]",
                                                               "ffn_grads += [dW01[F_:], dW01[:F_]"))),
    "LN2 adjoint overwrites dx": ("text", "keep", dict(edit=("dx, eps=layer.final_layer_norm.eps, accumulate=True",
                                                             "dx, eps=layer.final_layer_norm.eps, accumulate=False"))),
    "datt gathered with to_mm": ("vl", "keep", dict(edit=("datt = K.row_gather(datt, lay.to_bm)",
                                                          "datt = K.row_gather(datt, lay.to_mm)"))),
    "attention adjoint without drop-path": ("drop_path", "keep", dict(edit=(
        'do = K.scale_resid_bwd(dx, s["o"], p["g1"], row_scale', 'do = K.scale_resid_bwd(dx, s["o"], p["g1"], None'))),
    "attention residual without drop-path": ("drop_path", "keep", dict(edit=(
        'x2 = K.scale_resid_fwd(x, o, p["g1"], row_scale', 'x2 = K.scale_resid_fwd(x, o, p["g1"], None'))),
    "dW01 from the first part's rows": ("vl", "keep", dict(edit=('dW01 = _dw(dgl, s["h2"][rs]', 'dW01 = _dw(dgl, s["h2"][:n]'))),
    "recompute from the layer below's input": ("text", "recompute", dict(edit=(
        "_, saved = layer_forward(layer, ctx.xs[i]", "_, saved = layer_forward(layer, ctx.xs[max(i - 1, 0)]"))),
    "every layer's bias gradient into table 0": ("vl", "keep", dict(edit=("_b3(_pick(dbiases, i))",
                                                                          "_b3(_pick(dbiases, 0))"))),
    "transposed bias gradient never folded": ("text", "keep", dict(edit=("K.relpos_dbias_fold(dt, db)", "pass"))),
    "transposed bias gradient stored, not added": ("text", "keep", dict(flags=dict(dbias_t_overwrite=True))),
}


@pytest.mark.parametrize("name", sorted(MISTAKES))
def test_planted_mistake_exceeds_bound(name):
    case, policy, how = MISTAKES[name]
    r = stack_case(Emu(**how.get("flags", {})), policy=policy, edit=how.get("edit"), **{**SMALL, **CASES[case]})
    worst = max(r.shares, key=r.shares.get)
    assert r.shares[worst] >= MISS, f"{name}: largest share of a bound only {r.shares[worst]:.3g} ({worst})"


def test_exact_zeros():
    """dk / dv of padded keys, the bias gradient under -inf canvas entries and in padding columns, no dgamma for an absent
    gamma, no gradient at all for the FFN of a modality the pass does not contain"""
    r = stack_case(Emu(), **{**SMALL, **CASES["text"]})
    d, S = r.d, r.lay.S
    dead = r.key_pad.reshape(-1).bool()
    calls = [e for e in r.bwd_log if e.name == "attention_bwd_t"]
    assert len(calls) == r.L
    for e in calls:
        assert not e.r[dead, d:].any(), "dk / dv of a padded key"
    assert not r.biases[0].grad[..., S:].any()
    for name, p in r.enc.layers.named_parameters():
        if "image_ffn" in name or "audio_ffn" in name:
            assert p.grad is None, name
        else:
            assert p.grad is not None, name

    r = stack_case(Emu(), **{**SMALL, **CASES["vl"]})
    dead = r.key_pad.bool()[:, None, None, :].expand(-1, 2, r.lay.S, -1)
    for b in r.biases:
        assert torch.isinf(b.detach()[..., :r.lay.S][dead]).all()
        assert (b.grad[..., :r.lay.S][dead] == 0).all(), "bias gradient under a -inf entry"
        assert not b.grad[..., r.lay.S:].any()
    for name, p in r.enc.layers.named_parameters():
        assert (p.grad is None) == ("audio_ffn" in name), name

    r = stack_case(Emu(), **{**SMALL, **CASES["decoder"]})
    assert all(layer.gamma_1 is None and layer.gamma_2 is None for layer in r.enc.layers)
    srb = [e for e in r.bwd_log if e.name == "scale_resid_bwd"]
    assert len(srb) == 2 * r.L and all(e.kw.get("dgamma") is None for e in srb), "a dgamma for an absent gamma"
