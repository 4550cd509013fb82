"""fp64 stage references of the fused-LayerNorm layer loops of inference (one_peace_b200/transformer: ``TransformerEncoder.
run_fused``, ``TransformerEncoderLayer.forward_rows_fused``; vision/det.py: ``OnePeace.forward``; vision/video.py:
``VideoLayer.forward_video``), with an error bound for every output element.

Plain PyTorch on whatever device the inputs live on; nothing here calls the extension.  Every bound is a single-kernel
bound of ``kernel_ref``: ``gemm_ref`` (fused LayerNorm from mu / rstd or from partial records, ``stats``, GeGLU and
residual epilogues, and the ``ln_colsum_err`` / ``bias_err`` terms of the folded operands), ``ln_fold_ref``,
``attention_ref`` with its ``stats``, ``scale_resid_ref``, ``relpos_lut_ref``, ``row_gather_ref``-style exact copies,
``det_ref.proj_ref`` / ``decomp_attention_ref``, and ``layernorm_ref``'s ``raw`` statistics (``row_stats_cast``).

No LayerNorm of the loop runs as a kernel.  Each one is folded into the GEMM that reads its output: the GEMM reads the
un-normalised bf16 rows, the folded weight W diag(g), its column sums and the bias W beta + b, and the row statistics
from (sum, sum of squares) records that the kernel which wrote those rows left behind:

  layer 0   xb = bf16(x0), mu, rstd = row_stats_cast(x0)
  per layer qkv = LN1(x) Wqkv^T + b (q scaled)          ln1: mu / rstd (layer 0), else the previous fc2's records (n_t)
            o, rec_a = attention(qkv, bias)              H per-head records
            x2, xb, rec_b = x + g1 (LN_attn(o) Wo^T + bo)  n_t = ceil(d / 256) records
            u, rec_c = geglu(LN2(x2) W01^T)              2 * (2F / 256) records, every second one zero
            x3, xb, rec_d = x2 + g2 (LN_ffn(u) W2^T + b2)  records of the next layer's LN1
  detection the loop runs on window-major rows (one row_gather in, one back to grid order, both exact); the attention
            is rel_h, rel_w = relpos_decomp_proj(qkv) of the unscaled q (``det_ref.proj_ref``), then attention_decomp over
            the layer's windows or the whole grid (``det_ref.decomp_attention_ref`` on the recorded rel_h / rel_w)
  video     a temporal, a spatial and a joint pass per layer (``video_checks``)

Each stage is checked on its own, from the layer's PARAMETERS (the folds are ``ln_fold_ref`` of them) and from the
recorded OUTPUTS of the stages that feed it in the model: the bf16 operand of a GEMM that reads xb is bf16 of the
recorded fp32 x, the residual is the recorded x, the statistics are the records the producing stage wrote.  Nothing is
taken from the arguments the code under test passed to the kernel under check, so a GEMM given stale rows, the wrong
records, the wrong record count, eps, gamma or FFN fails its check.  The records themselves, xb == bf16(x) (bit for bit)
and the stack output (the last recorded x, exactly) are checked as outputs.

The kernel calls come from a log of copies (``Snapshots`` in tests/test_layer_ref.py), since the loop updates x, xb and
its workspace in place.  ``route`` sends the loop's kernel calls (the module-level ``K`` of the transformer, detection
and video modules) through such a recorder and plants a one-line source edit in one of the loop's methods."""
import contextlib
import inspect
import textwrap
from types import SimpleNamespace as NS

import torch

import det_ref as D
import kernel_ref as R

BF, F32 = torch.bfloat16, torch.float32
# outputs exempt from the lower floor of a share: exact copies, records and row statistics
EXEMPT = ("xb", "xb0", "stats", "mu", "rstd", "y", "kept", "lut", "wmajor", "grid")


def is_exempt(name):
    return name.split(".")[-1] in EXEMPT


def _f(t):
    return None if t is None else t.detach().float()


# ----------------------------------------------------------------------------------------------------------------------
# routing the loop's kernels through a recorder, planting an edit
# ----------------------------------------------------------------------------------------------------------------------
def _loop_modules():
    from one_peace_b200.transformer import multihead_attention as MHA
    from one_peace_b200.transformer import transformer_encoder as TE
    from one_peace_b200.transformer import transformer_layer as TL
    from one_peace_b200.vision import det as DET
    from one_peace_b200.vision import video as VID
    return TL, TE, MHA, DET, VID


def _loop_methods():
    TL, TE, _, DET, VID = _loop_modules()
    return [(TL, TL.TransformerEncoderLayer, n) for n in ("forward_rows_fused", "_fused_attn_pack", "_fused_ffn_pack")] + \
           [(TE, TE.TransformerEncoder, "run_fused"), (DET, DET.DetAttention, "run_attention"), (DET, DET.OnePeace, "forward"),
            (VID, VID.VideoLayer, "forward_video"), (VID, VID.TransformerEncoder, "run")]


@contextlib.contextmanager
def route(rec, edit=None):
    """Within the block the fused loop calls its kernels through ``rec``; edit = (old, new) replaces the one occurrence of
    ``old`` in the loop's methods (an edited copy of that method is set onto its class).  Everything is restored on exit."""
    mods = _loop_modules()
    old_k = [m.K for m in mods]
    patched = []
    try:
        for m in mods:
            m.K = rec
        if edit is not None:
            hits = [(mod, cls, n, textwrap.dedent(inspect.getsource(getattr(cls, n)))) for mod, cls, n in _loop_methods()]
            hits = [h for h in hits if edit[0] in h[3]]
            assert len(hits) == 1 and hits[0][3].count(edit[0]) == 1, edit[0]
            mod, cls, n, src = hits[0]
            ns = dict(vars(mod))
            exec(compile(src.replace(*edit), mod.__file__, "exec"), ns)
            patched.append((cls, n, cls.__dict__[n]))
            setattr(cls, n, ns[n])
        yield rec
    finally:
        for cls, n, f in patched:
            setattr(cls, n, f)
        for m, k in zip(mods, old_k):
            m.K = k


# ----------------------------------------------------------------------------------------------------------------------
# the folded operands, from the parameters
# ----------------------------------------------------------------------------------------------------------------------
def fold_ref(weights, ln, biases, interleave=False):
    """``TransformerEncoderLayer._fold`` of the parameters: ``ln_fold_ref`` of each weight, placed as the pack places it
    (stacked along N, or the GeGLU tile interleave).  -> NS(w bf16 [N, K], cs, cs_err, b, b_err [N])"""
    outs = [R.ln_fold_ref(w.detach(), _f(ln.weight), _f(ln.bias), _f(b), interleave=i + 1 if interleave else 0)
            for i, (w, b) in enumerate(zip(weights, biases))]
    if not interleave:
        return NS(w=torch.cat([o.wg for o in outs]), cs=torch.cat([o.colsum for o in outs]),
                  cs_err=torch.cat([o.colsum_err for o in outs]), b=torch.cat([o.bias for o in outs]),
                  b_err=torch.cat([o.bias_err for o in outs]))
    N, Kd = sum(o.wg.shape[0] for o in outs), outs[0].wg.shape[1]
    dev = outs[0].wg.device
    r = NS(w=torch.empty(N, Kd, dtype=BF, device=dev), **{k: torch.empty(N, dtype=torch.float64, device=dev)
                                                          for k in ("cs", "cs_err", "b", "b_err")})
    for o in outs:
        r.w[o.rows], r.cs[o.rows], r.cs_err[o.rows], r.b[o.rows], r.b_err[o.rows] = o.wg, o.colsum, o.colsum_err, o.bias, o.bias_err
    return r


def layer_folds(layer, modality):
    a = layer.self_attn
    ffn = getattr(layer, f"{modality}_ffn")
    d = layer.embed_dim
    qs = torch.ones(3 * d, dtype=torch.float64, device=a.q_proj.weight.device)
    qs[:d] = a.scaling
    return NS(qkv=fold_ref([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], layer.self_attn_layer_norm,
                           [a.q_proj.bias, None, a.v_proj.bias]),
              qscale=qs, o=fold_ref([a.out_proj.weight], a.ln, [a.out_proj.bias]),
              w01=fold_ref([ffn[0].wi_0.weight, ffn[0].wi_1.weight], layer.final_layer_norm, [None, None], interleave=True),
              w2=fold_ref([ffn[3].weight], ffn[2], [ffn[3].bias]), lnf_eps=ffn[2].eps,
              g1=_f(layer.gamma_1), g2=_f(layer.gamma_2))


def _gemm(a, fold, epi, **kw):
    """gemm_ref of a GEMM that reads the fold ``fold`` -> (namespace, bound of y, bound of the records or None)"""
    g = R.gemm_ref(a, fold.w, epi, ln_colsum=fold.cs, ln_colsum_err=fold.cs_err, bias=fold.b, bias_err=fold.b_err, **kw)
    sb = R.TAU * g.stats_mag + g.stats_extra if g.stats is not None else None
    return g, R.TAU * g.mag + g.extra, sb


def _plain(a, w, epi, bias=None, **kw):
    """gemm_ref of a GEMM on a Linear's own weight (bf16, as the packs round it) and fp32 bias"""
    g = R.gemm_ref(a, w.detach().to(BF), epi, bias=_f(bias), **kw)
    sb = R.TAU * g.stats_mag + g.stats_extra if g.stats is not None else None
    return g, R.TAU * g.mag + g.extra, sb


def _xb(e):
    """the bf16 side output of a residual GEMM as recorded, NaN where the call wrote none"""
    xb = e.kw.get("out_bf16")
    return xb if xb is not None else torch.full(e.r.shape, float("nan"), device=e.r.device)


# ----------------------------------------------------------------------------------------------------------------------
# the log
# ----------------------------------------------------------------------------------------------------------------------
class Calls:
    """the calls of a log in order, from its first ``start``; the folds of the packs (``ln_fold``, built inside the first
    forward) are skipped"""

    def __init__(self, log, start):
        self.calls = log
        self.i = next(i for i, e in enumerate(log) if e.name == start)

    def next(self, *names):
        while True:
            e = self.calls[self.i]
            self.i += 1
            if e.name in names:
                return e
            assert e.name == "ln_fold", f"expected {names}, got {e.name}"

    def done(self):
        assert all(e.name == "ln_fold" for e in self.calls[self.i:]), "calls left over"


class Checks:
    """checks[name] = (reference, bound, dtype) and got[name] for ``stem_ref.shares``, every name under ``prefix``"""

    def __init__(self, prefix="fused"):
        self.prefix, self.chk, self.got = prefix, {}, {}

    def put(self, name, ref, bound, dt, g):
        self.chk[f"{self.prefix}.{name}"] = (ref, bound, dt)
        self.got[f"{self.prefix}.{name}"] = g

    def exact(self, name, ref, dt, g):
        ref = ref.double()
        self.put(name, ref, torch.zeros_like(ref), dt, g)


def _first(c, ck, X, eps):
    """row_stats_cast of the loop's input rows X: bf16(X) exactly, mu / rstd with the ``raw`` bounds -> LN1 of layer 0"""
    e = c.next("row_stats_cast")
    r = R.layernorm_ref(X, None, None, eps)
    ck.exact("xb0", X.to(BF), BF, e.post[1])
    ck.put("mu", r.mu, r.dmu, F32, e.post[2])
    ck.put("rstd", r.rstd, r.rel * r.rstd, F32, e.post[3])
    return dict(ln_mu=e.post[2], ln_rstd=e.post[3])


# ----------------------------------------------------------------------------------------------------------------------
# the encoder loop
# ----------------------------------------------------------------------------------------------------------------------
def encoder_checks(encoder, x0, biases, key_pad, B, S, modality, log, prefix="fused", calls=None):
    """stage checks of one ``run_fused`` from its log.  x0 fp32 [B S, d] the loop's input rows; biases: the dense fp32
    values each layer's attention adds ((H,S,S) logical columns; [] / one / one per layer, as the loop picks them), or
    for the detection layers NS(dense (H,S,S), B, S, side, pos_y, pos_x) of each layer's DetBias.
    Returns (checks, got, xs): checks[name] = (reference, bound, dtype) for ``stem_ref.shares``, xs the recorded x after
    each layer.  calls: a ``Calls`` positioned at the loop's first call, when the log goes on after the loop."""
    layers = list(encoder.layers)
    d = x0.shape[1]
    n_t = (d + 255) // 256
    xs = []
    c = calls or Calls(log, "row_stats_cast")
    ck = Checks(prefix)
    put = ck.put
    X = x0.detach().float()
    ln1 = _first(c, ck, X, layers[0].self_attn_layer_norm.eps)
    for i, layer in enumerate(layers):
        P = layer_folds(layer, modality)
        H, F_ = layer.self_attn.num_heads, layer.ffn_embed_dim
        bias = None if not biases else (biases[0] if len(biases) == 1 else biases[i])
        L = f"L{i}"
        e = c.next("gemm_ln")
        g, b, _ = _gemm(X.to(BF), P.qkv, R.EPI_STORE_BF16, colscale=P.qscale, **ln1)
        put(f"{L}.qkv", g.y, b, BF, e.r)
        qkv = e.r
        if hasattr(layer.self_attn, "rel_pos_h"):
            # detection: the decomposed terms of the unscaled q, then the attention over bias.B sequences of bias.S rows
            e = c.next("relpos_decomp_proj")
            sa = layer.self_attn
            rh, eh, rw, ew = D.proj_ref(qkv, _f(sa.rel_pos_h), _f(sa.rel_pos_w), bias.pos_y, bias.pos_x, bias.B, bias.S, H,
                                        bias.side, bias.side)
            put(f"{L}.rel_h", rh, eh, F32, e.r[0])
            put(f"{L}.rel_w", rw, ew, F32, e.r[1])
            rel_h, rel_w = e.r
            e = c.next("attention_decomp")
            f = D.decomp_attention_ref(qkv, bias.dense, rel_h, torch.zeros_like(rel_h), rel_w, torch.zeros_like(rel_w),
                                       bias.pos_y, bias.pos_x, bias.B, bias.S, H)
        else:
            e = c.next("attention", "attention_tc")
            f = R.attention_ref(qkv, bias, key_pad, B, S, H)
        put(f"{L}.att", f.out, f.out_err, BF, e.kw["out"])
        put(f"{L}.att.stats", f.stats, f.stats_err, F32, e.kw["ln_stats"])
        att, rec_a = e.kw["out"], e.kw["ln_stats"]
        e = c.next("gemm_ln")
        g, b, sb = _gemm(att, P.o, R.EPI_RESID_F32, gamma=P.g1, resid=X, ln_partial=(rec_a, H, d, layer.self_attn.ln.eps),
                         stats=True)
        put(f"{L}.x2", g.y, b, F32, e.r)
        put(f"{L}.x2.stats", g.stats, sb, F32, e.kw["stats_out"])
        x2, rec_b = e.r, e.kw["stats_out"]
        put(f"{L}.x2.xb", x2.to(BF).double(), torch.zeros_like(g.y), BF, _xb(e))
        e = c.next("gemm_ln")
        g, b, sb = _gemm(x2.to(BF), P.w01, R.EPI_GEGLU_BF16, ln_partial=(rec_b, n_t, d, layer.final_layer_norm.eps),
                         stats=True)
        put(f"{L}.u", g.y, b, BF, e.r)
        put(f"{L}.u.stats", g.stats, sb, F32, e.kw["stats_out"])
        u, rec_c = e.r, e.kw["stats_out"]
        e = c.next("gemm_ln")
        g, b, sb = _gemm(u, P.w2, R.EPI_RESID_F32, gamma=P.g2, resid=x2, ln_partial=(rec_c, 2 * ((2 * F_) // 256), F_, P.lnf_eps),
                         stats=True)
        put(f"{L}.x3", g.y, b, F32, e.r)
        put(f"{L}.x3.stats", g.stats, sb, F32, e.kw["stats_out"])
        put(f"{L}.x3.xb", e.r.to(BF).double(), torch.zeros_like(g.y), BF, _xb(e))
        X = e.r
        xs.append(X)
        if i + 1 < len(layers):
            ln1 = dict(ln_partial=(e.kw["stats_out"], n_t, d, layers[i + 1].self_attn_layer_norm.eps))
    if calls is None:
        c.done()
    return ck.chk, ck.got, xs


# ----------------------------------------------------------------------------------------------------------------------
# the detection backbone: window-major rows around the loop (OnePeace.forward)
# ----------------------------------------------------------------------------------------------------------------------
def window_major(B, side, win, dev):
    """row-major grid row of each window-major row: windows row-major, rows row-major inside a window, B grids"""
    n = side // win
    wy, wx, ly, lx = torch.meshgrid(*(torch.arange(k) for k in (n, n, win, win)), indexing="ij")
    one = ((wy * win + ly) * side + wx * win + lx).reshape(-1)
    return (torch.arange(B)[:, None] * side * side + one[None]).reshape(-1).to(dev)


def det_checks(model, x0, B, log, prefix="fused"):
    """stage checks of one ``OnePeace.forward`` whose stem gave the grid-order rows x0 [B side^2, d]: the window-major
    gather (exact), the two LUT builds of the shared table (exact: ``relpos_lut_ref`` of the resized table), the loop
    (``encoder_checks`` with each layer's LUT values and window or grid geometry), and the gather back to grid order
    (exact, against the window-major order rebuilt here).  Returns (checks, got, grid reference)."""
    from one_peace_b200.vision.det import resize_table
    ad = model.image_adapter
    side, win, S = ad.bucket_size, ad.window_size, ad.bucket_size ** 2
    dev = x0.device
    perm = window_major(B, side, win, dev)
    ck = Checks(prefix)
    c = Calls(log, "row_gather")
    e = c.next("row_gather")
    ck.exact("wmajor", x0[perm], F32, e.r)
    rows = e.r
    table = _f(ad.rel_pos_table.weight)
    luts = []
    for name, s in (("global.lut", side), ("window.lut", win)):
        e = c.next("relpos_lut_build")
        t = resize_table(table, 2 * ad.pretrain_bucket_size - 1, 2 * s - 1)
        ck.exact(name, R.relpos_lut_ref(t, torch.arange((2 * s - 1) ** 2, device=dev)), F32, e.r)
        luts.append(e.r)
    _, _, glob, wind = ad.layout(B, dev)
    refs = []
    for layer in model.encoder.layers:
        lay, lut = (wind, luts[1]) if layer.window_size > 0 else (glob, luts[0])
        cr, cc = lay["codes"]
        refs.append(NS(dense=lut[:, (cr[:lay["S"], None] - cc[None, :lay["S"]]).long()], B=lay["B"], S=lay["S"],
                       side=lay["side"], pos_y=lay["pos_y"], pos_x=lay["pos_x"]))
    chk, got, xs = encoder_checks(model.encoder, rows, refs, None, B, S, "image", log, prefix, calls=c)
    e = c.next("row_gather")
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(perm.numel(), device=dev)
    grid = xs[-1][inv]
    ck.exact("grid", grid, F32, e.r)
    c.done()
    return {**ck.chk, **chk}, {**ck.got, **got}, grid


# ----------------------------------------------------------------------------------------------------------------------
# the video backbone's layer (VideoLayer.forward_video)
# ----------------------------------------------------------------------------------------------------------------------
def frame_major(Bv, T, N, dev):
    """the frame-major row (b T + t) N + n of each (clip b, token n, frame t), in that order: sequence b N + n of T rows"""
    b, n, t = torch.meshgrid(torch.arange(Bv), torch.arange(N), torch.arange(T), indexing="ij")
    return ((b * T + t) * N + n).reshape(-1).to(dev)


def video_checks(encoder, x0, bias, Bv, T, N, log, prefix="fused"):
    """stage checks of one video ``TransformerEncoder.run`` (``VideoLayer.forward_video``) from its log.  x0 fp32
    [Bv T N, d] frame-major rows; bias the dense (H, N, N) values of the spatial attention's table.  Per layer:

      temporal  qkv = LN1(x) -> attention over the T frames of each (clip, token), H records -> a = LN_attn(o) Wo^T + bo
                -> h = gelu(a T1^T + t1) -> y, yb, rec = x + h T2^T + t2
      spatial   qkv = LN1(y) from rec -> attention over the N tokens of each frame -> a -> h = gelu(a S1^T + s1)
                -> ys = x + g1 a -> x2, xb, rec = ys + g1 (h S2^T + s2)
      joint     u, rec_c = geglu(LN2(x2) W01^T) and hm = gelu(LN2(x2) M1^T + m1), both from rec
                -> x3 = x2 + g2 (LN_ffn(u) W2^T + b2) -> x4, xb, rec = x3 + scale (hm M2^T + m2)

    Returns (checks, got, xs)."""
    layers = list(encoder.layers)
    d = x0.shape[1]
    n_t = (d + 255) // 256
    idx = frame_major(Bv, T, N, x0.device)
    c = Calls(log, "row_stats_cast")
    ck = Checks(prefix)
    put = ck.put
    X = x0.detach().float()
    ln1 = _first(c, ck, X, layers[0].self_attn_layer_norm.eps)
    xs = []
    for i, layer in enumerate(layers):
        P = layer_folds(layer, "image")
        H, F_ = layer.self_attn.num_heads, layer.ffn_embed_dim
        ta, sa, ma = layer.T_Adapter, layer.S_Adapter, layer.MLP_Adapter
        eps1, eps_in, eps2 = layer.self_attn_layer_norm.eps, layer.self_attn.ln.eps, layer.final_layer_norm.eps
        L = f"L{i}"

        def attn_pass(tag, A, ln, attend):
            """QKV of A, the attention, out_proj and the adapter's fc1 -> (a, h)"""
            e = c.next("gemm_ln")
            g, b, _ = _gemm(A.to(BF), P.qkv, R.EPI_STORE_BF16, colscale=P.qscale, **ln)
            put(f"{L}.{tag}.qkv", g.y, b, BF, e.r)
            att, rec = attend(e.r)
            e = c.next("gemm_ln")
            g, b, _ = _gemm(att, P.o, R.EPI_STORE_BF16, ln_partial=(rec, H, d, eps_in))
            put(f"{L}.{tag}.a", g.y, b, BF, e.r)
            a = e.r
            fc1 = ta.D_fc1 if tag == "t" else sa.D_fc1
            e = c.next("gemm")
            g, b, _ = _plain(a, fc1.weight, R.EPI_GELU_BF16, bias=fc1.bias)
            put(f"{L}.{tag}.h", g.y, b, BF, e.r)
            return a, e.r

        def temporal(qkv):
            e = c.next("attention_temporal")
            f = R.attention_ref(qkv[idx], None, None, Bv * N, T, H)
            put(f"{L}.t.att", f.out, f.out_err, BF, e.kw["out"][idx])
            put(f"{L}.t.att.stats", f.stats, f.stats_err, F32, e.kw["ln_stats"].view(H, -1, 2)[:, idx])
            return e.kw["out"], e.kw["ln_stats"]

        def spatial(qkv):
            e = c.next("attention", "attention_tc")
            f = R.attention_ref(qkv, bias, None, Bv * T, N, H)
            put(f"{L}.s.att", f.out, f.out_err, BF, e.kw["out"])
            put(f"{L}.s.att.stats", f.stats, f.stats_err, F32, e.kw["ln_stats"])
            return e.kw["out"], e.kw["ln_stats"]

        _, h = attn_pass("t", X, ln1, temporal)
        e = c.next("gemm_ln")
        g, b, sb = _plain(h, ta.D_fc2.weight, R.EPI_RESID_F32, bias=ta.D_fc2.bias, resid=X, stats=True)
        put(f"{L}.t.out", g.y, b, F32, e.r)
        put(f"{L}.t.out.stats", g.stats, sb, F32, e.kw["stats_out"])
        ck.exact(f"{L}.t.out.xb", e.r.to(BF), BF, _xb(e))
        Y, rec_y = e.r, e.kw["stats_out"]
        a, h = attn_pass("s", Y, dict(ln_partial=(rec_y, n_t, d, eps1)), spatial)
        e = c.next("scale_resid_fwd")
        ys, b = R.scale_resid_ref(X, a, P.g1, None)
        put(f"{L}.s.skip", ys, b, F32, e.r)
        ys = e.r
        e = c.next("gemm_ln")
        g, b, sb = _plain(h, sa.D_fc2.weight, R.EPI_RESID_F32, bias=sa.D_fc2.bias, gamma=P.g1, resid=ys, stats=True)
        put(f"{L}.x2", g.y, b, F32, e.r)
        put(f"{L}.x2.stats", g.stats, sb, F32, e.kw["stats_out"])
        ck.exact(f"{L}.x2.xb", e.r.to(BF), BF, _xb(e))
        x2, rec2 = e.r, e.kw["stats_out"]
        ln2 = (rec2, n_t, d, eps2)
        e = c.next("gemm_ln")
        g, b, sb = _gemm(x2.to(BF), P.w01, R.EPI_GEGLU_BF16, ln_partial=ln2, stats=True)
        put(f"{L}.u", g.y, b, BF, e.r)
        put(f"{L}.u.stats", g.stats, sb, F32, e.kw["stats_out"])
        u, rec_c = e.r, e.kw["stats_out"]
        e = c.next("gemm_ln")
        g, b, _ = _gemm(x2.to(BF), fold_ref([ma.D_fc1.weight], layer.final_layer_norm, [ma.D_fc1.bias]), R.EPI_GELU_BF16,
                        ln_partial=ln2)
        put(f"{L}.m.h", g.y, b, BF, e.r)
        hm = e.r
        e = c.next("gemm_ln")
        g, b, _ = _gemm(u, P.w2, R.EPI_RESID_F32, gamma=P.g2, resid=x2, ln_partial=(rec_c, 2 * ((2 * F_) // 256), F_, P.lnf_eps))
        put(f"{L}.x3", g.y, b, F32, e.r)
        x3 = e.r
        e = c.next("gemm_ln")
        scale = torch.full((d,), float(layer.scale), dtype=torch.float64, device=X.device)
        g, b, sb = _plain(hm, ma.D_fc2.weight, R.EPI_RESID_F32, bias=ma.D_fc2.bias, gamma=scale, resid=x3, stats=True)
        put(f"{L}.x4", g.y, b, F32, e.r)
        put(f"{L}.x4.stats", g.stats, sb, F32, e.kw["stats_out"])
        ck.exact(f"{L}.x4.xb", e.r.to(BF), BF, _xb(e))
        X = e.r
        xs.append(X)
        if i + 1 < len(layers):
            ln1 = dict(ln_partial=(e.kw["stats_out"], n_t, d, layers[i + 1].self_attn_layer_norm.eps))
    c.done()
    return ck.chk, ck.got, xs
