"""fp64 stage references of the encoder stack of the training path (one_peace_b200/autograd.py: ``layer_forward``,
``layer_backward``, ``EncoderStackFn``), forward and adjoint, with an error bound for every output element.

Plain PyTorch on whatever device the inputs live on; nothing here calls the extension.  Every bound is a single-kernel
bound of ``kernel_ref`` (``gemm_ref``, ``attention_ref`` / ``attention_bwd_ref`` with ``EPS_B_HALF`` for the half2
tables, ``dbias_ref``, ``center_ref``, ``layernorm_ref`` / ``layernorm_bwd_ref``, ``geglu_ref`` / ``geglu_bwd_ref``,
``scale_resid_ref`` / ``scale_resid_bwd_ref``, ``colsum_ref``, ``row_gather_ref``); nothing here adds a tolerance.

Stages and what feeds them
--------------------------
Each stage of a layer (transformer_layer.py:165-228, the per-modality FFN of :203-219) is checked on its own, from the
recorded OUTPUTS of the stages that feed it in the model, never from the arguments the code under test passed to the
kernel under check.  The kernel calls come from a log of copies taken at each call (``Snapshots`` in
tests/test_layer_ref.py), because the stack updates its gradient buffer and its bias-gradient tables in place.

  forward   h1 = LN1(x)  ->  qkv = h1 Wqkv^T + b (q scaled)  ->  [batch-major gather]  ->  att, lse = attention(qkv, bias)
            ->  [modality-major gather]  ->  a2 = LN_attn(att)  ->  o = a2 Wo^T + bo  ->  x2 = x + rs g1 o  ->  h2 = LN2(x2)
            ->  per part p, on rows(p): gl = h2 W01^T, u = geglu(gl), u2 = LN_ffn(u), f = u2 W2^T + b2  ->  x3 = x2 + rs g2 f
  adjoint   df = rs g2 dx3 (dg2; db2 fused for one part)  ->  per part: db2 = colsum(df_p) (several parts), dW2 = df_p^T u2,
            du2 = df_p W2, du = LN_ffn'(u; du2), dgl = geglu'(gl; du), dW01 = dgl^T h2_p, dh2_p = dgl W01
            ->  dx2 = dx3 + LN2'(x2; dh2)  ->  do = rs g1 dx2 (dg1, dbo)  ->  dWo = do^T a2, da2 = do Wo
            ->  datt = LN_attn'(att; da2)  ->  [batch-major gather]  ->  dqkv = attention'(qkv, att, lse; datt)
            ->  [modality-major gather]  ->  dbqkv = colsum(dqkv), dWqkv = dqkv^T h1, dh1 = dqkv Wqkv
            ->  dx = dx2 + LN1'(x; dh1)
The input x of layer i is the recorded output x3 of layer i - 1 (or, after the fused forward, the rows it kept for the
recompute, each checked to be the fused forward's recorded x after layer i - 1; the fused forward's own stages are those
of tests/fused_ref.py); dx3 of layer i is the recorded dx of layer i + 1 (or the upstream gradient).  The drop-path row
scale rs is not read from any call: it is drawn again from the RNG state saved before the stack ran, as the stack draws
it.  Row maps (parts, batch-major order) are rebuilt here from the part lengths.

Stack: the bias gradient of each table is ``dbias_ref`` over the dS of every (layer, sample) that used it, on zero (one
launch per layer through the transposed table and its fold, or straight into the dense table), then ``center_ref`` when
the tables are shared by a single-modality pass.  Every parameter's ``.grad`` and ``dx0`` are checked in their dtype.
"""
from types import SimpleNamespace as NS

import torch

import fused_ref as FR
import kernel_ref as R
from stem_ref import b64

BF, F32 = torch.bfloat16, torch.float32
SHARED = ("q_w", "q_b", "k_w", "v_w", "v_b", "o_w", "o_b", "lni_w", "lni_b", "ln1_w", "ln1_b", "ln2_w", "ln2_b", "g1",
          "g2")
FFN = ("wi0", "wi1", "lnf_w", "lnf_b", "w2", "b2")
# outputs that are column reductions (sums over rows: bias, LayerNorm and LayerScale gradients, the bias tables) and
# outputs that are exact row copies (y: the stack output is the last layer's x3; kept: the layer inputs the fused forward
# kept)
REDUCTIONS = ("q_b", "v_b", "o_b", "lni_w", "lni_b", "ln1_w", "ln1_b", "ln2_w", "ln2_b", "g1", "g2", "lnf_w", "lnf_b", "b2",
              "db2", "dbias")
EXACT = ("qkv_bm", "att_mm", "datt_bm", "dqkv_mm", "y", "kept")


def is_reduction(name):
    return name.split(".")[-1] in REDUCTIONS


def is_exact(name):
    return name.split(".")[-1] in EXACT


def shared_params(layer):
    a = layer.self_attn
    return [a.q_proj.weight, a.q_proj.bias, a.k_proj.weight, a.v_proj.weight, a.v_proj.bias, a.out_proj.weight,
            a.out_proj.bias, a.ln.weight, a.ln.bias, layer.self_attn_layer_norm.weight, layer.self_attn_layer_norm.bias,
            layer.final_layer_norm.weight, layer.final_layer_norm.bias, layer.gamma_1, layer.gamma_2]


def ffn_params(layer, m):
    f = getattr(layer, f"{m}_ffn")
    return [f[0].wi_0.weight, f[0].wi_1.weight, f[2].weight, f[2].bias, f[3].weight, f[3].bias]


def _f(t):
    return None if t is None else t.detach().float()


# ----------------------------------------------------------------------------------------------------------------------
# row layout and drop-path
# ----------------------------------------------------------------------------------------------------------------------
def layout(B, parts, dev):
    """parts [(modality, S_p)]: modality-major rows (part p owns rows off_p + b S_p + s); to_bm[r] = the modality-major row
    of batch-major row r = b S + lo_p + s, to_mm its inverse"""
    S = sum(s for _, s in parts)
    offs, los, off, lo = [], [], 0, 0
    for _, s in parts:
        offs.append(off)
        los.append(lo)
        off += B * s
        lo += s
    to_bm = torch.empty(B * S, dtype=torch.long)
    for (_, s), o, l in zip(parts, offs, los):
        for b in range(B):
            for t in range(s):
                to_bm[b * S + l + t] = o + b * s + t
    to_mm = torch.empty_like(to_bm)
    to_mm[to_bm] = torch.arange(B * S)
    return NS(B=B, S=S, M=B * S, parts=list(parts), rows=[slice(o, o + B * s) for (_, s), o in zip(parts, offs)],
              to_bm=to_bm.to(dev), to_mm=to_mm.to(dev), several=len(parts) > 1)


def row_scales(layers, lay, rng_state, dev):
    """the drop-path row scale of each layer (or None), drawn again from the RNG state saved before the stack ran: one
    torch.rand(B) per layer with drop_path_prob > 0, keep = draw < 1 - p, scale keep / (1 - p) on every row of sample b"""
    out = []
    with torch.random.fork_rng(devices=[dev] if dev.type == "cuda" else []):
        if dev.type == "cuda":
            torch.cuda.set_rng_state(rng_state, dev)
        else:
            torch.set_rng_state(rng_state)
        for layer in layers:
            if not (layer.training and layer.drop_path_prob > 0):
                out.append(None)
                continue
            kp = 1.0 - layer.drop_path_prob
            per = (torch.rand(lay.B, device=dev) < kp).float() / kp
            out.append(torch.cat([per.repeat_interleave(s) for _, s in lay.parts]))
    return out


# ----------------------------------------------------------------------------------------------------------------------
# the recorded kernel calls of one layer
# ----------------------------------------------------------------------------------------------------------------------
def segments(log, lay):
    """[(kind, calls)] for each layer pass in a log of ``Snapshots`` entries: 'fwd' runs from its first layernorm to its
    second scale_resid_fwd, 'bwd' from its first scale_resid_bwd to its last layernorm_bwd (one per part, then LN2,
    the attention's LayerNorm and LN1).  Stack-level calls between them (bias-table transposes, folds, centring) belong
    to no segment."""
    out, cur, kind, n = [], None, None, 0
    for e in log:
        if cur is None:
            if e.name not in ("layernorm", "scale_resid_bwd"):
                continue
            kind, cur, n = ("fwd" if e.name == "layernorm" else "bwd"), [], 0
        cur.append(e)
        n += e.name == ("scale_resid_fwd" if kind == "fwd" else "layernorm_bwd")
        if n == (2 if kind == "fwd" else len(lay.parts) + 3):
            out.append((kind, cur))
            cur = None
    assert cur is None, "a layer pass ends early"
    return out


class Calls:
    """the calls of one segment in order; ``transpose_bf16`` (the K-major copies of ``_dw``) is skipped"""

    def __init__(self, calls):
        self.calls, self.i = calls, 0

    def next(self, *names):
        while True:
            e = self.calls[self.i]
            self.i += 1
            if e.name in names:
                return e
            assert e.name == "transpose_bf16", f"expected {names}, got {e.name}"

    def done(self):
        assert all(e.name == "transpose_bf16" for e in self.calls[self.i:]), "calls left over"


def parse_fwd(calls, lay):
    c = Calls(calls)
    r = NS()
    r.h1 = c.next("layernorm").r
    r.qkv = c.next("gemm").r
    r.qkv_bm = c.next("row_gather").r if lay.several else r.qkv
    e = c.next("attention", "attention_tc")
    r.att, r.lse = e.r, e.kw["lse"]
    r.att_mm = c.next("row_gather").r if lay.several else r.att
    r.a2 = c.next("layernorm").r
    r.o = c.next("gemm").r
    r.x2 = c.next("scale_resid_fwd").r
    r.h2 = c.next("layernorm").r
    r.gl, r.u, r.u2, fs = [], [], [], []
    for _ in lay.parts:
        r.gl.append(c.next("gemm").r)
        r.u.append(c.next("geglu_fwd").r)
        r.u2.append(c.next("layernorm").r)
        fs.append(c.next("gemm").r)
    r.f = torch.cat(fs)
    r.x3 = c.next("scale_resid_fwd").r
    c.done()
    return r


def parse_bwd(calls, lay):
    c = Calls(calls)
    r = NS()
    e = c.next("scale_resid_bwd")
    r.df, r.dg2, r.db2 = e.r, e.kw.get("dgamma"), e.kw.get("dbias")
    r.ffn = []
    for _ in lay.parts:
        p = NS()
        p.db2 = c.next("colsum").r if lay.several else None
        c.next("gemm_t", "gemm")                                      # dW2: checked as .grad
        p.du2 = c.next("gemm_t").r
        e = c.next("layernorm_bwd")
        p.du = e.r
        p.dgl = c.next("geglu_bwd").r
        c.next("gemm_t", "gemm")                                      # dW01: checked as .grad
        p.dh2 = c.next("gemm_t").r
        r.ffn.append(p)
    r.dh2 = torch.cat([p.dh2 for p in r.ffn])
    r.dx2 = c.next("layernorm_bwd").r
    e = c.next("scale_resid_bwd")
    r.do = e.r
    c.next("gemm_t", "gemm")                                          # dWo
    r.da2 = c.next("gemm_t").r
    r.datt = c.next("layernorm_bwd").r
    r.datt_bm = c.next("row_gather").r if lay.several else r.datt
    e = c.next("attention_bwd", "attention_bwd_t")
    r.dqkv_bm, r.transposed = e.r, e.name == "attention_bwd_t"
    r.dqkv = c.next("row_gather").r if lay.several else r.dqkv_bm
    r.dbqkv = c.next("colsum").r
    c.next("gemm_t", "gemm")                                          # dWqkv
    r.dh1 = c.next("gemm_t").r
    r.dx = c.next("layernorm_bwd").r
    c.done()
    return r


# ----------------------------------------------------------------------------------------------------------------------
# one layer
# ----------------------------------------------------------------------------------------------------------------------
def _gemm(a, w, dt=BF, **kw):
    """(y, bound) of gemm_ref: a [M, K] @ w[N, K]^T"""
    g = R.gemm_ref(a, w, R.EPI_STORE_BF16 if dt == BF else R.EPI_STORE_F32, **kw)
    return g.y, R.TAU * g.mag + g.extra


def _dw(dy, x):
    """dW = dy^T x over the rows"""
    return _gemm(dy.t(), x.t())


def _ln(x, w, b, eps):
    r = R.layernorm_ref(x, _f(w), _f(b), eps)
    return r.y, r.err


def _gather(src, idx):
    """exact row copy: (reference, zero bound)"""
    v = R.row_gather_ref(src, idx, src.dtype).double()
    return v, torch.zeros_like(v)


def packs(layer, modalities):
    """the reference's bf16 weights and fp32 vectors, from the layer's parameters"""
    a = layer.self_attn
    d = layer.embed_dim
    dev = a.q_proj.weight.device
    P = NS(wqkv=torch.cat([b64(a.q_proj.weight), b64(a.k_proj.weight), b64(a.v_proj.weight)]),
           bqkv=torch.cat([_f(a.q_proj.bias), torch.zeros(d, device=dev), _f(a.v_proj.bias)]),
           qscale=torch.cat([torch.full((d,), a.scaling, device=dev), torch.ones(2 * d, device=dev)]),
           wo=b64(a.out_proj.weight), bo=_f(a.out_proj.bias), g1=_f(layer.gamma_1), g2=_f(layer.gamma_2), ffn={})
    for m in modalities:
        f = getattr(layer, f"{m}_ffn")
        P.ffn[m] = NS(w01=torch.cat([b64(f[0].wi_0.weight), b64(f[0].wi_1.weight)]), w2=b64(f[3].weight),
                      b2=_f(f[3].bias), lnf=f[2])
    return P


def layer_fwd_checks(layer, X, r, lay, bias, key_pad):
    """stage checks of one layer forward: r = parse_fwd of its calls, X its fp32 input rows, bias the dense values the
    attention adds ((H,S,S) or (B,H,S,S), logical columns)"""
    P = packs(layer, [m for m, _ in lay.parts])
    a = layer.self_attn
    H = a.num_heads
    chk = {}
    chk["h1"] = _ln(X, layer.self_attn_layer_norm.weight, layer.self_attn_layer_norm.bias,
                    layer.self_attn_layer_norm.eps) + (BF,)
    chk["qkv"] = _gemm(r.h1, P.wqkv, bias=P.bqkv, colscale=P.qscale) + (BF,)
    if lay.several:
        chk["qkv_bm"] = _gather(r.qkv, lay.to_bm) + (BF,)
    f = R.attention_ref(r.qkv_bm, bias, key_pad, lay.B, lay.S, H)
    chk["att"] = (f.out, f.out_err, BF)
    chk["lse"] = (f.lse.reshape(-1), f.dlse.reshape(-1), F32)
    if lay.several:
        chk["att_mm"] = _gather(r.att, lay.to_mm) + (BF,)
    chk["a2"] = _ln(r.att_mm, a.ln.weight, a.ln.bias, a.ln.eps) + (BF,)
    chk["o"] = _gemm(r.a2, P.wo, bias=P.bo) + (BF,)
    return chk, P


def fwd_got(r):
    """the recorded forward outputs of parse_fwd under the names of ``layer_checks``"""
    g = {k: v for k, v in vars(r).items() if k not in ("gl", "u", "u2")}
    for pi in range(len(r.gl)):
        g[f"gl_{pi}"], g[f"u_{pi}"], g[f"u2_{pi}"] = r.gl[pi], r.u[pi], r.u2[pi]
    return g


def layer_checks(layer, X, r, lay, bias, key_pad, rs):
    """forward stage checks of one layer (``layer_fwd_checks`` and the residual / FFN stages)"""
    chk, P = layer_fwd_checks(layer, X, r, lay, bias, key_pad)
    chk["x2"] = R.scale_resid_ref(X, r.o, P.g1, rs) + (F32,)
    ln2 = layer.final_layer_norm
    chk["h2"] = _ln(r.x2, ln2.weight, ln2.bias, ln2.eps) + (BF,)
    fr, fb = [], []
    for pi, (m, _) in enumerate(lay.parts):
        q = P.ffn[m]
        chk[f"gl_{pi}"] = _gemm(r.h2[lay.rows[pi]], q.w01) + (BF,)
        chk[f"u_{pi}"] = R.geglu_ref(r.gl[pi]) + (BF,)
        chk[f"u2_{pi}"] = _ln(r.u[pi], q.lnf.weight, q.lnf.bias, q.lnf.eps) + (BF,)
        y, e = _gemm(r.u2[pi], q.w2, bias=q.b2)
        fr.append(y)
        fb.append(e)
    chk["f"] = (torch.cat(fr), torch.cat(fb), BF)
    chk["x3"] = R.scale_resid_ref(r.x2, r.f, P.g2, rs) + (F32,)
    return chk


def layer_bwd_checks(layer, X, r, b, dxo, lay, bias, key_pad, rs, eps_b):
    """stage checks of one layer adjoint and the reference gradients of its parameters.  r: parse_fwd of the forward
    the adjoint read (kept or recomputed), b: parse_bwd of its calls, dxo: the gradient of its output (the recorded dx of
    the layer above, or the upstream gradient).  Returns (checks, got, grads, attention_bwd_ref namespace); grads[name] =
    (reference, bound) in SHARED / FFN order names."""
    P = packs(layer, [m for m, _ in lay.parts])
    a = layer.self_attn
    H, F_ = a.num_heads, layer.ffn_embed_dim
    chk, got, grads = {}, {}, {}
    s = R.scale_resid_bwd_ref(dxo, r.f, P.g2, rs)
    chk["df"] = (s.d_o, s.d_o_err, BF)
    got["df"] = b.df
    if P.g2 is not None:
        grads["g2"] = (s.dgamma, s.dgamma_err)
    for pi, (m, _) in enumerate(lay.parts):
        q, bp = P.ffn[m], b.ffn[pi]
        rows = lay.rows[pi]
        dfp = b.df[rows]
        if lay.several:
            grads[f"{m}.b2"] = R.colsum_ref(dfp)
        else:
            grads[f"{m}.b2"] = (s.dbias, s.dbias_err)
        grads[f"{m}.w2"] = _dw(dfp, r.u2[pi])
        chk[f"du2_{pi}"] = _gemm(dfp, q.w2.t()) + (BF,)
        got[f"du2_{pi}"] = bp.du2
        lb = R.layernorm_bwd_ref(r.u[pi], bp.du2, _f(q.lnf.weight), _f(q.lnf.bias), q.lnf.eps)
        chk[f"du_{pi}"] = (lb.dx, lb.dx_err, BF)
        got[f"du_{pi}"] = bp.du
        grads[f"{m}.lnf_w"], grads[f"{m}.lnf_b"] = (lb.dgamma, lb.dgamma_err), (lb.dbeta, lb.dbeta_err)
        chk[f"dgl_{pi}"] = R.geglu_bwd_ref(r.gl[pi], bp.du) + (BF,)
        got[f"dgl_{pi}"] = bp.dgl
        w01, e01 = _dw(bp.dgl, r.h2[rows])
        grads[f"{m}.wi0"], grads[f"{m}.wi1"] = (w01[:F_], e01[:F_]), (w01[F_:], e01[F_:])
        chk[f"dh2_{pi}"] = _gemm(bp.dgl, q.w01.t()) + (BF,)
        got[f"dh2_{pi}"] = bp.dh2
    ln2 = layer.final_layer_norm
    lb = R.layernorm_bwd_ref(r.x2, b.dh2, _f(ln2.weight), _f(ln2.bias), ln2.eps, old=dxo)
    chk["dx2"], got["dx2"] = (lb.dx, lb.dx_err, F32), b.dx2
    grads["ln2_w"], grads["ln2_b"] = (lb.dgamma, lb.dgamma_err), (lb.dbeta, lb.dbeta_err)
    s = R.scale_resid_bwd_ref(b.dx2, r.o, P.g1, rs)
    chk["do"], got["do"] = (s.d_o, s.d_o_err, BF), b.do
    if P.g1 is not None:
        grads["g1"] = (s.dgamma, s.dgamma_err)
    grads["o_b"] = (s.dbias, s.dbias_err)
    grads["o_w"] = _dw(b.do, r.a2)
    chk["da2"], got["da2"] = _gemm(b.do, P.wo.t()) + (BF,), b.da2
    lb = R.layernorm_bwd_ref(r.att_mm, b.da2, _f(a.ln.weight), _f(a.ln.bias), a.ln.eps)
    chk["datt"], got["datt"] = (lb.dx, lb.dx_err, BF), b.datt
    grads["lni_w"], grads["lni_b"] = (lb.dgamma, lb.dgamma_err), (lb.dbeta, lb.dbeta_err)
    if lay.several:
        chk["datt_bm"], got["datt_bm"] = _gather(b.datt, lay.to_bm) + (BF,), b.datt_bm
    br = R.attention_bwd_ref(r.qkv_bm, r.att, b.datt_bm, r.lse, bias, key_pad, lay.B, lay.S, H, a.scaling, eps_b=eps_b)
    chk["dqkv"], got["dqkv"] = (br.dqkv, br.dqkv_err, BF), b.dqkv_bm
    if lay.several:
        chk["dqkv_mm"], got["dqkv_mm"] = _gather(b.dqkv_bm, lay.to_mm) + (BF,), b.dqkv
    d = layer.embed_dim
    cs, ce = R.colsum_ref(b.dqkv)
    grads["q_b"], grads["v_b"] = (cs[:d], ce[:d]), (cs[2 * d:], ce[2 * d:])
    wq, eq = _dw(b.dqkv, r.h1)
    grads["q_w"], grads["k_w"], grads["v_w"] = (wq[:d], eq[:d]), (wq[d:2 * d], eq[d:2 * d]), (wq[2 * d:], eq[2 * d:])
    chk["dh1"], got["dh1"] = _gemm(b.dqkv, P.wqkv.t()) + (BF,), b.dh1
    ln1 = layer.self_attn_layer_norm
    lb = R.layernorm_bwd_ref(X, b.dh1, _f(ln1.weight), _f(ln1.bias), ln1.eps, old=b.dx2)
    chk["dx"], got["dx"] = (lb.dx, lb.dx_err, F32), b.dx
    grads["ln1_w"], grads["ln1_b"] = (lb.dgamma, lb.dgamma_err), (lb.dbeta, lb.dbeta_err)
    return chk, got, grads, br


# ----------------------------------------------------------------------------------------------------------------------
# the stack
# ----------------------------------------------------------------------------------------------------------------------
def bias_grad_refs(biases, brs, shared_tables, S):
    """reference gradient and bound of each bias input (the stack's order): brs[i] is layer i's attention_bwd_ref.  A
    batch-shared table gathers dS over every (layer, sample) that used it, a per-sample canvas over the layers; centred
    when the tables are shared by a single-modality pass.  Padding columns [S, S_pad) stay zero."""
    out = []
    for t, bias in enumerate(biases):
        users = [br for i, br in enumerate(brs) if len(biases) == 1 or i == t]
        per_sample = bias.dim() == 4 and bias.shape[0] > 1
        dS = torch.stack([br.dS for br in users]) if per_sample else torch.cat([br.dS for br in users])
        dS_err = torch.stack([br.dS_err for br in users]) if per_sample else torch.cat([br.dS_err for br in users])
        init = torch.zeros(dS.shape[1:], dtype=torch.float64, device=dS.device)
        v, e = R.dbias_ref(NS(dS=dS, dS_err=dS_err), init)
        if shared_tables:
            v, e = R.center_ref(v, e)
        pad = bias.shape[-1] - S
        v = torch.nn.functional.pad(v, (0, pad)).reshape(bias.shape)
        e = torch.nn.functional.pad(e, (0, pad)).reshape(bias.shape)
        out.append((v, e))
    return out


def stack_checks(encoder, lay, x0, dy, y, biases, key_pad, rs, fwd_log, bwd_log, shared_tables, kept_inputs=None):
    """every check of one EncoderStackFn forward and backward.  fwd_log / bwd_log: ``Snapshots`` entries of the forward
    and of the backward; biases: the stack's bias inputs (leaves whose .grad is checked); rs: ``row_scales``;
    kept_inputs: the layer inputs the fused forward kept for the recompute (None when the forward ran layer by layer; the
    fused forward's calls are then checked from fwd_log by ``fused_ref.encoder_checks``).
    Returns (checks, got) for ``stem_ref.shares``."""
    layers = list(encoder.layers)
    L, d = len(layers), x0.shape[-1]
    chk, got = {}, {}
    fw = [parse_fwd(c, lay) for k, c in segments(fwd_log, lay) if k == "fwd"]
    seg = segments(bwd_log, lay)
    recompute = [parse_fwd(c, lay) for k, c in seg if k == "fwd"]
    bw = [parse_bwd(c, lay) for k, c in seg if k == "bwd"][::-1]          # layer order
    assert len(bw) == L and len(fw) in (0, L) and len(recompute) in (0, L)
    assert fw or kept_inputs is not None
    recompute = recompute[::-1]
    bias_i = [None if not biases else (biases[0] if len(biases) == 1 else biases[i]) for i in range(L)]
    logical = [None if b is None else (b[0] if b.dim() == 4 and b.shape[0] == 1 else b)[..., :lay.S].detach()
               for b in bias_i]
    transposed = bw[0].transposed
    if not fw:
        # the fused-LayerNorm forward: its stages from its own log (fused_ref), each kept input the recorded x after the
        # layer below (exactly), the output the last recorded x
        chk, got, xs = FR.encoder_checks(encoder, x0.detach().reshape(-1, d), logical if biases else [], key_pad, lay.B,
                                         lay.S, lay.parts[0][0], fwd_log)
        for i, t in enumerate(kept_inputs):
            ref = (x0.detach().reshape(-1, d) if i == 0 else xs[i - 1]).double()
            chk[f"L{i}.kept"], got[f"L{i}.kept"] = (ref, torch.zeros_like(ref), F32), t
        chk["y"] = (xs[-1].double(), torch.zeros_like(xs[-1], dtype=torch.float64), F32)
        got["y"] = y.detach().reshape(-1, d)
    X = [x0.detach().reshape(-1, d)] + ([f.x3 for f in fw[:-1]] if fw else [t for t in kept_inputs[1:]])

    def add(prefix, c, g):
        for k in c:
            chk[f"{prefix}.{k}"] = c[k]
            got[f"{prefix}.{k}"] = g[k]
    for i in range(L):
        if fw:
            add(f"L{i}.fwd", layer_checks(layers[i], X[i], fw[i], lay, logical[i], key_pad, rs[i]), fwd_got(fw[i]))
        if recompute:
            add(f"L{i}.recompute", layer_checks(layers[i], X[i], recompute[i], lay, logical[i], key_pad, rs[i]),
                fwd_got(recompute[i]))
    if fw:
        chk["y"] = (fw[-1].x3.double(), torch.zeros_like(fw[-1].x3, dtype=torch.float64), F32)
        got["y"] = y.detach().reshape(-1, d)
    brs = [None] * L
    dxo = dy.detach().float().reshape(-1, d)
    for i in reversed(range(L)):
        r = (recompute or fw)[i]
        c, g, grads, brs[i] = layer_bwd_checks(layers[i], X[i], r, bw[i], dxo, lay, logical[i], key_pad, rs[i],
                                               R.EPS_B_HALF if transposed else None)
        add(f"L{i}", c, g)
        prm = dict(zip(SHARED, shared_params(layers[i])))
        for m, _ in lay.parts:
            prm.update({f"{m}.{k}": p for k, p in zip(FFN, ffn_params(layers[i], m))})
        for k, (v, e) in grads.items():
            chk[f"L{i}.{k}"] = (v, e, prm[k].dtype)
            got[f"L{i}.{k}"] = prm[k].grad
        dxo = bw[i].dx
    chk["dx0"] = (chk["L0.dx"][0], chk["L0.dx"][1], F32)
    got["dx0"] = x0.grad.reshape(-1, d)
    for t, (v, e) in enumerate(bias_grad_refs(biases, brs, shared_tables, lay.S)):
        chk[f"bias{t}.dbias"] = (v, e, F32)
        got[f"bias{t}.dbias"] = biases[t].grad
    return chk, got
