"""Training path: hand-written backward of the modality-shared encoder, wired into ``torch.autograd``.

The reference trains through torch autograd (transformer_layer.py:165-228, multihead_attention.py:103-126, with
``checkpoint_activations`` in the 4B recipes).  Here every adjoint is an sm_90a kernel behind the C-ABI
(csrc/backward.cu, csrc/attention_bwd.cu + the wgmma GEMM for all dX / dW products); autograd only carries the
graph edges between ``Function`` nodes:

    TextEmbedFn / ImageEmbedFn  ->  EncoderStackFn (L layers, activations kept or recomputed)  ->  HeadFn  ->  criterion
    RelPosBiasFn (table -> dense (H,S,S_pad) bias, shared by the layers) ----^

EncoderStackFn runs every encoder and decoder pass: single-modality passes (run_encoder_stack: fine-tuning, contrastive
steps) and the concatenated 'vl' / 'al' sequences, preserve_ids student passes and the decoder of pretraining
(run_general_stack, with the Functions of autograd_general.py around it).  Its rows are laid out by a SeqLayout, and one
layer_forward / layer_backward pair serves both.

Activation policy (keep_activations below): when the whole stack's activations fit in half of the free HBM they are KEPT (the
training forward then runs layer_forward, the un-fused LayerNorm form, whose normalised operands the dW GEMMs need) and the
backward is the adjoint only; otherwise the forward keeps each layer's fp32 input rows, running the fused-LayerNorm loop of
inference (TransformerEncoder.run_fused) where EncoderStackFn allows it and layer_forward elsewhere, and the backward
re-runs layer_forward for one layer at a time before its adjoint — the reference's checkpoint_wrapper.  dW = dY^T X is an
M-reduction whose operands the wgmma GEMM reads in place as MN-major tiles (opb_gemm_bf16_t); dX = dY W reads the forward
weight the same way: nothing is transposed in memory.  Attention backward: csrc/attention_bwd.cu (mma.sync; S <= 224:
transposed bias tables shared by the stack).

torch is used here for what the task calls plumbing only: allocation, dtype / layout copies (`.to`, `cat`, slicing
`copy_`), the drop-path Bernoulli draw, and autograd's own accumulation of gradients that reach a tensor twice.
"""
import torch

from . import kernels as K
from .components import PackCache, bf16, f32


class TrainBias:
    """Relative-position bias of a training forward: `dense` = autograd-tracked fp32 (H,S,S_pad) tensor (what the
    backward kernels read and what receives the gradient), `fast` = the same values as a kernels.RelPosBias in LUT
    form for the attention kernel (None when S > kernels.ATTN_TC_MAX_S).  `lut` is always None, so that code reading a
    kernels.RelPosBias sees a TrainBias as one in dense form."""

    def __init__(self, dense, fast=None):
        self.dense, self.fast, self.lut = dense, fast, None


def _pad8(n):
    return (n + 7) // 8 * 8


def keep_activations(n_layers, rows, d, ffn, device, row_bytes=None):
    """Activation policy of the training stack.  The reference wraps every layer in checkpoint_wrapper (one_peace_pretrain.py
    :83-91, `checkpoint_activations` in the 4B recipes) because 12,608 rows x 40 layers of layer activations (1.05 GB per layer
    at d = 1536, ffn = 6144) do not fit an 80 GB part next to the model.  When the activations of the whole
    stack fit in half of the memory that is free right now they are KEPT and the backward skips the recompute (a quarter of
    the step's GEMM work); otherwise each layer is recomputed while its adjoint runs, as the reference does.
    OPB_ACTIVATIONS=keep | recompute overrides the choice (tests exercise both).  `row_bytes`: the saved bytes per row of
    a layer whose activations differ from the encoder layer's (the video layer's)."""
    mode = __import__("os").environ.get("OPB_ACTIVATIONS", "auto")
    if mode in ("keep", "recompute"):
        return mode == "keep"
    key = (n_layers, rows, d, ffn, row_bytes)
    if torch.cuda.is_current_stream_capturing():               # no driver queries under capture: reuse the warm-up's decision
        return _POLICY.get(key, False)
    if row_bytes is None:
        row_bytes = 22 * d + 8 * ffn + 64                      # bytes: h1 qkv att a2 o x2(fp32) h2 f | gl u u2 | lse
    need = n_layers * rows * row_bytes
    free, _ = torch.cuda.mem_get_info(device)
    _POLICY[key] = need < free // 2
    return _POLICY[key]


_POLICY = {}


def _tr(x):
    """bf16 [M, n] -> [n, pad8(M)]: K-major operand of an M-reduction GEMM (zero columns past M)."""
    M, n = x.shape
    if M % 8 == 0:
        return K.transpose_bf16(x)
    xp = torch.zeros(_pad8(M), n, dtype=x.dtype, device=x.device)
    xp[:M].copy_(x)
    return K.transpose_bf16(xp)


def _dw(dy, x, dtype):
    """dW [N, Kw] = dy[M, N]^T x[M, Kw]  (fp32 accumulate; stored in the parameter's dtype).  A reduction over the M rows:
    both operands are MN-major for the tensor cores and are read in place (opb_gemm_bf16_t) when their rows are 16-byte
    aligned; otherwise they go through transposed copies and the K-major GEMM."""
    out = torch.empty(dy.shape[1], x.shape[1], dtype=torch.float32 if dtype == torch.float32 else torch.bfloat16,
                      device=dy.device)
    epi = K.EPI_STORE_F32 if out.dtype == torch.float32 else K.EPI_STORE_BF16
    if dy.shape[1] % 8 == 0 and x.shape[1] % 8 == 0 and dy.stride(0) % 8 == 0 and x.stride(0) % 8 == 0 \
            and dy.data_ptr() % 16 == 0 and x.data_ptr() % 16 == 0:
        K.gemm_t(dy, x, epi, out, a_mn=True, b_mn=True)
    else:
        K.gemm(_tr(dy), _tr(x), epi, out)
    return out if out.dtype == dtype else out.to(dtype)


def _dx(dy, w, n_out, out=None):
    """dX [M, n_out] = dy[M, N] W[N, n_out]: a contraction over the OUTPUT features of the Linear, for which the weight
    [N, n_out] as stored is the MN-major B operand (opb_gemm_bf16_t): no transposed weight copies are kept."""
    if out is None:
        out = torch.empty(dy.shape[0], n_out, dtype=torch.bfloat16, device=dy.device)
    K.gemm_t(dy, w, K.EPI_STORE_BF16 if out.dtype == torch.bfloat16 else K.EPI_STORE_F32, out, b_mn=True)
    return out


# ----------------------------------------------------------------------------------------------------------------
# row layout
# ----------------------------------------------------------------------------------------------------------------
class SeqLayout:
    """parts = [(modality, S_p), ...] in sequence order (text first, transformer_encoder.py:127-134).

    Rows are MODALITY-MAJOR: part p owns the contiguous rows [off_p, off_p + B*S_p) of the residual stream, row =
    off_p + b*S_p + s.  Every GEMM (shared QKV / out_proj over all rows, per-modality GeGLU / fc2 over one part's rows —
    transformer_layer.py:210-217) then runs on a plain contiguous row range.  Only attention needs a sample's tokens
    adjacent (batch-major rows b*S + lo_p + s): with several parts the QKV rows are permuted there and the attention output
    back by `opb_row_gather` (two 16-byte-vector copies per layer).  A single-modality pass is one part, and both orders
    coincide (to_bm = to_mm = None)."""

    def __init__(self, B, parts, device):
        self.B, self.parts = B, list(parts)
        self.S = sum(s for _, s in parts)
        self.M = B * self.S
        self.offs, self.los = [], []
        off = lo = 0
        for _, s in parts:
            self.offs.append(off)
            self.los.append(lo)
            off += B * s
            lo += s
        self.to_bm = self.to_mm = None
        if len(parts) > 1:
            # batch-major row (b, lo_p + s)  <-  modality-major row off_p + b * S_p + s
            cols = []
            for (_, s), off in zip(parts, self.offs):
                cols.append(off + torch.arange(B, device=device)[:, None] * s + torch.arange(s, device=device)[None, :])
            self.to_bm = torch.cat(cols, dim=1).reshape(-1).contiguous()              # [B*S]: source mm row of every bm row
            inv = torch.empty_like(self.to_bm)
            inv[self.to_bm] = torch.arange(self.M, device=device)
            self.to_mm = inv.contiguous()                                             # source bm row of every mm row

    def rows(self, p):
        return slice(self.offs[p], self.offs[p] + self.B * self.parts[p][1])

    def row_scale(self, per_sample):
        """per-sample fp32 [B] -> per-row fp32 [M] in modality-major order (drop-path, transformer_layer.py:80-86)."""
        return torch.cat([per_sample.repeat_interleave(s) for _, s in self.parts]).contiguous()


# ----------------------------------------------------------------------------------------------------------------
# one encoder layer
# ----------------------------------------------------------------------------------------------------------------
def shared_params(layer):
    """The 15 modality-shared parameters of a layer, in the order layer_backward returns their gradients; gamma_1 /
    gamma_2 are None when the layer was built with use_layer_scale=False (the pretraining decoder, pretrain_vl_3B.yaml:168)."""
    a = layer.self_attn
    return [a.q_proj.weight, a.q_proj.bias, a.k_proj.weight, a.v_proj.weight, a.v_proj.bias, a.out_proj.weight,
            a.out_proj.bias, a.ln.weight, a.ln.bias, layer.self_attn_layer_norm.weight, layer.self_attn_layer_norm.bias,
            layer.final_layer_norm.weight, layer.final_layer_norm.bias, layer.gamma_1, layer.gamma_2]


def ffn_params(layer, modality):
    """The 6 parameters of one modality's FFN, in the order layer_backward returns their gradients."""
    ffn = getattr(layer, f"{modality}_ffn")
    layer.check_structure()
    return [ffn[0].wi_0.weight, ffn[0].wi_1.weight, ffn[2].weight, ffn[2].bias, ffn[3].weight, ffn[3].bias]


def shared_train_pack(layer):
    """bf16 operands of the modality-shared half of a layer (one orientation: dX reads W as an MN-major operand), rebuilt
    after each optimizer step."""
    cache = layer._cache.setdefault("_train_shared", PackCache())
    ps = shared_params(layer)

    def build():
        d = layer.embed_dim
        dev = ps[0].device
        wqkv = torch.cat([bf16(ps[0]), bf16(ps[2]), bf16(ps[3])], 0).contiguous()
        bqkv = torch.cat([f32(ps[1]), torch.zeros(d, device=dev), f32(ps[4])]).contiguous()
        qs = torch.ones(3 * d, device=dev)
        qs[:d] = layer.self_attn.scaling
        wo = bf16(ps[5])
        return dict(wqkv=wqkv, bqkv=bqkv, qscale=qs, wo=wo,
                    bo=f32(ps[6]), lni_w=f32(ps[7]), lni_b=f32(ps[8]), ln1_w=f32(ps[9]), ln1_b=f32(ps[10]),
                    ln2_w=f32(ps[11]), ln2_b=f32(ps[12]), g1=f32(ps[13]) if ps[13] is not None else None,
                    g2=f32(ps[14]) if ps[14] is not None else None)
    return cache.get([q for q in ps if q is not None], build)


def ffn_train_pack(layer, modality):
    cache = layer._cache.setdefault("_train_ffn_" + modality, PackCache())
    ps = ffn_params(layer, modality)

    def build():
        w01 = torch.cat([bf16(ps[0]), bf16(ps[1])], 0).contiguous()      # [g | l] halves, not tile-interleaved
        w2 = bf16(ps[4])
        return dict(w01=w01, lnf_w=f32(ps[2]), lnf_b=f32(ps[3]), w2=w2,
                    b2=f32(ps[5]), lnf_eps=getattr(layer, f"{modality}_ffn")[2].eps)
    return cache.get(ps, build)


def layer_forward(layer, x, lay, bias, key_pad, row_scale, keep, fast_bias=None):
    """x fp32 [M, d] (rows laid out by `lay`) -> (x_out fp32 [M, d], saved activations or None).  Un-fused LayerNorm form of
    transformer_layer.py:165-228 with the per-modality FFN of :203-219, so every normalised operand of the dW GEMMs is in HBM.
    bias: dense fp32 (H,S,S_pad) / (B,H,S,S_pad) or None; fast_bias: the same values as a kernels.RelPosBias in LUT form, or
    None; key_pad uint8 (B,S) batch-major or None; row_scale [M] = drop-path keep mask / keep_prob (:80-86) or None."""
    p = shared_train_pack(layer)
    d, F_, H = layer.embed_dim, layer.ffn_embed_dim, layer.self_attn.num_heads
    B, S, M = lay.B, lay.S, lay.M
    dev = x.device

    def e(rows, n):
        return torch.empty(rows, n, dtype=torch.bfloat16, device=dev)
    h1 = K.layernorm(x, p["ln1_w"], p["ln1_b"], e(M, d), eps=layer.self_attn_layer_norm.eps)
    qkv = K.gemm(h1, p["wqkv"], K.EPI_STORE_BF16, e(M, 3 * d), bias=p["bqkv"], colscale=p["qscale"])
    if lay.to_bm is not None:
        qkv = K.row_gather(qkv, lay.to_bm)
    lse = torch.empty(B * H * S, dtype=torch.float32, device=dev)
    if fast_bias is not None:
        att = K.attention_tc(qkv, fast_bias, key_pad, B, S, H, out=e(M, d), lse=lse)
    else:
        att = K.attention(qkv, bias, key_pad, B, S, H, out=e(M, d), lse=lse)
    att_mm = K.row_gather(att, lay.to_mm) if lay.to_mm is not None else att
    a2 = K.layernorm(att_mm, p["lni_w"], p["lni_b"], e(M, d), eps=layer.self_attn.ln.eps)
    o = K.gemm(a2, p["wo"], K.EPI_STORE_BF16, e(M, d), bias=p["bo"])
    x2 = K.scale_resid_fwd(x, o, p["g1"], row_scale, torch.empty_like(x))
    h2 = K.layernorm(x2, p["ln2_w"], p["ln2_b"], e(M, d), eps=layer.final_layer_norm.eps)
    f = e(M, d)
    ffn_saved = []
    for pi, (m, _) in enumerate(lay.parts):
        fp = ffn_train_pack(layer, m)
        rs = lay.rows(pi)
        n = rs.stop - rs.start
        gl = K.gemm(h2[rs], fp["w01"], K.EPI_STORE_BF16, e(n, 2 * F_))
        u = K.geglu_fwd(gl, e(n, F_))
        u2 = K.layernorm(u, fp["lnf_w"], fp["lnf_b"], e(n, F_), eps=fp["lnf_eps"])
        K.gemm(u2, fp["w2"], K.EPI_STORE_BF16, f[rs], bias=fp["b2"])
        ffn_saved.append(dict(gl=gl, u=u, u2=u2) if keep else None)
    x3 = K.scale_resid_fwd(x2, f, p["g2"], row_scale, torch.empty_like(x))
    saved = dict(h1=h1, qkv=qkv, lse=lse, att=att, att_mm=att_mm, a2=a2, o=o, x2=x2, h2=h2, f=f, ffn=ffn_saved) if keep else None
    return x3, saved


def layer_backward(layer, x, s, dx, lay, bias, dbias, key_pad, row_scale, bias_t=None, dbias_t=None):
    """Adjoint of layer_forward.  `dx` (fp32 [M, d]) holds dL/dx_out on entry and dL/dx_in on return (in place); `dbias`
    (shaped like `bias`, or None) accumulates the relative-position-bias gradient, or `dbias_t` does when the transposed
    tables `bias_t` are given (S <= 224; the caller folds dbias_t back).  Returns the 15 shared_params gradients, then the 6
    ffn_params gradients of each part, in each parameter's dtype (None for an absent gamma)."""
    p = shared_train_pack(layer)
    sp = shared_params(layer)
    d, F_, H = layer.embed_dim, layer.ffn_embed_dim, layer.self_attn.num_heads
    B, S, M = lay.B, lay.S, lay.M
    dev = x.device

    def e(rows, n):
        return torch.empty(rows, n, dtype=torch.bfloat16, device=dev)

    def g(n):
        return torch.empty(n, dtype=torch.float32, device=dev)
    # ---- FFN branch: x3 = x2 + rs * g2 * f, per modality on its own rows ----
    one_part = len(lay.parts) == 1
    dg2 = g(d) if p["g2"] is not None else None
    db2 = g(d) if one_part else None           # one part: the fc2 bias gradient is the reduction fused into scale_resid_bwd
    df = K.scale_resid_bwd(dx, s["f"], p["g2"], row_scale, e(M, d), dgamma=dg2, dbias=db2)
    dh2 = e(M, d)
    ffn_grads, ffn_ps = [], []
    for pi, (m, _) in enumerate(lay.parts):
        fp = ffn_train_pack(layer, m)
        fps = ffn_params(layer, m)
        rs = lay.rows(pi)
        n = rs.stop - rs.start
        fs = s["ffn"][pi]
        dfp = df[rs]
        db2p = db2 if one_part else K.colsum(dfp, g(d))
        dW2 = _dw(dfp, fs["u2"], fps[4].dtype)
        du2 = _dx(dfp, fp["w2"], F_)
        dlnf_w, dlnf_b = g(F_), g(F_)
        du = K.layernorm_bwd(fs["u"], du2, fp["lnf_w"], fp["lnf_b"], e(n, F_), eps=fp["lnf_eps"], dgamma=dlnf_w, dbeta=dlnf_b)
        dgl = K.geglu_bwd(fs["gl"], du, e(n, 2 * F_))
        dW01 = _dw(dgl, s["h2"][rs], fps[0].dtype)
        _dx(dgl, fp["w01"], d, out=dh2[rs])
        ffn_grads += [dW01[:F_], dW01[F_:], dlnf_w, dlnf_b, dW2, db2p]
        ffn_ps += fps
    dln2_w, dln2_b = g(d), g(d)
    K.layernorm_bwd(s["x2"], dh2, p["ln2_w"], p["ln2_b"], dx, eps=layer.final_layer_norm.eps, accumulate=True,
                    dgamma=dln2_w, dbeta=dln2_b)                                   # dx = dL/dx2
    # ---- attention branch: x2 = x + rs * g1 * o ----
    dg1 = g(d) if p["g1"] is not None else None
    dbo = g(d)
    do = K.scale_resid_bwd(dx, s["o"], p["g1"], row_scale, e(M, d), dgamma=dg1, dbias=dbo)
    dWo = _dw(do, s["a2"], sp[5].dtype)
    da2 = _dx(do, p["wo"], d)
    dlni_w, dlni_b = g(d), g(d)
    datt = K.layernorm_bwd(s["att_mm"], da2, p["lni_w"], p["lni_b"], e(M, d), eps=layer.self_attn.ln.eps, dgamma=dlni_w,
                           dbeta=dlni_b)
    if lay.to_bm is not None:
        datt = K.row_gather(datt, lay.to_bm)
    if bias_t is not None:
        dqkv = K.attention_bwd_t(s["qkv"], s["att"], datt, bias_t, key_pad, s["lse"], e(M, 3 * d), dbias_t, B, S, H,
                                 layer.self_attn.scaling)
    else:
        dqkv = K.attention_bwd(s["qkv"], s["att"], datt, bias, key_pad, s["lse"], e(M, 3 * d), dbias, B, S, H,
                               layer.self_attn.scaling)
    if lay.to_mm is not None:
        dqkv = K.row_gather(dqkv, lay.to_mm)
    dbqkv = K.colsum(dqkv, g(3 * d))
    dWqkv = _dw(dqkv, s["h1"], sp[0].dtype)
    dh1 = _dx(dqkv, p["wqkv"], d)
    dln1_w, dln1_b = g(d), g(d)
    K.layernorm_bwd(x, dh1, p["ln1_w"], p["ln1_b"], dx, eps=layer.self_attn_layer_norm.eps, accumulate=True,
                    dgamma=dln1_w, dbeta=dln1_b)                                   # dx = dL/dx
    grads = [dWqkv[:d], dbqkv[:d], dWqkv[d:2 * d], dWqkv[2 * d:], dbqkv[2 * d:], dWo, dbo, dlni_w, dlni_b, dln1_w, dln1_b,
             dln2_w, dln2_b, dg1, dg2] + ffn_grads
    return [None if gr is None else (gr if gr.dtype == prm.dtype else gr.to(prm.dtype)) for gr, prm in zip(grads, sp + ffn_ps)]


# ----------------------------------------------------------------------------------------------------------------
# the layer stack
# ----------------------------------------------------------------------------------------------------------------
def _pick(lst, i):
    """The entry of layer i in a per-stack list that holds nothing, one entry for every layer, or one per layer."""
    return None if not lst else (lst[0] if len(lst) == 1 else lst[i])


def _b3(b):
    """(1,H,S,S_pad) canvases are passed to the kernels as batch-shared (H,S,S_pad) tables."""
    if b is not None and b.dim() == 4 and b.shape[0] == 1:
        return b[0]
    return b


class EncoderStackFn(torch.autograd.Function):
    """x0 [M, d] fp32 (rows laid out by a SeqLayout) -> x_L [M, d] fp32 through all layers (transformer_encoder.py:172-188).

    meta = (lay, key_pad, need_grad, fast, shared_tables).  `fast` holds the LUT forms of the biases (TrainBias.fast) or is
    empty.  `shared_tables` says that the biases are batch-shared (H,S,S_pad) tables of one relative-position table that
    covers every column of the sequence, as in a single-modality pass.  Only then
      - the forward runs the fused-LayerNorm loop of inference (TransformerEncoder.run_fused) when the activations are not
        kept, no drop-path is active and every bias has a LUT form;
      - the attention backward reads the biases from transposed half2 tables when S <= 224;
      - the accumulated bias gradient is projected onto zero row sums.
    The block canvases of concatenated sequences hold constant zeros between modalities, for which that projection is wrong.
    Backward: per layer, the saved activations or a recompute (un-fused form), then the adjoint."""

    @staticmethod
    def forward(ctx, encoder, meta, x0, n_bias, *tensors):
        lay, key_pad, need_grad, fast, shared_tables = meta
        biases = list(tensors[:n_bias])
        layers = list(encoder.layers)
        x = x0.contiguous()
        scales = []
        for layer in layers:
            rs = None
            if layer.training and layer.drop_path_prob > 0 and need_grad:
                # per-sample keep mask / keep_prob, one value per batch column (transformer_layer.py:80-86)
                keep = 1.0 - layer.drop_path_prob
                rs = lay.row_scale((torch.rand(lay.B, device=x.device) < keep).float() / keep)
            if layer.training and layer.dropout_prob > 0:
                raise NotImplementedError("dropout > 0 (every ONE-PEACE recipe trains with dropout 0.0)")
            scales.append(rs)
        keep_all = need_grad and keep_activations(len(layers), lay.M, x.shape[1], encoder.cfg.ffn_embed_dim, x.device)
        fused = shared_tables and not keep_all and all(r is None for r in scales) and all(f is not None for f in fast)
        xs, saved_all = [], ([] if keep_all else None)
        if fused:
            # run_fused updates the residual stream in place: x0 stays untouched
            x = encoder.run_fused(x.clone(), fast, key_pad, lay.B, lay.S, lay.parts[0][0], inputs=xs)
        else:
            for i, layer in enumerate(layers):
                if need_grad:
                    xs.append(x)
                x, saved = layer_forward(layer, x, lay, _b3(_pick(biases, i)), key_pad, scales[i], keep_all, _pick(fast, i))
                if keep_all:
                    saved_all.append(saved)
        ctx.encoder, ctx.meta = encoder, meta
        ctx.xs, ctx.scales, ctx.biases, ctx.saved_all = xs, scales, biases, saved_all
        return x

    @staticmethod
    def backward(ctx, grad_out):
        lay, key_pad, _, fast, shared_tables = ctx.meta
        layers = list(ctx.encoder.layers)
        biases = ctx.biases
        dx = grad_out.to(torch.float32).contiguous().clone()
        dbiases = [torch.zeros_like(b) for b in biases]
        # S <= 224: the attention backward reads the batch-shared bias from a transposed half2 table and accumulates its
        # gradient in a transposed fp32 table shared by every layer that uses the same bias; both conversions run once per stack
        bias_ts, dbias_ts = [], []
        if shared_tables and biases and lay.S <= K.BIAS_T_Q and all(b.dim() == 3 for b in biases):
            bias_ts = [K.relpos_bias_transpose(b) for b in biases]
            dbias_ts = [torch.zeros(b.shape[0], K.BIAS_T_KEYS, K.BIAS_T_Q, dtype=torch.float32, device=b.device) for b in biases]
        grads = [None] * len(layers)
        for i in reversed(range(len(layers))):
            layer = layers[i]
            bias, dbias = _b3(_pick(biases, i)), _b3(_pick(dbiases, i))
            if ctx.saved_all is not None:
                saved, ctx.saved_all[i] = ctx.saved_all[i], None
            else:
                _, saved = layer_forward(layer, ctx.xs[i], lay, bias, key_pad, ctx.scales[i], True, _pick(fast, i))
            grads[i] = layer_backward(layer, ctx.xs[i], saved, dx, lay, bias, dbias, key_pad, ctx.scales[i],
                                      _pick(bias_ts, i), _pick(dbias_ts, i))
            ctx.xs[i] = None
            del saved
        for dt, db in zip(dbias_ts, dbiases):
            K.relpos_dbias_fold(dt, db)
        if shared_tables:
            # zero-row-sum projection of the bias gradient (csrc/attention_bwd.cu: relpos_dbias_center_kernel).  Padded keys
            # carry dS = 0, so every sample's row sums to zero over all S columns and so does the batch sum.
            for db in dbiases:
                K.relpos_dbias_center(db)
        flat = [g for lg in grads for g in lg]
        return (None, None, dx, None, *dbiases, *flat)


def _stack_params(encoder, lay):
    """Per layer: the 15 shared parameters, then the 6 FFN parameters of each part (EncoderStackFn's gradient order)."""
    params = []
    for layer in encoder.layers:
        params += shared_params(layer)
        for m, _ in lay.parts:
            params += ffn_params(layer, m)
    return params


def run_encoder_stack(encoder, x, bias_list, key_pad, modality):
    """Single-modality pass: x fp32 [B, S, d] (autograd-tracked) -> fp32 [B, S, d].  bias_list: TrainBias or dense fp32
    (H,S,S_pad) tensors (len 0, 1 or L)."""
    B, S, d = x.shape
    if any(layer.gamma_1 is None for layer in encoder.layers):
        raise NotImplementedError("single-modality fast path expects use_layer_scale (the encoder of every recipe)")
    lay = SeqLayout(B, [(modality, S)], x.device)
    params = _stack_params(encoder, lay)
    tb = list(bias_list) if bias_list else []
    biases = [b.dense if isinstance(b, TrainBias) else b for b in tb]
    fast = [b.fast if isinstance(b, TrainBias) else None for b in tb]
    if any(not torch.is_tensor(b) for b in biases):
        raise RuntimeError("training needs the dense relative-position bias (adapters' forward_train provides it)")
    out = EncoderStackFn.apply(encoder, (lay, key_pad, True, fast, True), x.reshape(B * S, d), len(biases), *biases, *params)
    return out.view(B, S, d)


def run_general_stack(encoder, x_mm, lay, key_pad, biases, need_grad):
    """Concatenated sequences, preserve_ids student passes and the decoder: x_mm fp32 [M, d] modality-major -> fp32 [M, d].
    biases: list (len 0, 1 or L) of dense fp32 (Bb,H,S,S_pad) canvases (autograd_general.BlockBiasFn)."""
    return EncoderStackFn.apply(encoder, (lay, key_pad, need_grad, [], False), x_mm, len(biases), *biases,
                                *_stack_params(encoder, lay))


# ----------------------------------------------------------------------------------------------------------------
# relative-position bias, heads, adapters
# ----------------------------------------------------------------------------------------------------------------
class RelPosBiasFn(torch.autograd.Function):
    """rel_pos_table.weight [NB, H] -> dense fp32 (H, S, S_pad) bias (adapter/text.py:84-91, image.py:164-171)."""

    @staticmethod
    def forward(ctx, table, bucket, S, H):
        ctx.bucket, ctx.S, ctx.shape, ctx.dtype = bucket, S, table.shape, table.dtype
        return K.relpos_bias_build(f32(table), bucket, S, H)

    @staticmethod
    def backward(ctx, dbias):
        dtable = torch.zeros(ctx.shape, dtype=torch.float32, device=dbias.device)
        K.relpos_bias_bwd(dbias.contiguous(), ctx.bucket, dtable, ctx.S)
        return dtable.to(ctx.dtype), None, None, None


class HeadFn(torch.autograd.Function):
    """CLS row -> modality LayerNorm -> *_proj -> F.normalize (one_peace_retrieval.py:107-119)."""

    @staticmethod
    def forward(ctx, x, ln_w, ln_b, w, b, eps):
        B, S, d = x.shape
        x = x.contiguous()
        cls = torch.empty(B, d, dtype=torch.bfloat16, device=x.device)
        K.layernorm(x, f32(ln_w), f32(ln_b), cls, rows=B, dim=d, ld_in=S * d, ld_out=d, eps=eps)
        logits = torch.empty(B, w.shape[0], dtype=torch.float32, device=x.device)
        K.gemm(cls, bf16(w), K.EPI_STORE_F32, logits, bias=f32(b))
        ctx.save_for_backward(x, ln_w, ln_b, w, b, cls, logits)
        ctx.eps = eps
        return K.l2_normalize_rows(logits)

    @staticmethod
    def backward(ctx, dy):
        x, ln_w, ln_b, w, b, cls, logits = ctx.saved_tensors
        B, S, d = x.shape
        dlog = K.l2_normalize_bwd(logits, dy.to(torch.float32).contiguous())
        db = K.colsum(dlog, torch.empty(w.shape[0], dtype=torch.float32, device=x.device))
        dW = _dw(dlog, cls, w.dtype)
        dcls = _dx(dlog, bf16(w), d)
        dxf = torch.zeros_like(x)
        dg = torch.empty(d, dtype=torch.float32, device=x.device)
        dbt = torch.empty(d, dtype=torch.float32, device=x.device)
        K.layernorm_bwd(x, dcls, f32(ln_w), f32(ln_b), dxf, eps=ctx.eps, dgamma=dg, dbeta=dbt, rows=B, dim=d, ldx=S * d,
                        ld_dx=S * d)
        return dxf, dg.to(ln_w.dtype), dbt.to(ln_b.dtype), dW, db.to(b.dtype), None


class TextEmbedFn(torch.autograd.Function):
    """tokens -> x [B, T+1, d] fp32 with padded rows zeroed (adapter/text.py:125-129,144-146,153)."""

    @staticmethod
    def forward(ctx, tokens, table, pos, cls, pad_idx):
        tab = table.detach()
        if tab.dtype not in (torch.float32, torch.bfloat16):
            tab = tab.float()
        x, pad = K.text_embed(tokens.contiguous(), tab.contiguous(), f32(pos), f32(cls).view(-1), pad_idx)
        ctx.save_for_backward(tokens)
        ctx.pad_idx = pad_idx
        ctx.meta = (table.shape, table.dtype, pos.shape, pos.dtype, cls.shape, cls.dtype)
        ctx.mark_non_differentiable(pad)
        return x, pad

    @staticmethod
    def backward(ctx, dx, _dpad):
        (tokens,) = ctx.saved_tensors
        tshape, tdt, pshape, pdt, cshape, cdt = ctx.meta
        dev = dx.device
        dtable = torch.zeros(tshape, dtype=torch.float32, device=dev)
        dpos = torch.zeros(pshape, dtype=torch.float32, device=dev)
        dcls = torch.zeros(cshape[-1], dtype=torch.float32, device=dev)
        K.text_embed_bwd(dx.to(torch.float32).contiguous(), tokens.contiguous(), dtable, dpos, dcls, ctx.pad_idx)
        return None, dtable.to(tdt), dpos.to(pdt), dcls.view(cshape).to(cdt), None


def pack_image_stem(w1, b1, ln1w, ln1b, w2, b2, ln2w, ln2b, w3, b3):
    """The hMLP stem's parameters (convs [out, c, ky, kx], LayerNorm2D affines) as image_stem reads them: each conv weight
    as a bf16 GEMM weight [out, (ky, kx, c)], the column order in which the LayerNorm kernel's pixel-merge scatter writes
    that GEMM's operand; biases and affines fp32."""
    c4, d = w1.shape[0], w3.shape[0]
    return dict(w1=bf16(w1.reshape(c4, 48)), b1=f32(b1), ln1w=f32(ln1w), ln1b=f32(ln1b),
                w2=bf16(w2.permute(0, 2, 3, 1).reshape(c4, 4 * c4)), b2=f32(b2), ln2w=f32(ln2w), ln2b=f32(ln2b),
                w3=bf16(w3.permute(0, 2, 3, 1).reshape(d, 4 * c4)), b3=f32(b3))


def image_stem(pk, img, pos, cls=None):
    """hMLP stem (adapter/image.py:66-75) of images [B, 3, R, R] with the pack `pk` of pack_image_stem: patchify, then three
    patch GEMMs with LayerNorm + GELU between them, the last GEMM adding the fp32 positional rows `pos`.
    With `cls` (fp32 [d]): x fp32 [B, w*w+1, d], row 0 = cls + pos[0], row 1 + p = patch p + pos[1 + p].
    Without: x fp32 [B*w*w, d], row-major patches, patch p + pos[p] (pos [w*w, d]).
    Returns (x, (im, y1, a2, y2, a3)): im is the image as the patchify read it (fp32 or bf16), the rest the stages'
    bf16 outputs, which ImageEmbedFn's backward reads."""
    B, _, R, _ = img.shape
    c4, d = pk["w1"].shape[0], pk["w3"].shape[0]
    g1, g2, w = R // 4, R // 8, R // 16
    dev = img.device
    im = img if img.dtype in (torch.float32, torch.bfloat16) else img.float()
    a1 = K.image_patchify4(im.contiguous())
    y1 = K.gemm(a1, pk["w1"], K.EPI_STORE_BF16, torch.empty(B * g1 * g1, c4, dtype=torch.bfloat16, device=dev), bias=pk["b1"])
    a2 = K.layernorm(y1, pk["ln1w"], pk["ln1b"], torch.empty(B * g2 * g2, 4 * c4, dtype=torch.bfloat16, device=dev),
                     gelu=True, merge_grid_w=g1)
    y2 = K.gemm(a2, pk["w2"], K.EPI_STORE_BF16, torch.empty(B * g2 * g2, c4, dtype=torch.bfloat16, device=dev), bias=pk["b2"])
    a3 = K.layernorm(y2, pk["ln2w"], pk["ln2b"], torch.empty(B * w * w, 4 * c4, dtype=torch.bfloat16, device=dev),
                     gelu=True, merge_grid_w=g2)
    if cls is None:
        x = K.gemm(a3, pk["w3"], K.EPI_RESID_F32, torch.empty(B * w * w, d, dtype=torch.float32, device=dev),
                   bias=pk["b3"], resid=pos, resid_period=w * w)
    else:
        S = w * w + 1
        x = torch.empty(B, S, d, dtype=torch.float32, device=dev)
        K.gemm(a3, pk["w3"], K.EPI_RESID_F32, x.view(B * S, d), bias=pk["b3"], resid=pos, out_group=w * w,
               out_group_stride=S, out_row_offset=1, resid_period=w * w, resid_row_offset=1)
        K.cls_row_init(cls, pos, x)
    return x, (im, y1, a2, y2, a3)


class ImageEmbedFn(torch.autograd.Function):
    """hMLP stem + CLS + positions (adapter/image.py:66-75,239-253) as three patch GEMMs (image_stem); `pos` [S, d] is
    the (possibly bicubic-resized, by torch autograd) positional table."""

    @staticmethod
    def forward(ctx, img, pos, w1, b1, ln1w, ln1b, w2, b2, ln2w, ln2b, w3, b3, cls):
        B, _, R, _ = img.shape
        d = w3.shape[0]
        c4 = w1.shape[0]
        pk = pack_image_stem(w1, b1, ln1w, ln1b, w2, b2, ln2w, ln2b, w3, b3)
        x, (im, y1, a2, y2, a3) = image_stem(pk, img, f32(pos), f32(cls).view(-1))
        ctx.save_for_backward(im, ln1w, ln1b, ln2w, ln2b, w1, w2, w3, y1, a2, y2, a3)
        ctx.pk = pk
        ctx.meta = (B, R, d, c4, pos.dtype, b1.dtype, cls.shape, cls.dtype)
        return x

    @staticmethod
    def backward(ctx, dx):
        im, ln1w, ln1b, ln2w, ln2b, w1, w2, w3, y1, a2, y2, a3 = ctx.saved_tensors
        B, R, d, c4, pos_dt, b_dt, cls_shape, cls_dt = ctx.meta
        g1, g2, w = R // 4, R // 8, R // 16
        S = w * w + 1
        dev = dx.device
        pk = ctx.pk
        dx = dx.to(torch.float32).contiguous()

        def g(n):
            return torch.empty(n, dtype=torch.float32, device=dev)
        dcls = K.batch_sum(dx, g(d), B, d, S * d)
        dpos = K.batch_sum(dx, torch.empty(S, d, dtype=torch.float32, device=dev), B, S * d, S * d)
        db3 = g(d)
        dy3 = K.scale_resid_bwd(dx, None, None, None, torch.empty(B * w * w, d, dtype=torch.bfloat16, device=dev), dbias=db3,
                                in_period=S, in_valid=w * w, in_shift=1)
        dW3 = _dw(dy3, a3, w3.dtype).view(d, 2, 2, c4).permute(0, 3, 1, 2)
        da3 = _dx(dy3, pk["w3"], 4 * c4)
        dln2w, dln2b = g(c4), g(c4)
        dy2 = K.layernorm_bwd(y2, da3, f32(ln2w), f32(ln2b), torch.empty_like(y2), gelu=True, dgamma=dln2w, dbeta=dln2b,
                              dy_merge_w=g2)
        db2 = K.colsum(dy2, g(c4))
        dW2 = _dw(dy2, a2, w2.dtype).view(c4, 2, 2, c4).permute(0, 3, 1, 2)
        da2 = _dx(dy2, pk["w2"], 4 * c4)
        dln1w, dln1b = g(c4), g(c4)
        dy1 = K.layernorm_bwd(y1, da2, f32(ln1w), f32(ln1b), torch.empty_like(y1), gelu=True, dgamma=dln1w, dbeta=dln1b,
                              dy_merge_w=g1)
        db1 = K.colsum(dy1, g(c4))
        a1 = K.image_patchify4(im)
        dW1 = _dw(dy1, a1, w1.dtype).view(c4, 3, 4, 4)
        return (None, dpos.to(pos_dt), dW1, db1.to(b_dt), dln1w.to(ln1w.dtype), dln1b.to(ln1b.dtype), dW2.contiguous(),
                db2.to(b_dt), dln2w.to(ln2w.dtype), dln2b.to(ln2b.dtype), dW3.contiguous(), db3.to(b_dt),
                dcls.view(cls_shape).to(cls_dt))


class AudioFeatFn(torch.autograd.Function):
    """Waveform -> frame features fp32 [B*T, d] (adapter/audio.py:183: `self.embed_audios(src_audios)`): wav2vec conv feature
    extractor (:254-311) + post LayerNorm + Linear (:46-55).  Training form: every convolution is a GEMM over a MATERIALISED
    window matrix (opb_window_gather) in compact per-clip frame space; col2im (opb_window_scatter) is the adjoint.  (The
    inference path, adapter/audio.py here, reads overlapping TMA views instead and never materialises windows.)

    Inputs after (wav, meta): conv weights [n_fe], LN weights [n_fe], LN biases [n_fe], post_ln w, b, proj w, b."""

    @staticmethod
    def forward(ctx, wav, meta, *ps):
        spec, d = meta
        n_fe = len(spec)
        conv_w, ln_w, ln_b = ps[:n_fe], ps[n_fe:2 * n_fe], ps[2 * n_fe:3 * n_fe]
        post_w, post_b, proj_w, proj_b = ps[3 * n_fe:3 * n_fe + 4]
        B, N = wav.shape
        dev = wav.device
        C = spec[0][0]
        frames, L = [], N
        for _, k, s in spec:
            L = (L - k) // s + 1
            frames.append(L)
        T = frames[-1]

        def e(rows, n, dt=torch.bfloat16):
            return torch.empty(rows, n, dtype=dt, device=dev)
        wv = wav if wav.dtype in (torch.float32, torch.bfloat16) else wav.float()
        a0 = K.audio_frame10(wv.contiguous(), frames[0], e(B * frames[0], 16))
        w0 = torch.zeros(C, 16, dtype=torch.bfloat16, device=dev)
        w0[:, :spec[0][1]] = conv_w[0].detach()[:, 0, :].to(torch.bfloat16)
        wk = [w0] + [bf16(conv_w[k].permute(0, 2, 1).reshape(C, -1)) for k in range(1, n_fe)]     # [out, (tap, c)]
        ys, zs = [], []
        y = K.gemm(a0, wk[0], K.EPI_STORE_BF16, e(B * frames[0], C))
        z = K.layernorm(y, f32(ln_w[0]), f32(ln_b[0]), e(B * frames[0], C), gelu=True)
        ys.append(y); zs.append(z)
        for k in range(1, n_fe):
            A = K.window_gather(z, B, frames[k - 1], frames[k], spec[k][2], spec[k][1], 0, 1)[0]
            y = K.gemm(A, wk[k], K.EPI_STORE_BF16, e(B * frames[k], C))
            z = K.layernorm(y, f32(ln_w[k]), f32(ln_b[k]), e(B * frames[k], C), gelu=True)
            ys.append(y); zs.append(z)
        yP = K.layernorm(z, f32(post_w), f32(post_b), e(B * T, C))
        feats = K.gemm(yP, bf16(proj_w), K.EPI_STORE_F32, e(B * T, d, torch.float32), bias=f32(proj_b))
        ctx.saved = dict(a0=a0, wk=wk, ys=ys, zs=zs, yP=yP)
        ctx.params = ps
        ctx.meta = (meta, frames, B)
        return feats

    @staticmethod
    def backward(ctx, dfeats):
        (spec, d), frames, B = ctx.meta
        s = ctx.saved
        ps = ctx.params
        n_fe = len(spec)
        conv_w, ln_w, ln_b = ps[:n_fe], ps[n_fe:2 * n_fe], ps[2 * n_fe:3 * n_fe]
        post_w, post_b, proj_w, proj_b = ps[3 * n_fe:3 * n_fe + 4]
        C, T = spec[0][0], frames[-1]
        dev = dfeats.device

        def e(rows, n):
            return torch.empty(rows, n, dtype=torch.bfloat16, device=dev)

        def g32(n):
            return torch.empty(n, dtype=torch.float32, device=dev)
        dfeats = dfeats.to(torch.float32).contiguous()
        dproj_b = g32(d)
        dfb = K.scale_resid_bwd(dfeats, None, None, None, e(B * T, d), dbias=dproj_b)
        dproj_w = _dw(dfb, s["yP"], proj_w.dtype)
        dyP = _dx(dfb, bf16(proj_w), C)
        dpost_w, dpost_b = g32(C), g32(C)
        dz = K.layernorm_bwd(s["zs"][-1], dyP, f32(post_w), f32(post_b), e(B * T, C), dgamma=dpost_w, dbeta=dpost_b)
        dconv, dlnw, dlnb = [None] * n_fe, [None] * n_fe, [None] * n_fe
        for k in reversed(range(n_fe)):
            dg, db = g32(C), g32(C)
            dy = K.layernorm_bwd(s["ys"][k], dz, f32(ln_w[k]), f32(ln_b[k]), e(B * frames[k], C), gelu=True, dgamma=dg, dbeta=db)
            dlnw[k], dlnb[k] = dg.to(ln_w[k].dtype), db.to(ln_b[k].dtype)
            if k == 0:
                dW0 = _dw(dy, s["a0"], conv_w[0].dtype)                                     # [C, 16]
                dconv[0] = dW0[:, :spec[0][1]].reshape(C, 1, spec[0][1]).contiguous()
            else:
                kw, st = spec[k][1], spec[k][2]
                A = K.window_gather(s["zs"][k - 1], B, frames[k - 1], frames[k], st, kw, 0, 1)[0]
                dconv[k] = _dw(dy, A, conv_w[k].dtype).view(C, kw, C).permute(0, 2, 1).contiguous()
                dA = _dx(dy, s["wk"][k], kw * C)
                dz = K.window_scatter(dA.view(1, B * frames[k], kw * C), B, frames[k - 1], frames[k], st, kw, 0)
        grads = list(dconv) + dlnw + dlnb + [dpost_w.to(post_w.dtype), dpost_b.to(post_b.dtype), dproj_w, dproj_b.to(proj_b.dtype)]
        return (None, None, *grads)


class AudioPosFn(torch.autograd.Function):
    """Frame features fp32 [B*T, d] -> x fp32 [B, T+1, d] (adapter/audio.py:190-199): 5-layer grouped conv positional encoder on
    the un-normalised features (:57-80), `x = cat(cls, feats) + cat(cls_pos, pos)`, padded rows zeroed
    (transformer_encoder.py:139-142).  `feats` may be the preserve_ids-gathered sequence of a student pass (:184-189: the
    gather happens BEFORE the positional convolution).  Every convolution is a GEMM over a materialised window matrix.

    Inputs after (feats, pad, meta): pos conv weights [n_pos], pos conv biases [n_pos], cls_embedding, cls_pos_embed."""

    @staticmethod
    def forward(ctx, feats, pad, meta, *ps):
        B, T, pos_k, pos_groups, d = meta
        n_pos = (len(ps) - 2) // 2
        pos_w, pos_b = ps[:n_pos], ps[n_pos:2 * n_pos]
        cls, cls_pos = ps[-2], ps[-1]
        dev = feats.device
        S = T + 1
        feats = feats.to(torch.float32).contiguous()

        def e(rows, n, dt=torch.bfloat16):
            return torch.empty(rows, n, dtype=dt, device=dev)
        G = pos_groups
        cg = d // G
        pk = [bf16(pos_w[i].permute(0, 2, 1).reshape(d, pos_k * cg)) for i in range(n_pos)]     # [(g, co), (tap, ci)]
        p_in = e(B * T, d)
        K.row_stats_cast(feats, p_in, torch.empty(B * T, device=dev), torch.empty(B * T, device=dev))
        p_ins, cs = [], []
        for i in range(n_pos):
            Xw = K.window_gather(p_in, B, T, T, 1, pos_k, pos_k // 2, G)
            c = e(B * T, d)
            bi = f32(pos_b[i])
            for g in range(G):
                K.gemm(Xw[g], pk[i][g * cg:(g + 1) * cg], K.EPI_STORE_BF16, c[:, g * cg:(g + 1) * cg], bias=bi[g * cg:(g + 1) * cg])
            p_ins.append(p_in); cs.append(c)
            p_in = K.layernorm(c, None, None, e(B * T, d), gelu=True)
        body = K.scale_resid_fwd(feats, p_in, None, None, torch.empty_like(feats))
        x = torch.empty(B, S, d, dtype=torch.float32, device=dev)
        x[:, 1:].copy_(body.view(B, T, d))
        K.cls_row_init(f32(cls).view(-1), f32(cls_pos).view(-1), x)
        padu = pad.to(torch.uint8).contiguous()
        K.zero_padded_rows(x, padu)
        ctx.saved = dict(p_ins=p_ins, cs=cs, pk=pk, padu=padu)
        ctx.params = ps
        ctx.meta = meta
        ctx.mark_non_differentiable(padu)
        return x, padu

    @staticmethod
    def backward(ctx, dxs, _dpad):
        B, T, pos_k, pos_groups, d = ctx.meta
        s = ctx.saved
        ps = ctx.params
        n_pos = len(s["cs"])
        pos_w, pos_b = ps[:n_pos], ps[n_pos:2 * n_pos]
        cls, cls_pos = ps[-2], ps[-1]
        S = T + 1
        G = pos_groups
        cg = d // G
        dev = dxs.device

        def e(rows, n):
            return torch.empty(rows, n, dtype=torch.bfloat16, device=dev)

        def g32(n):
            return torch.empty(n, dtype=torch.float32, device=dev)
        dxs = dxs.to(torch.float32).contiguous().clone()
        K.zero_padded_rows(dxs, s["padu"])                                  # padded rows were zeroed in the forward
        dcls = K.batch_sum(dxs, g32(d), B, d, S * d)
        dbody = dxs[:, 1:].reshape(B * T, d).contiguous()                   # = d feats (direct) = d pos
        dp = K.scale_resid_bwd(dbody, None, None, None, e(B * T, d))
        dpos_w, dpos_b = [None] * n_pos, [None] * n_pos
        for i in reversed(range(n_pos)):
            dc = K.layernorm_bwd(s["cs"][i], dp, None, None, e(B * T, d), gelu=True)
            dpos_b[i] = K.colsum(dc, g32(d)).to(pos_b[i].dtype)
            Xw = K.window_gather(s["p_ins"][i], B, T, T, 1, pos_k, pos_k // 2, G)
            dW = torch.empty(d, pos_k * cg, dtype=pos_w[i].dtype, device=dev)
            dXw = torch.empty(G, B * T, pos_k * cg, dtype=torch.bfloat16, device=dev)
            for g in range(G):
                sl = slice(g * cg, (g + 1) * cg)
                dW[sl] = _dw(dc[:, sl], Xw[g], pos_w[i].dtype)
                _dx(dc[:, sl], s["pk"][i][sl], pos_k * cg, out=dXw[g])
            dpos_w[i] = dW.view(d, pos_k, cg).permute(0, 2, 1).contiguous()
            dp = K.window_scatter(dXw, B, T, T, 1, pos_k, pos_k // 2)
        dfeats = K.scale_resid_fwd(dbody, dp, None, None, torch.empty_like(dbody))      # direct + through the pos branch
        grads = dpos_w + dpos_b + [dcls.view(cls.shape).to(cls.dtype), dcls.view(cls_pos.shape).to(cls_pos.dtype)]
        return (dfeats, None, None, *grads)
