"""CPU: the bounds of tests/stem_ref.py against the training Functions of one_peace_b200/autograd.py run on an fp64
emulation of their kernels.

``Emu`` stands in for ``one_peace_b200.kernels``: each kernel computes in fp64 and rounds to its output's dtype (bf16
activations and gradients, fp32 records), with the row maps of the C header (pixel merges, the CLS-row shift, window
gathers, strided rows).  The Functions run unchanged on it, packs, views and shifts included, from a fresh copy of the
autograd module's source.  Their results must stay within the bounds, and each planted mistake (a one-line change of that
source, or of one emulated kernel) must exceed them at least 100-fold somewhere.  tests/test_head_ref.py runs the
classification heads, the criteria and the pretraining-path Functions on the same ``Emu``, ``Recorder`` and
``functions``; tests/test_layer_ref.py runs the encoder stack on them."""
import inspect
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import det_ref as D
import kernel_ref as R
import stem_ref as SR
import test_classify_host_logic as CH
from grounding_ref import refcoco
from one_peace_b200 import autograd as AG
from one_peace_b200.kernels import RelPosBias
from vit_ref import head_bwd, head_fwd

BF = torch.bfloat16
MISS = 100.0            # a planted mistake must use at least this many times its bound


class Emu:
    """fp64 emulation of the kernels the training Functions call, around and inside the encoder stack
    (``one_peace_b200.kernels`` signatures).  Flags plant mistakes inside a kernel: ``text_pad_grad`` (padding tokens get a gradient),
    ``text_pos_shift`` (position gradients one row early), ``l2_no_radial`` (l2-normalize backward without the radial
    projection), ``scatter_overwrite`` (row_scatter_add stores instead of adding, so a repeated index keeps one row),
    ``dbias_t_overwrite`` (attention_bwd_t stores its bias gradient into the transposed table instead of adding, so layers
    that share a table keep only the last one's).  tests/test_layer_ref.py runs the encoder stack on it."""
    EPI_STORE_BF16, EPI_GEGLU_BF16, EPI_RESID_F32, EPI_STORE_F32, EPI_GELU_BF16 = 0, 1, 2, 3, 4
    BIAS_T_KEYS, BIAS_T_Q = 256, 224        # the transposed bias tables of the attention backward
    RelPosBias = RelPosBias                 # the bias container, as kernels.RelPosBias

    def __init__(self, **flags):
        self.text_pad_grad = flags.pop("text_pad_grad", False)
        self.text_pos_shift = flags.pop("text_pos_shift", False)
        self.l2_no_radial = flags.pop("l2_no_radial", False)
        self.scatter_overwrite = flags.pop("scatter_overwrite", False)
        self.dbias_t_overwrite = flags.pop("dbias_t_overwrite", False)
        assert not flags

    @staticmethod
    def _rows(t, rows, dim, ld):
        return t.as_strided((rows, dim), (ld, 1))

    def gemm(self, a, w, epi, out, *, bias=None, colscale=None, out_group=0, out_group_stride=0, out_row_offset=0,
             resid=None, resid_period=0, resid_row_offset=0, **kw):
        assert not kw
        y = a.double() @ w.double().t()
        if bias is not None:
            y = y + bias.double()
        if colscale is not None:
            y = y * colscale.double()
        if epi == self.EPI_GELU_BF16:
            y = F.gelu(y)
        if epi == self.EPI_RESID_F32:
            N = y.shape[1]
            m = torch.arange(y.shape[0])
            rows = (m // out_group) * out_group_stride + m % out_group + out_row_offset if out_group else m
            rr = m % resid_period + resid_row_offset if resid_period else rows
            out.view(-1, N)[rows] = (y + resid.reshape(-1, N).double()[rr]).float()
        else:
            out.copy_(y.to(out.dtype))
        return out

    def gemm_t(self, a, b, epi, out, a_mn=False, b_mn=False, bias=None):
        A = a.double().t() if a_mn else a.double()
        B = b.double() if b_mn else b.double().t()
        out.copy_((A @ B).to(out.dtype))
        return out

    def transpose_bf16(self, x):
        return x.t().contiguous()

    def layernorm(self, x, gamma, beta, out, *, rows=None, dim=None, ld_in=None, ld_out=None, eps=1e-5, gelu=False,
                  merge_grid_w=0):
        rows = x.shape[0] if rows is None else rows
        dim = x.shape[-1] if dim is None else dim
        X = self._rows(x, rows, dim, x.stride(-2) if ld_in is None else ld_in).double()
        y = F.layer_norm(X, (dim,), None if gamma is None else gamma.double(), None if beta is None else beta.double(), eps)
        if gelu:
            y = F.gelu(y)
        if merge_grid_w:
            orow, col, _ = R.ln_layout(rows, dim, merge_grid_w=merge_grid_w)
            out.view(-1)[orow[:, None] * out.stride(0) + col] = y.to(out.dtype)
        else:
            self._rows(out, rows, dim, out.stride(-2) if ld_out is None else ld_out).copy_(y.to(out.dtype))
        return out

    def layernorm_bwd(self, x, dy, gamma, beta, dx, *, eps=1e-5, gelu=False, accumulate=False, dgamma=None, dbeta=None,
                      rows=None, dim=None, ldx=None, ld_dx=None, dy_merge_w=0):
        rows = x.shape[0] if rows is None else rows
        dim = x.shape[-1] if dim is None else dim
        X = self._rows(x, rows, dim, x.stride(-2) if ldx is None else ldx).double().requires_grad_()
        if dy_merge_w:
            orow, col0 = R.merge_rows(rows, dim, dy_merge_w)
            DY = dy.reshape(-1)[orow[:, None] * dy.stride(0) + col0[:, None] + torch.arange(dim)].double()
        else:
            DY = self._rows(dy, rows, dim, dy.stride(-2)).double()
        g = gamma.double().requires_grad_() if gamma is not None else None
        b = beta.double().requires_grad_() if beta is not None else None
        with torch.enable_grad():                          # called from inside a Function's backward
            y = F.layer_norm(X, (dim,), g, b, eps)
            if gelu:
                y = F.gelu(y)
            ins = [X] + [t for t in (g, b) if t is not None]
            gs = torch.autograd.grad(y, ins, DY)
        o = self._rows(dx, rows, dim, dx.stride(-2) if ld_dx is None else ld_dx)
        o.copy_((gs[0] + (o.double() if accumulate else 0)).to(dx.dtype))
        if dgamma is not None:
            dgamma.copy_(gs[1])
        if dbeta is not None:
            dbeta.copy_(gs[2])
        return dx

    def image_patchify4(self, img):
        B, _, R_, _ = img.shape
        q = R_ // 4
        return img.reshape(B, 3, q, 4, q, 4).permute(0, 2, 4, 1, 3, 5).reshape(B * q * q, 48).to(BF)

    def cls_row_init(self, cls, pos0, x):
        x[:, 0, :] = cls.float() + pos0.reshape(-1)[:x.shape[2]].float()
        return x

    def batch_sum(self, x, out, B, n, ld, accumulate=False):
        flat = x.reshape(-1)
        out.view(-1).copy_(sum(flat[b * ld:b * ld + n].double() for b in range(B)))
        return out

    def scale_resid_bwd(self, dx, o, gamma, row_scale, d_o, dgamma=None, dbias=None, in_period=0, in_valid=0, in_shift=0):
        rows, n = d_o.shape
        r = R.scale_resid_bwd_ref(dx.reshape(-1, n)[R.scale_resid_rows(rows, in_period, in_valid, in_shift)], o, gamma,
                                  row_scale)
        d_o.copy_(r.d_o.to(BF))
        if dgamma is not None:
            dgamma.copy_(r.dgamma)
        if dbias is not None:
            dbias.copy_(r.dbias)
        return d_o

    def scale_resid_fwd(self, x, o, gamma, row_scale, out):
        out.copy_(R.scale_resid_ref(x, o, gamma, row_scale)[0])
        return out

    def geglu_fwd(self, gl, u):
        u.copy_(R.geglu_ref(gl)[0])
        return u

    def geglu_bwd(self, gl, du, dgl):
        dgl.copy_(R.geglu_bwd_ref(gl, du)[0])
        return dgl

    def colsum(self, y, out):
        out.copy_(y.double().sum(0))
        return out

    def l2_normalize_rows(self, x):
        X = x.double()
        return (X / X.norm(dim=1, keepdim=True).clamp_min(1e-12)).float()

    def l2_normalize_bwd(self, x, dy, want_f32=False):
        X, G = x.double(), dy.double()
        n = X.norm(dim=1, keepdim=True)
        dx = G / n if self.l2_no_radial else G / n - X * (X * G).sum(1, keepdim=True) / n ** 3
        return (dx.to(BF), dx.float()) if want_f32 else dx.to(BF)

    def text_embed(self, tokens, table, pos, cls, pad_idx=1):
        return R.text_embed_ref(tokens, table, pos, cls, pad_idx)

    def text_embed_bwd(self, dx, tokens, dtable, dpos, dcls, pad_idx=1):
        B, T = tokens.shape
        D = dx.double()
        dt, dp = dtable.double(), dpos.double()
        dc = dcls.double() + D[:, 0].sum(0)
        dp[0] += D[:, 0].sum(0)
        for b in range(B):
            for s in range(1, T + 1):
                tok = int(tokens[b, s - 1])
                if tok == pad_idx and not self.text_pad_grad:
                    continue
                dt[tok] += D[b, s]
                dp[s - 1 if self.text_pos_shift else s] += D[b, s]
        dtable.copy_(dt)
        dpos.copy_(dp)
        dcls.copy_(dc)

    def relpos_bias_build(self, table, bucket, S, H):
        return R.relpos_bias_ref(table, bucket, S, (S + 7) // 8 * 8)

    def relpos_bias_bwd(self, dbias, bucket, dtable, S):
        H = dbias.shape[0]
        dt = dtable.double().index_add(0, bucket[:S, :S].reshape(-1), dbias[..., :S].double().permute(1, 2, 0).reshape(-1, H))
        dtable.copy_(dt)
        return dtable

    def row_stats_cast(self, x, out_bf16, mu, rstd, eps=1e-5):
        out_bf16.copy_(x.to(BF))
        r = R.layernorm_ref(x, None, None, eps)
        mu.copy_(r.mu)
        rstd.copy_(r.rstd)
        return out_bf16

    # the fused-LayerNorm layer loops (TransformerEncoder.run_fused, VideoLayer.forward_video): the GEMM with its LayerNorm
    # fold, records and bf16 side output (csrc/gemm.h) and the fold itself (csrc/pack.cu), on their fp64 references
    def gemm_ln(self, a, w, epi, out, *, ln_partial=None, stats_out=None, out_bf16=None, workspace=None, cta_group=0, **kw):
        M, N = a.shape[0], out.shape[-1]
        if ln_partial is not None:                          # the kernel reads the first `parts` records of every row
            rec, parts, dim, eps = ln_partial
            ln_partial = (rec.reshape(-1)[:parts * M * 2], parts, dim, eps)
        g = R.gemm_ref(a, w, epi, ln_partial=ln_partial, stats=stats_out is not None, **kw)
        o = out.view(-1, N)
        o[g.rows[g.valid]] = g.y[g.valid].to(out.dtype)
        if out_bf16 is not None:
            out_bf16.view(-1, N)[g.rows[g.valid]] = o[g.rows[g.valid]].to(BF)
        if stats_out is not None:
            stats_out.view(-1)[:g.stats.numel()] = g.stats.reshape(-1).float()
        return out

    def ln_fold(self, weight, ln_w, ln_b, bias, out_w, colsum, bias_out, interleave=0):
        r = R.ln_fold_ref(weight, ln_w, ln_b, bias, interleave)
        out_w[r.rows] = r.wg
        colsum[r.rows] = r.colsum.float()
        bias_out[r.rows] = r.bias.float()

    def window_gather(self, x, B, t_in, t_out, stride, kw, pad, groups):
        cg = x.shape[1] // groups
        hi = (t_out - 1) * stride + kw
        Xp = F.pad(x.double().view(B, t_in, groups * cg), (0, 0, pad, max(0, hi - pad - t_in)))
        idx = torch.arange(t_out)[:, None] * stride + torch.arange(kw)[None, :]
        win = Xp[:, idx].view(B, t_out, kw, groups, cg)
        return win.permute(3, 0, 1, 2, 4).reshape(groups, B * t_out, kw * cg).to(BF)

    def window_scatter(self, dwin, B, t_in, t_out, stride, kw, pad):
        return R.window_scatter_ref(dwin, B, t_in, t_out, stride, kw, pad)[0].to(BF)

    def audio_frame10(self, wav, pitch, out):
        B = wav.shape[0]
        win = wav.unfold(1, 10, 5)[:, :pitch]                      # [B, pitch, 10]: wav[b, 5t + j]
        out.copy_(F.pad(win, (0, 6)).reshape(B * pitch, 16).to(BF))
        return out

    def zero_padded_rows(self, x, pad_mask):
        x.view(-1, x.shape[-1])[pad_mask.reshape(-1).bool()] = 0
        return x

    # the classification heads and criteria (csrc/classify.cu, vit_head.cu, grounding.cu): their fp64 references
    def attn_pool_fwd(self, kv, q, key_pad, B, T):
        out, lse, _, _ = CH.pool_fwd_ref(kv, q, key_pad, B, T)
        return out.to(BF), lse.float()

    def attn_pool_bwd(self, kv, q, key_pad, lse, dout, B, T):
        dkv, dq, _, _ = CH.pool_bwd_ref(kv, q, key_pad, dout, B, T)
        return dkv.to(BF), dq.float()

    def classify_loss(self, logits, n_valid, mode, labels=None, targets=None, eps=0.0, num_choices=1):
        r = CH.loss_ref(logits, n_valid, mode, labels=labels, targets=targets, eps=eps, num_choices=num_choices)
        dl = torch.full((logits.shape[0], logits.stride(0)), float("nan"))      # columns past n_valid are not defined
        dl[:, :r["dlogits"].shape[1]] = r["dlogits"].float()
        return r["row_loss"].float(), dl, r["row_correct"].float(), torch.stack([r["loss"], r["n_correct"]]).float()

    def refcoco_loss(self, logits, targets, nsentences):
        with torch.enable_grad():                          # refcoco's bounds are taken by autograd
            r = refcoco(logits, targets, nsentences)
        dl = torch.full((logits.shape[0], logits.stride(0)), float("nan"))
        dl[:, :4] = r["dlogits"].float()
        out = torch.tensor([float(r["loss"]), float(r["l1"]), float(r["n_valid"])])
        return out, r["valid"].int(), r["giou"].float(), dl

    def token_mean_ln_fwd(self, x, gamma, beta, eps):
        f = head_fwd(x, gamma, beta, eps)
        return f["y"].to(BF), f["m"].float(), f["mean"].float(), f["rstd"].float()

    def token_mean_ln_bwd(self, dy, m, mean, rstd, gamma, dx):
        hb = head_bwd(dy, m, mean, rstd, gamma, dx.shape[1])
        dx.copy_(hb["dx"])
        return hb["dgamma"].float(), hb["dbeta"].float()

    # the pretraining path: gathers, bias blocks, the DCL loss's InfoNCE
    def row_gather(self, src, idx, out=None, fill=None, out_dtype=None, add=None):
        rows, dim = idx.numel(), src.shape[1]
        if out is None:
            out = torch.empty(rows, dim, dtype=out_dtype or src.dtype)
        v = torch.where((idx >= 0)[:, None], src.double()[idx.clamp_min(0)], fill.double() if fill is not None else 0.0)
        if add is not None:
            a = add.reshape(-1, dim).double()
            v = v + a[torch.arange(rows) % a.shape[0]]
        out.copy_(v.to(out.dtype))
        return out

    def row_scatter_add(self, dout, idx, dsrc):
        keep = idx >= 0
        if self.scatter_overwrite:
            dsrc[idx[keep]] = dout[keep].to(dsrc.dtype)
        else:
            dsrc.copy_(dsrc.double().index_add(0, idx[keep], dout.double()[keep]))
        return dsrc

    def relpos_bias_block(self, table, bucket, ids, n, lo, bias, S, H):
        bias.copy_(R.relpos_bias_block_ref(table, bucket, ids, n, lo, bias)[0])
        return bias

    def relpos_bias_block_bwd(self, dbias, bucket, ids, n, lo, dtable, S, H):
        Bb = dbias.shape[0]
        p = torch.arange(n).expand(Bb, n) if ids is None else torch.where(ids < 0, n - 1, ids)
        dest = bucket[p[:, :, None], p[:, None, :]].reshape(-1)
        src = dbias[:, :, lo:lo + n, lo:lo + n].double().permute(0, 2, 3, 1).reshape(-1, H)
        dtable.copy_(dtable.double().index_add(0, dest, src))
        return dtable

    # the encoder stack's attention (csrc/attention.cu, attention_bwd.cu): the fp64 references on the values the kernels read
    def attention(self, qkv, bias, key_pad, B, S, H, out=None, lse=None, ln_stats=None):
        f = R.attention_ref(qkv, None if bias is None else bias[..., :S], key_pad, B, S, H)
        out.copy_(f.out)
        if lse is not None:
            lse.copy_(f.lse.reshape(-1))
        if ln_stats is not None:                            # [H, B S, 2] of the fp32 rows before rounding
            ln_stats.view(-1).copy_(f.stats.reshape(-1))
        return out

    def attention_tc(self, qkv, rp, key_pad, B, S, H, out=None, ln_stats=None, lse=None):
        assert not getattr(rp, "seg_split", 0)
        dense = rp.lut[:, (rp.code_row[:S, None] - rp.code_col[None, :S]).long()]
        return self.attention(qkv, dense, key_pad, B, S, H, out=out, lse=lse, ln_stats=ln_stats)

    def relpos_decomp_proj(self, qkv, rel_pos_h, rel_pos_w, pos_y, pos_x, B, S, H, kh, kw, q_unscale=8.0, rel_h=None,
                           rel_w=None):
        rh, _, rw, _ = D.proj_ref(qkv, rel_pos_h, rel_pos_w, pos_y, pos_x, B, S, H, kh, kw)
        s = q_unscale / D.Q_UNSCALE                         # proj_ref multiplies q by the model's unscale
        return (rh * s).float(), (rw * s).float()

    def attention_decomp(self, qkv, rp, rel_h, rel_w, key_y, key_x, B, S, H, kh, kw, out=None, ln_stats=None, lse=None):
        dense = rp.lut[:, (rp.code_row[:S, None] - rp.code_col[None, :S]).long()]
        f = D.decomp_attention_ref(qkv, dense, rel_h, torch.zeros_like(rel_h), rel_w, torch.zeros_like(rel_w), key_y, key_x,
                                   B, S, H)
        out.copy_(f.out)
        if lse is not None:
            lse.copy_(f.lse.reshape(-1))
        if ln_stats is not None:
            ln_stats.view(-1).copy_(f.stats.reshape(-1))
        return out

    def attention_temporal(self, qkv, Bv, T, N, H, out=None, ln_stats=None):
        b, n, t = torch.meshgrid(torch.arange(Bv), torch.arange(N), torch.arange(T), indexing="ij")
        idx = ((b * T + t) * N + n).reshape(-1)               # sequence b N + n: the T frames of token n of clip b
        f = R.attention_ref(qkv[idx], None, None, Bv * N, T, H)
        out[idx] = f.out.to(out.dtype)
        ln_stats.view(H, -1, 2)[:, idx] = f.stats.float()
        return out, ln_stats

    def relpos_lut_build(self, table, idx):
        return R.relpos_lut_ref(table, idx).contiguous()

    def attention_bwd(self, qkv, out, d_out, bias, key_pad, lse, dqkv, dbias, B, S, H, q_scale):
        r = R.attention_bwd_ref(qkv, out, d_out, lse, None if bias is None else bias[..., :S], key_pad, B, S, H, q_scale)
        dqkv.copy_(r.dqkv)
        if dbias is not None:
            d = dbias[..., :S]
            d.copy_(d.double() + (r.dS if dbias.dim() == 4 else r.dS.sum(0)))
        return dqkv

    def relpos_bias_transpose(self, bias):
        """(H,S,S_pad) -> (H,256,224) fp16(b log2 e), transposed, zero-padded, stored as (H,256,112) half2 words"""
        H, S, _ = bias.shape
        t = torch.zeros(H, self.BIAS_T_KEYS, self.BIAS_T_Q, dtype=torch.float16, device=bias.device)
        t[:, :S, :S] = (bias[..., :S].float() * 1.4426950408889634).transpose(1, 2).half()
        return t.view(torch.int32)

    def attention_bwd_t(self, qkv, out, d_out, bias_t, key_pad, lse, dqkv, dbias_t, B, S, H, q_scale):
        bias = bias_t.view(torch.float16)[:, :S, :S].transpose(1, 2).double() / 1.4426950408889634
        r = R.attention_bwd_ref(qkv, out, d_out, lse, bias, key_pad, B, S, H, q_scale)
        dqkv.copy_(r.dqkv)
        d = dbias_t[:, :S, :S]
        d.copy_(r.dS.sum(0).transpose(1, 2) + (0.0 if self.dbias_t_overwrite else d.double()))
        return dqkv

    def relpos_dbias_fold(self, dbias_t, dbias):
        S = dbias.shape[1]
        d = dbias[..., :S]
        d.copy_(d.double() + dbias_t[:, :S, :S].double().transpose(1, 2))
        return dbias

    def relpos_dbias_center(self, dbias):
        S = dbias.shape[1]
        d = dbias[..., :S]
        d.copy_(d.double() - d.double().mean(-1, keepdim=True))
        return dbias

    def split_bf16x3(self, xs, sides):
        outs = []
        for x, side in zip(xs, sides):
            hi = x.to(BF)
            lo = (x - hi.float()).to(BF)
            outs.append(torch.cat([hi, hi, lo] if side == 0 else [hi, lo, hi], 1))
        return outs

    @staticmethod
    def _infonce(a3, b3, scale, n_valid, target_offset, eps):
        """z = s a3 b3^T over the n class columns, the targets, the smoothing weights (kernel_ref.infonce_ref)"""
        n = n_valid or b3.shape[0]
        z = float(scale) * (a3.double() @ b3.double().t())[:, :n]
        rows = torch.arange(z.shape[0])
        eps_i = eps / (n - 1) if eps else 0.0
        return z, rows, rows + target_offset, eps_i, 1.0 - eps - eps_i

    def infonce_forward(self, pairs, scale, target_offset, eps, n_valid=0, rows=False):
        ((a3, b3),) = pairs
        assert not rows
        z, r, tgt, eps_i, hit = self._infonce(a3, b3, scale, n_valid, target_offset, eps)
        lse = torch.logsumexp(z, 1)
        loss = hit * (lse - z[r, tgt]) + eps_i * (z.shape[1] * lse - z.sum(1))
        out3 = torch.stack([loss.mean(), (z.argmax(1) == tgt).double().sum(), torch.zeros((), dtype=torch.float64)])
        return [lse.float()], out3.float()

    def infonce_grad(self, a_local, b_all, scale, row_lse, target_offset, eps, d, n_valid=0, coef=0.0):
        z, r, tgt, eps_i, hit = self._infonce(a_local, b_all, scale, n_valid, target_offset, eps)
        G = (z - row_lse.double()[:, None]).exp() - eps_i
        G[r, tgt] -= hit
        return (float(scale) * coef * (G @ b_all[:z.shape[1], :d].double())).float(), None


class Recorder:
    """Forwards every kernel call to ``kernels`` and logs (name, args, kwargs, result): the backward's intermediates are
    read from what each kernel was given and returned."""

    def __init__(self, kernels):
        self.kernels, self.log = kernels, []

    def __getattr__(self, name):
        f = getattr(self.kernels, name)
        if not callable(f):
            return f

        def call(*a, **kw):
            r = f(*a, **kw)
            self.log.append((name, a, kw, r))
            return r
        return call


def functions(kernels, edit=None, module=AG, recorder=Recorder):
    """The Functions of a fresh copy of ``module`` (one_peace_b200/autograd.py by default) whose kernels are ``kernels``
    behind a ``recorder`` (``Recorder`` or a subclass; ``.K``); edit = (old, new) replaces the one occurrence of ``old`` in its source.  What the
    module imports from autograd (``_dw``, ``_dx``, ``_pad8``) is taken from a fresh copy of autograd on the same Recorder,
    so that those helpers' GEMMs and transposes also run on ``kernels`` and appear in the log."""
    rec = recorder(kernels)

    def fresh(mod, ed):
        src = inspect.getsource(mod)
        if ed is not None:
            assert src.count(ed[0]) == 1, ed[0]
            src = src.replace(*ed)
        ns = {"__name__": mod.__name__ + "_emulated", "__package__": "one_peace_b200"}
        exec(compile(src, mod.__file__, "exec"), ns)
        ns["K"] = rec
        return ns
    ns = fresh(module, edit)
    if module is not AG:
        ag = fresh(AG, None)
        for k, v in ns.items():
            if k != "K" and getattr(AG, k, None) is v:
                ns[k] = ag[k]
    return SimpleNamespace(**ns)


# ----------------------------------------------------------------------------------------------------------------------
# cases: each runs one Function (two for audio) and returns ({output: share of its bound}, outputs that may be exact)
# ----------------------------------------------------------------------------------------------------------------------
def image_case(fns, B=2, R_=32, c4=16, d=32, img_dtype=torch.float32, p_dtype=torch.float32, seed=0, one_channel=False,
               dev="cpu"):
    """one_channel: the upstream gradient only on output channel 0"""
    g = torch.Generator().manual_seed(seed)
    w = R_ // 16
    S = w * w + 1
    rn = lambda *s, sc=1.0: (sc * torch.randn(*s, generator=g)).to(dev, p_dtype).requires_grad_()
    img = torch.randn(B, 3, R_, R_, generator=g).to(dev, img_dtype)
    sw = (4 * c4) ** -0.5
    params = [rn(S, d, sc=0.5), rn(c4, 3, 4, 4, sc=0.3), rn(c4, sc=0.1), (1 + rn(c4, sc=0.2)).detach().requires_grad_(),
              rn(c4, sc=0.1), rn(c4, c4, 2, 2, sc=sw), rn(c4, sc=0.1), (1 + rn(c4, sc=0.2)).detach().requires_grad_(),
              rn(c4, sc=0.1), rn(d, c4, 2, 2, sc=sw), rn(d, sc=0.1), rn(1, 1, d, sc=0.5)]
    x = fns.ImageEmbedFn.apply(img, *params)
    dx = torch.randn(B, S, d, generator=g).to(dev)
    if one_channel:
        dx[..., 1:] = 0
    saved = x.grad_fn.saved_tensors
    fns.K.log.clear()
    got = dict(zip(SR.IMAGE_GRADS, torch.autograd.grad(x, params, dx)))
    chk, inter = SR.image_embed_ref(img, params, saved, dx, fns.K.log)
    got.update(inter, x=x)
    return SR.shares(got, chk), (("cls", "pos") if B == 1 else ())


def head_case(fns, B=3, S=5, d=32, n=24, p_dtype=torch.float32, seed=1, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, sc=1.0, off=0.0: (off + sc * torch.randn(*s, generator=g)).to(dev, p_dtype).requires_grad_()
    x = (torch.randn(B, S, d, generator=g) + 0.3).to(dev).requires_grad_()
    ps = [rn(d, sc=0.2, off=1.0), rn(d, sc=0.1), rn(n, d, sc=0.2), rn(n, sc=0.1)]
    y = fns.HeadFn.apply(x, *ps, 1e-5)
    dy = torch.randn(B, n, generator=g).to(dev)
    saved = y.grad_fn.saved_tensors
    fns.K.log.clear()
    got = dict(zip(SR.HEAD_GRADS, torch.autograd.grad(y, [x] + ps, dy)))
    chk, inter = SR.head_ref(x, *ps, 1e-5, saved, dy, fns.K.log)
    got.update(inter, y=y)
    return SR.shares(got, chk), (("w",) if B == 1 else ())          # dW over one row: one exact bf16 product


def text_case(fns, B=3, T=7, V=20, d=16, pad_idx=1, pads=((1, 4), (2, 6)), seed=2, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randint(2, V - 4, (B, T), generator=g)           # rows V-4.. stay unused
    for b, t in pads:
        tokens[b, t:] = pad_idx
    tokens = tokens.to(dev)
    table = torch.randn(V, d, generator=g).to(dev).requires_grad_()
    pos = torch.randn(T + 3, d, generator=g).to(dev).requires_grad_()
    cls = torch.randn(1, 1, d, generator=g).to(dev).requires_grad_()
    x, pad = fns.TextEmbedFn.apply(tokens, table, pos, cls, pad_idx)
    dx = torch.randn(B, T + 1, d, generator=g).to(dev)
    got = dict(zip(("table", "pos", "cls"), torch.autograd.grad(x, [table, pos, cls], dx)), x=x)
    chk, pad_ref = SR.text_embed_fn_ref(tokens, table, pos, cls, pad_idx, dx)
    assert torch.equal(pad, pad_ref)
    return SR.shares(got, chk), ("cls",) if B == 1 else ()


def relpos_case(fns, S=9, H=4, NB=30, seed=3, bucket=None, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    if bucket is None:
        bucket = torch.randint(0, NB - 3, (S + 2, S + 2), generator=g)   # the last three buckets stay unused
    bucket = bucket.to(dev)
    table = torch.randn(NB, H, generator=g).to(dev).requires_grad_()
    b = fns.RelPosBiasFn.apply(table, bucket, S, H)
    db = torch.randn(b.shape, generator=g).to(dev)
    (gt,) = torch.autograd.grad(b, [table], db)
    return SR.shares(dict(bias=b, table=gt), SR.relpos_fn_ref(table, bucket, S, db)), ("bias",)


SPEC = ((16, 10, 5),) + ((16, 3, 2),) * 4 + ((16, 2, 2),) * 2      # the wav2vec extractor's kernels, 16 channels


def audio_case(fns, B=2, T=23, d=32, G=16, k=19, n=5, pad_from=(None, 15), p_dtype=torch.float32, seed=4, samples=0,
               spec=SPEC, wav_dtype=torch.float32, dev="cpu"):
    """AudioPosFn on random features of T frames, or (samples > 0) AudioFeatFn on a waveform followed by AudioPosFn"""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, sc=1.0, off=0.0: (off + sc * torch.randn(*s, generator=g)).to(dev, p_dtype).requires_grad_()
    fparams = []
    if samples:
        C = spec[0][0]
        wav = torch.randn(B, samples, generator=g).to(dev, wav_dtype)
        fparams = ([rn(C, 1, spec[0][1], sc=spec[0][1] ** -0.5)]
                   + [rn(C, C, kk, sc=(C * kk) ** -0.5) for _, kk, _ in spec[1:]]
                   + [rn(C, sc=0.2, off=1.0) for _ in spec] + [rn(C, sc=0.1) for _ in spec]
                   + [rn(C, sc=0.2, off=1.0), rn(C, sc=0.1), rn(d, C, sc=C ** -0.5), rn(d, sc=0.1)])
        feats = fns.AudioFeatFn.apply(wav, (spec, d), *fparams)
        T = feats.shape[0] // B
    else:
        feats = torch.randn(B * T, d, generator=g).to(dev).requires_grad_()
    pad = torch.zeros(B, T + 1, dtype=torch.bool)
    for b, p in enumerate(pad_from):
        if p is not None:
            pad[b, 1 + p:] = True
    pad = pad.to(dev)
    cg = d // G
    ps = ([rn(d, cg, k, sc=1.5 / (k * cg) ** 0.5) for _ in range(n)] + [rn(d, sc=0.1) for _ in range(n)]
          + [rn(1, 1, d) for _ in range(2)])
    meta = (B, T, k, G, d)
    x, padu = fns.AudioPosFn.apply(feats, pad, meta, *ps)
    dxs = torch.randn(B, T + 1, d, generator=g).to(dev)
    s = x.grad_fn.saved
    fns.K.log.clear()
    names = [f"w{i}" for i in range(n)] + [f"b{i}" for i in range(n)] + ["cls", "cls_pos"]
    if samples:
        fnames = ([f"conv{i}" for i in range(len(spec))] + [f"lnw{i}" for i in range(len(spec))]
                  + [f"lnb{i}" for i in range(len(spec))] + ["post_w", "post_b", "proj_w", "proj_b"])
        gs = torch.autograd.grad(x, ps + fparams, dxs)
        got = dict(zip(names + fnames, gs))
        # AudioFeatFn reads the gradient of its output first (scale_resid_bwd with the projection's bias gradient)
        dfeats = [a[0] for nm, a, kw, _ in fns.K.log if nm == "scale_resid_bwd" and kw.get("dbias") is not None][0]
        fs = feats.grad_fn.saved
        fchk, finter = SR.audio_feat_ref(wav, spec, d, fparams, fs, feats, fns.K.log)
        got.update(finter)
    else:
        gs = torch.autograd.grad(x, [feats] + ps, dxs)
        got = dict(zip(["feats"] + names, gs))
        dfeats, fchk = gs[0], {}
    chk, inter = SR.audio_pos_ref(feats, pad, meta, ps, s, dxs, dfeats, fns.K.log)
    got.update(inter, x=x)
    return SR.shares(got, {**chk, **fchk}), ("a0",) + (("cls", "cls_pos") if B == 1 else ())     # a0: bf16 copies


CASES = {
    "image": image_case,
    "image_bf16": lambda f: image_case(f, B=3, R_=48, img_dtype=BF, p_dtype=BF, seed=5),
    "image_one_channel": lambda f: image_case(f, B=1, one_channel=True, seed=9),
    "head": head_case,
    "head_b1_bf16": lambda f: head_case(f, B=1, S=3, p_dtype=BF, seed=6),
    "text": text_case,
    "relpos": relpos_case,
    "audio_pos": audio_case,
    "audio_pos_1layer": lambda f: audio_case(f, B=3, T=17, d=16, n=1, pad_from=(None, 9, 0), seed=8),
    "audio_wave": lambda f: audio_case(f, B=2, samples=2000, pad_from=(None, 3), seed=10),
    "audio_wave_bf16": lambda f: audio_case(f, B=1, samples=1500, pad_from=(None,), p_dtype=BF, wav_dtype=BF, seed=11),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_emulation_within_bounds(case):
    sh, _ = CASES[case](functions(Emu()))
    bad = {k: v for k, v in sh.items() if not v <= 1.0}
    assert not bad, f"{case}: outside the bound: {bad}"


# name -> (case, case arguments, source edit or kernel flags)
MISTAKES = {
    "dW2 taps transposed": ("image", {}, dict(edit=(".view(c4, 2, 2, c4).permute(0, 3, 1, 2)\n        da2",
                                                    ".view(c4, 2, 2, c4).permute(0, 3, 2, 1)\n        da2"))),
    "CLS row read as a patch": ("image", {}, dict(edit=("in_valid=w * w, in_shift=1)", "in_valid=w * w, in_shift=0)"))),
    "dcls from sample 0 only": ("image", {}, dict(edit=("dcls = K.batch_sum(dx, g(d), B, d, S * d)",
                                                        "dcls = K.batch_sum(dx, g(d), 1, d, S * d)"))),
    "stage-1 merge width g2 (forward)": ("image", {}, dict(edit=("merge_grid_w=g1)", "merge_grid_w=g2)"))),
    "stage-1 merge width g2 (backward)": ("image", {}, dict(edit=("dy_merge_w=g1)", "dy_merge_w=g2)"))),
    "dW0 from taps 6..15": ("audio", dict(samples=2000), dict(edit=("dW0[:, :spec[0][1]]", "dW0[:, 6:]"))),
    "window_scatter with stride 1": ("audio", dict(samples=2000), dict(edit=("frames[k], st, kw, 0)", "frames[k], 1, kw, 0)"))),
    "padded rows not zeroed": ("audio", {}, dict(edit=('K.zero_padded_rows(dxs, s["padu"])', "pass"))),
    "group g's dW from group g+1": ("audio", {}, dict(edit=("_dw(dc[:, sl], Xw[g],", "_dw(dc[:, sl], Xw[(g + 1) % G],"))),
    "direct residual dropped": ("audio", {}, dict(edit=(
        "dfeats = K.scale_resid_fwd(dbody, dp, None, None, torch.empty_like(dbody))", "dfeats = dp.float()"))),
    "gradient reaches pad_idx": ("text", {}, dict(flags=dict(text_pad_grad=True))),
    "positions shifted by the CLS row": ("text", {}, dict(flags=dict(text_pos_shift=True))),
    "l2 backward without the radial projection": ("head", {}, dict(flags=dict(l2_no_radial=True))),
    "head normalises token 1": ("head", {}, dict(edit=("K.layernorm(x, f32(ln_w)", "K.layernorm(x[:, 1:], f32(ln_w)"))),
}
CASE_FNS = dict(image=image_case, head=head_case, text=text_case, audio=audio_case)


@pytest.mark.parametrize("name", sorted(MISTAKES))
def test_planted_mistake_exceeds_bound(name):
    case, args, how = MISTAKES[name]
    sh, _ = CASE_FNS[case](functions(Emu(**how.get("flags", {})), how.get("edit")), **args)
    assert max(sh.values()) >= MISS, f"{name}: largest share of a bound only {max(sh.values()):.3g}"


def test_relpos_unused_bucket_exactly_zero():
    """a bound of zero admits only an exact zero: an unused bucket's gradient of 1e-30 fails"""
    fns = functions(Emu())
    g = torch.Generator().manual_seed(7)
    bucket = torch.randint(0, 10, (9, 9), generator=g)
    table = torch.randn(12, 2, generator=g).requires_grad_()
    b = fns.RelPosBiasFn.apply(table, bucket, 9, 2)
    db = torch.randn(b.shape, generator=g)
    (gt,) = torch.autograd.grad(b, [table], db)
    chk = SR.relpos_fn_ref(table, bucket, 9, db)
    assert SR.share(gt, *chk["table"]) <= 1.0
    gt = gt.clone()
    gt[11, 0] = 1e-30
    assert SR.share(gt, *chk["table"]) == float("inf")
