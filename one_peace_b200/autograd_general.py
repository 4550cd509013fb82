"""Pretraining path (SURVEY.md 8f rows 1-2) around the layer stack (autograd.run_general_stack): the block-diagonal
relative-position bias canvas of concatenated 'vl' / 'al' sequences with sample-dependent preserve_ids gathers, row
gathers (preserve_ids, the mask-token canvas of the decoder), padded-row zeroing, nn.Linear, the per-modality final
LayerNorm and the DCL loss — all as ``torch.autograd.Function`` nodes whose forward AND backward are sm_90a kernels behind
the C-ABI (the reference relies on torch autograd for every one of them).
"""
import torch

from . import kernels as K
from .autograd import _dw, _dx
from .components import bf16, f32


# ----------------------------------------------------------------------------------------------------------------
# dense relative-position bias canvas: per-modality diagonal blocks, optional per-sample preserve_ids gather
# ----------------------------------------------------------------------------------------------------------------
class BlockBiasFn(torch.autograd.Function):
    """tables (one rel_pos_table.weight per part that has a bias) -> fp32 [Bb, H, S, S_pad] canvas
    (adapter gather_features + transformer_encoder.py:144-158).  meta = (H, S, [(bucket, ids or None, n, lo)] per table)."""

    @staticmethod
    def forward(ctx, meta, *tables):
        H, S, blocks = meta
        Bb = max([1] + [ids.shape[0] for _, ids, _, _ in blocks if ids is not None])
        dev = tables[0].device
        s_pad = (S + 7) // 8 * 8
        bias = torch.zeros(Bb, H, S, s_pad, dtype=torch.float32, device=dev)
        for t, (bucket, ids, n, lo) in zip(tables, blocks):
            if ids is None and Bb > 1:                      # a shared block inside per-sample canvases: write it per sample
                for bb in range(Bb):
                    K.relpos_bias_block(f32(t), bucket, None, n, lo, bias[bb:bb + 1], S, H)
            else:
                K.relpos_bias_block(f32(t), bucket, ids, n, lo, bias, S, H)
        ctx.meta = meta
        ctx.shapes = [(t.shape, t.dtype) for t in tables]
        return bias

    @staticmethod
    def backward(ctx, dbias):
        H, S, blocks = ctx.meta
        dbias = dbias.contiguous()
        Bb = dbias.shape[0]
        out = []
        for (shape, dt), (bucket, ids, n, lo) in zip(ctx.shapes, blocks):
            dtable = torch.zeros(shape, dtype=torch.float32, device=dbias.device)
            if ids is None and Bb > 1:
                for bb in range(Bb):
                    K.relpos_bias_block_bwd(dbias[bb:bb + 1], bucket, None, n, lo, dtable, S, H)
            else:
                K.relpos_bias_block_bwd(dbias, bucket, ids, n, lo, dtable, S, H)
            out.append(dtable.to(dt))
        return (None, *out)


# ----------------------------------------------------------------------------------------------------------------
# small differentiable pieces
# ----------------------------------------------------------------------------------------------------------------
class RowGatherFn(torch.autograd.Function):
    """out[r] = src[idx[r]] (idx >= 0) else fill; + add[r % period].  src fp32 [n, dim]; fill fp32 [dim] (mask token) or
    None; add fp32 [period, dim] (positional table) or None.  Adjoint: scatter-add, masked column sum, batch sum."""

    @staticmethod
    def forward(ctx, src, idx, fill, add):
        s32 = src if src.dtype in (torch.float32, torch.bfloat16) else src.float()
        out = K.row_gather(s32.contiguous(), idx, fill=None if fill is None else f32(fill).view(-1),
                           add=None if add is None else f32(add), out_dtype=torch.float32)
        ctx.save_for_backward(idx)
        ctx.meta = (src.shape, src.dtype, None if fill is None else (fill.shape, fill.dtype),
                    None if add is None else (add.shape, add.dtype))
        return out

    @staticmethod
    def backward(ctx, dout):
        (idx,) = ctx.saved_tensors
        sshape, sdt, fmeta, ameta = ctx.meta
        dout = dout.to(torch.float32).contiguous()
        dim = dout.shape[1]
        dsrc = None
        if ctx.needs_input_grad[0]:
            dsrc = torch.zeros(sshape, dtype=torch.float32, device=dout.device)
            K.row_scatter_add(dout, idx, dsrc)
            dsrc = dsrc.to(sdt)
        dfill = None
        if fmeta is not None and ctx.needs_input_grad[2]:
            sel = torch.nonzero(idx < 0, as_tuple=False).flatten()
            dfill = torch.zeros(dim, dtype=torch.float32, device=dout.device)
            if sel.numel() > 0:
                rows = K.row_gather(dout, sel.contiguous())
                K.batch_sum(rows, dfill, sel.numel(), dim, dim)
            dfill = dfill.view(fmeta[0]).to(fmeta[1])
        dadd = None
        if ameta is not None and ctx.needs_input_grad[3]:
            period = ameta[0][0] if len(ameta[0]) == 2 else ameta[0].numel() // dim
            dadd = torch.empty(period * dim, dtype=torch.float32, device=dout.device)
            K.batch_sum(dout, dadd, dout.shape[0] // period, period * dim, period * dim)
            dadd = dadd.view(ameta[0]).to(ameta[1])
        return dsrc, None, dfill, dadd


class ZeroPadFn(torch.autograd.Function):
    """x * (1 - padding_mask) (transformer_encoder.py:139-142); the adjoint masks the same rows."""

    @staticmethod
    def forward(ctx, x, pad_rows):
        out = x.contiguous().clone()
        K.zero_padded_rows(out, pad_rows)
        ctx.save_for_backward(pad_rows)
        return out

    @staticmethod
    def backward(ctx, dx):
        (pad_rows,) = ctx.saved_tensors
        dx = dx.to(torch.float32).contiguous().clone()
        K.zero_padded_rows(dx, pad_rows)
        return dx, None


class LinearFn(torch.autograd.Function):
    """y = x W^T + b (components.py:29-35) on the wgmma GEMM: fp32 rows in, fp32 rows out (bf16 operands, fp32
    accumulate), dX / dW through the same GEMM, db by the column-sum kernel."""

    @staticmethod
    def forward(ctx, x, w, b):
        rows = x.shape[0]
        xb = torch.empty(rows, x.shape[1], dtype=torch.bfloat16, device=x.device)
        K.row_gather(x.contiguous() if x.dtype in (torch.float32, torch.bfloat16) else x.float().contiguous(),
                     torch.arange(rows, device=x.device), out=xb)
        y = torch.empty(rows, w.shape[0], dtype=torch.float32, device=x.device)
        K.gemm(xb, bf16(w), K.EPI_STORE_F32, y, bias=None if b is None else f32(b))
        ctx.save_for_backward(xb, w, b)
        ctx.xdt = x.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, w, b = ctx.saved_tensors
        rows = dy.shape[0]
        dyb = torch.empty(rows, dy.shape[1], dtype=torch.bfloat16, device=dy.device)
        K.row_gather(dy.to(torch.float32).contiguous(), torch.arange(rows, device=dy.device), out=dyb)
        db = None
        if b is not None:
            db = K.colsum(dyb, torch.empty(w.shape[0], dtype=torch.float32, device=dy.device)).to(b.dtype)
        dW = _dw(dyb, xb, w.dtype)
        dxf = torch.empty(rows, w.shape[1], dtype=torch.float32, device=dy.device)
        _dx(dyb, bf16(w), w.shape[1], out=dxf)
        return dxf.to(ctx.xdt), dW, db


class FinalNormFn(torch.autograd.Function):
    """Per-modality final LayerNorm over all rows (transformer_encoder.py:201-220)."""

    @staticmethod
    def forward(ctx, x, w, b, eps):
        x = x.contiguous()
        out = torch.empty_like(x)
        K.layernorm(x, f32(w), f32(b), out, eps=eps)
        ctx.save_for_backward(x, w, b)
        ctx.eps = eps
        return out

    @staticmethod
    def backward(ctx, dy):
        x, w, b = ctx.saved_tensors
        d = x.shape[1]
        dg = torch.empty(d, dtype=torch.float32, device=x.device)
        db = torch.empty(d, dtype=torch.float32, device=x.device)
        dx = torch.empty_like(x)
        K.layernorm_bwd(x, dy.to(torch.float32).contiguous(), f32(w), f32(b), dx, eps=ctx.eps, dgamma=dg, dbeta=db)
        return dx, dg.to(w.dtype), db.to(b.dtype), None


# ----------------------------------------------------------------------------------------------------------------
# DCL loss (criterions/image_text_pretrain_loss.py:187-208)
# ----------------------------------------------------------------------------------------------------------------
class DclLossFn(torch.autograd.Function):
    """student fp32 [R, d] rows (all positions, flattened), teacher [R, d] (detached), stu_idx int64 [n_m] = rows of the masked,
    non-padded, non-CLS positions, tea_idx int64 [n_t] = the same rows first, then every other non-padded non-CLS row
    (soft-max over the columns is permutation invariant, so the target of student row r is column r).  One direction of
    the InfoNCE kernels with scale = dcl_logit_scale, label smoothing and mean over the n_m rows."""

    @staticmethod
    def forward(ctx, student, teacher, stu_idx, tea_idx, scale, eps):
        dev = student.device
        n_m, n_t = stu_idx.numel(), tea_idx.numel()
        d = student.shape[1]
        n8 = (n_t + 7) // 8 * 8
        tidx = tea_idx if n8 == n_t else torch.cat([tea_idx, torch.full((n8 - n_t,), -1, dtype=torch.int64, device=dev)])
        s_rows = K.row_gather(student.detach().float().contiguous(), stu_idx)            # fp32 [n_m, d]
        t_rows = K.row_gather(teacher.detach().float().contiguous(), tidx.contiguous())  # fp32 [n8, d], zero rows past n_t
        s_n, t_n = K.l2_normalize_rows(s_rows), K.l2_normalize_rows(t_rows)              # F.normalize(x.float(), dim=1)
        a3, b3 = K.split_bf16x3([s_n, t_n], [0, 1])
        sc = torch.full((1,), float(scale), dtype=torch.float32, device=dev)
        (lse,), out = K.infonce_forward([(a3, b3)], sc, 0, eps, n_valid=n_t)           # out[0] = mean(row_loss)
        if student.requires_grad:
            grad_n, _ = K.infonce_grad(a3, b3, sc, lse, 0, eps, d, n_valid=n_t, coef=1.0 / n_m)
            dx16, dx32 = K.l2_normalize_bwd(s_rows, grad_n, want_f32=True)
            ctx.save_for_backward(dx32, stu_idx)
        ctx.meta = (student.shape, student.dtype)
        return out[0]

    @staticmethod
    def backward(ctx, g_loss):
        dx32, stu_idx = ctx.saved_tensors
        shape, dt = ctx.meta
        ds = torch.zeros(shape, dtype=torch.float32, device=dx32.device)
        K.row_scatter_add(dx32 * g_loss.to(torch.float32), stu_idx, ds)
        return ds.to(dt), None, None, None, None, None


def dcl_indices(mask_indices, padding_masks):
    """Row selections of compute_dcl_loss (image_text_pretrain_loss.py:190-202) as flat indices into the (B*S) rows:
    CLS dropped, padded tokens dropped, masked rows first.  mask_indices bool (B,S); padding_masks bool (B,S-1) or None."""
    B, S = mask_indices.shape
    pos = torch.arange(B * S, device=mask_indices.device).view(B, S)[:, 1:]
    m = mask_indices[:, 1:].bool()
    valid = torch.ones_like(m) if padding_masks is None else ~padding_masks.bool()
    stu = pos[m & valid]
    rest = pos[(~m) & valid]
    return stu.contiguous(), torch.cat([stu, rest]).contiguous()
