"""Tensor-level wrappers over the C-ABI: PyTorch allocates, the sm_90a kernels compute.

Every function takes CUDA tensors, passes raw device pointers + the current stream to
``libonepeace_b200.so`` and returns torch tensors.  Nothing here computes with torch ops.
"""
import ctypes

import torch

from . import _lib

F32, BF16 = 0, 1
EPI_STORE_BF16, EPI_GEGLU_BF16, EPI_RESID_F32, EPI_STORE_F32, EPI_GELU_BF16 = 0, 1, 2, 3, 4


# number of kernel launches issued through the C-ABI since import (bench.py reports it per step)
LAUNCHES = 0
# optional per-call profiler hook: bench.py installs a callable(name, flops) -> context manager
PROFILE_HOOK = None


def _count(n=1):
    global LAUNCHES
    LAUNCHES += n


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("one_peace_b200 kernels need CUDA tensors (there is no CPU path)")


def _dt(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise RuntimeError(f"unsupported dtype {t.dtype}")


def gemm(a, w, epi, out, *, bias=None, colscale=None, gamma=None, resid=None, out_group=0, out_group_stride=0,
         out_row_offset=0, out_group_valid=0, resid_period=0, resid_row_offset=0, cta_group=0, M=None, lda=None,
         K=None):
    """out = epilogue(a[M,K] @ w[N,K]^T).  a/w bf16; `lda`/`M`/`K` allow strided (even overlapping) row views."""
    _need_cuda(a, w, out)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
    if M is None:
        M = a.shape[0]
    if K is None:
        K = a.shape[1]
    if lda is None:
        lda = a.stride(0)
    N = w.shape[0]
    if PROFILE_HOOK is not None:
        PROFILE_HOOK("gemm_begin", 0.0, None)
    assert w.shape[1] == K and w.stride(1) == 1 and a.stride(-1) == 1
    ldr = resid.stride(-2) if resid is not None else 0
    st = _lib.load().opb_gemm_bf16(a.data_ptr(), lda, w.data_ptr(), w.stride(0), M, N, K, epi, out.data_ptr(),
                                   out.stride(-2), _ptr(bias), _ptr(colscale), _ptr(gamma), _ptr(resid), ldr,
                                   out_group, out_group_stride, out_row_offset, out_group_valid, resid_period,
                                   resid_row_offset, cta_group, _stream())
    _lib.check(st, "opb_gemm_bf16")
    _count()
    if PROFILE_HOOK is not None:
        PROFILE_HOOK("gemm", 2.0 * M * N * K, (M, N, K, epi))
    return out


class RelPosBias:
    """Relative-position bias of one forward in both forms the attention kernels take: the dense fp32 (H,S,S_pad)
    table (any S) and the LUT form (same kernels; the adapters build it for S <= ATTN_TC_MAX_S)."""

    def __init__(self, dense=None, lut=None, code_row=None, code_col=None, seg_split=0):
        self.dense, self.lut, self.code_row, self.code_col, self.seg_split = dense, lut, code_row, code_col, seg_split
        self.lut_max = None


def build_segmented_lut(parts, device):
    """Concatenated ('vl' / 'al') LUT-form bias for `attention_tc`.  parts = [(table fp32 [NB,H], lut_index, n)] per modality
    in sequence order, lut_index = relpos.build_lut_index(...) result (numpy lut_idx, code_row, code_col) or device tensors.
    The per-modality LUTs are laid end to end; row codes of the second modality are shifted by the length of the first LUT
    so that same-modality code differences land in that modality's LUT; the kernel zeroes the cross-modality bias."""
    assert len(parts) == 2, "two concatenated modalities (transformer_encoder.py:127-134)"
    luts, rows, cols, off = [], [], [], 0
    for table, li, n in parts:
        idx, cr, cc = (torch.as_tensor(a, device=device).to(torch.int32) for a in li)
        luts.append(relpos_lut_build(table, idx.contiguous()))
        rows.append(cr[:n] + off)
        cols.append(cc[:n])
        off += idx.numel()
    lut = torch.cat(luts, dim=1).contiguous()
    pad4 = lambda t: torch.cat([t, torch.zeros((-t.numel()) % 4, dtype=t.dtype, device=t.device)]).contiguous()
    return RelPosBias(lut=lut, code_row=pad4(torch.cat(rows)), code_col=pad4(torch.cat(cols)), seg_split=parts[0][2])


def relpos_lut_build(table, idx):
    """table fp32 [NB,H], idx int32 [L] -> lut fp32 [H, L]"""
    L, H = idx.numel(), table.shape[1]
    lut = torch.empty(H, L, dtype=torch.float32, device=table.device)
    st = _lib.load().opb_relpos_lut_build(table.data_ptr(), idx.data_ptr(), lut.data_ptr(), L, H, _stream())
    _lib.check(st, "opb_relpos_lut_build")
    _count()
    return lut


# LUT-form bias: the attention kernel gathers each score's bias from a per-head LUT instead of reading the dense (H,S,S_pad)
# table.  The adapters build the LUT form for S <= 384 and the dense table above that.
ATTN_TC_MAX_S = 384


def attention_tc(qkv, rp, key_pad, B, S, H, out=None, ln_stats=None, lse=None):
    """attention with the LUT-form bias (any S; for S <= 224 the kernel stages the head's LUT row in shared memory).  rp: RelPosBias with the LUT form
    (rp.seg_split > 0: two concatenated modalities, block-diagonal bias; S <= 384 then)."""
    D = H * 64
    assert qkv.dtype == torch.bfloat16 and qkv.shape == (B * S, 3 * D) and qkv.is_contiguous()
    if out is None:
        out = torch.empty(B * S, D, dtype=torch.bfloat16, device=qkv.device)
    if getattr(rp, "lut_max", None) is None:        # per-head bound of the bias (once per table build)
        mx = rp.lut.amax(dim=1)
        rp.lut_max = (mx.clamp_min(0.0) if int(getattr(rp, "seg_split", 0)) > 0 else mx).contiguous()
    st = _lib.load().opb_attention_tc_fwd(qkv.data_ptr(), rp.lut.data_ptr(), rp.lut_max.data_ptr(), rp.lut.shape[1], rp.code_row.data_ptr(),
                                          rp.code_col.data_ptr(), _ptr(key_pad), out.data_ptr(), _ptr(lse), _ptr(ln_stats), B, S,
                                          H, int(getattr(rp, "seg_split", 0)), _stream())
    _lib.check(st, "opb_attention_tc_fwd")
    _count()
    return out


def relpos_decomp_proj(qkv, rel_pos_h, rel_pos_w, pos_y, pos_x, B, S, H, kh, kw, q_unscale=8.0, rel_h=None, rel_w=None):
    """Decomposed relative-position terms (include/onepeace_b200.h): -> (rel_h fp32 [B, H, S, kh], rel_w fp32 [B, H, S, kw]).
    qkv bf16 [B*S, 3*H*64]; rel_pos_h / rel_pos_w fp32 [2k - 1, 64]; pos_y / pos_x int32 [S]."""
    _need_cuda(qkv, rel_pos_h, rel_pos_w, pos_y, pos_x)
    assert qkv.dtype == torch.bfloat16 and qkv.shape == (B * S, 3 * H * 64) and qkv.is_contiguous()
    for t in (rel_pos_h, rel_pos_w):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.shape[1] == 64
    assert rel_pos_h.shape[0] == 2 * kh - 1 and rel_pos_w.shape[0] == 2 * kw - 1
    for t in (pos_y, pos_x):
        assert t.dtype == torch.int32 and t.is_contiguous() and t.numel() == S
    if rel_h is None:
        rel_h = torch.empty(B, H, S, kh, dtype=torch.float32, device=qkv.device)
    if rel_w is None:
        rel_w = torch.empty(B, H, S, kw, dtype=torch.float32, device=qkv.device)
    st = _lib.load().opb_relpos_decomp_proj(qkv.data_ptr(), rel_pos_h.data_ptr(), rel_pos_w.data_ptr(), pos_y.data_ptr(),
                                            pos_x.data_ptr(), float(q_unscale), rel_h.data_ptr(), rel_w.data_ptr(), B, S, H,
                                            kh, kw, _stream())
    _lib.check(st, "opb_relpos_decomp_proj")
    _count()
    return rel_h, rel_w


def attention_decomp(qkv, rp, rel_h, rel_w, key_y, key_x, B, S, H, kh, kw, out=None, ln_stats=None, lse=None):
    """attention with the LUT-form bias `rp` (RelPosBias, no seg_split) plus rel_h[i][key_y[j]] + rel_w[i][key_x[j]]."""
    D = H * 64
    assert qkv.dtype == torch.bfloat16 and qkv.shape == (B * S, 3 * D) and qkv.is_contiguous()
    assert int(getattr(rp, "seg_split", 0)) == 0
    assert rel_h.shape == (B, H, S, kh) and rel_w.shape == (B, H, S, kw) and rel_h.is_contiguous() and rel_w.is_contiguous()
    if out is None:
        out = torch.empty(B * S, D, dtype=torch.bfloat16, device=qkv.device)
    st = _lib.load().opb_attention_decomp_fwd(qkv.data_ptr(), rp.lut.data_ptr(), rp.lut.shape[1], rp.code_row.data_ptr(),
                                              rp.code_col.data_ptr(), rel_h.data_ptr(), rel_w.data_ptr(), key_y.data_ptr(),
                                              key_x.data_ptr(), kh, kw, out.data_ptr(), _ptr(lse), _ptr(ln_stats), B, S, H,
                                              _stream())
    _lib.check(st, "opb_attention_decomp_fwd")
    _count()
    return out


def attention_temporal(qkv, Bv, T, N, H, out=None, ln_stats=None):
    """Softmax over the T frames of every (clip, token, head) in the frame-major rows (b * T + t) * N + n of qkv
    (include/onepeace_b200.h): -> (out bf16 [Bv * T * N, H * 64], ln_stats fp32 [H, Bv * T * N, 2])."""
    _need_cuda(qkv, out, ln_stats)
    D, M = H * 64, Bv * T * N
    assert qkv.dtype == torch.bfloat16 and qkv.shape == (M, 3 * D) and qkv.is_contiguous()
    if out is None:
        out = torch.empty(M, D, dtype=torch.bfloat16, device=qkv.device)
    if ln_stats is None:
        ln_stats = torch.empty(H, M, 2, dtype=torch.float32, device=qkv.device)
    assert out.dtype == torch.bfloat16 and out.shape == (M, D) and out.is_contiguous()
    assert ln_stats.dtype == torch.float32 and ln_stats.numel() == H * M * 2 and ln_stats.is_contiguous()
    st = _lib.load().opb_attention_temporal_fwd(qkv.data_ptr(), out.data_ptr(), ln_stats.data_ptr(), Bv, T, N, H, _stream())
    _lib.check(st, "opb_attention_temporal_fwd")
    _count()
    return out, ln_stats


def attention_temporal_bwd(qkv, out, d_out, Bv, T, N, H, q_scale, dqkv=None):
    """Adjoint of attention_temporal (include/onepeace_b200.h): -> dqkv bf16 [Bv * T * N, 3 * H * 64] in the same rows,
    dq multiplied by q_scale."""
    _need_cuda(qkv, out, d_out, dqkv)
    D, M = H * 64, Bv * T * N
    assert qkv.dtype == torch.bfloat16 and qkv.shape == (M, 3 * D) and qkv.is_contiguous()
    for t in (out, d_out):
        assert t.dtype == torch.bfloat16 and t.shape == (M, D) and t.is_contiguous()
    if dqkv is None:
        dqkv = torch.empty(M, 3 * D, dtype=torch.bfloat16, device=qkv.device)
    assert dqkv.dtype == torch.bfloat16 and dqkv.shape == (M, 3 * D) and dqkv.is_contiguous()
    st = _lib.load().opb_attention_temporal_bwd(qkv.data_ptr(), out.data_ptr(), d_out.data_ptr(), dqkv.data_ptr(), Bv, T, N,
                                                H, float(q_scale), _stream())
    _lib.check(st, "opb_attention_temporal_bwd")
    _count()
    return dqkv


def _msda_levels(shapes, starts):
    L = len(shapes)
    hw = (ctypes.c_int32 * (2 * L))(*[int(v) for s in shapes for v in s])
    st = (ctypes.c_int32 * L)(*[int(v) for v in starts])
    return hw, st


def _msda_check(value, proj, ref, N, S_in, Lq, H, L, P):
    assert value.dtype == torch.bfloat16 and value.shape == (N * S_in, H * 32) and value.is_contiguous()
    assert proj.dtype == torch.float32 and proj.shape == (N * Lq, 3 * H * L * P) and proj.is_contiguous()
    assert ref.dtype == torch.float32 and ref.dim() == 3 and ref.shape[0] == N * Lq and ref.shape[2] == 2 and ref.is_contiguous()


def ms_deform_attn_fwd(value, proj, ref, shapes, starts, N, Lq, H, P, out=None):
    """Multi-scale deformable attention core (include/onepeace_b200.h): value bf16 [N * S_in, H * 32], proj fp32
    [N * Lq, 3 * H * L * P] (offsets | logits), ref fp32 [N * Lq, L_ref, 2], shapes [(H_l, W_l)] and starts host ints
    -> out bf16 [N * Lq, H * 32]."""
    _need_cuda(value, proj, ref, out)
    L = len(shapes)
    S_in = value.shape[0] // N
    _msda_check(value, proj, ref, N, S_in, Lq, H, L, P)
    if out is None:
        out = torch.empty(N * Lq, H * 32, dtype=torch.bfloat16, device=value.device)
    assert out.dtype == torch.bfloat16 and out.shape == (N * Lq, H * 32) and out.is_contiguous()
    hw, st = _msda_levels(shapes, starts)
    s = _lib.load().opb_ms_deform_attn_fwd(value.data_ptr(), proj.data_ptr(), ref.data_ptr(), out.data_ptr(), N, S_in, Lq, H,
                                           32, L, P, ref.shape[1], hw, st, _stream())
    _lib.check(s, "opb_ms_deform_attn_fwd")
    _count()
    return out


def ms_deform_attn_bwd(value, proj, ref, d_out, shapes, starts, N, Lq, H, P, d_value=None, d_proj=None):
    """Adjoint of ms_deform_attn_fwd for d_out bf16 [N * Lq, H * 32] -> (d_value fp32 [N * S_in, H * 32], accumulated into
    (zeroed when not given), d_proj fp32 [N * Lq, 3 * H * L * P], overwritten)."""
    _need_cuda(value, proj, ref, d_out, d_value, d_proj)
    L = len(shapes)
    S_in = value.shape[0] // N
    _msda_check(value, proj, ref, N, S_in, Lq, H, L, P)
    assert d_out.dtype == torch.bfloat16 and d_out.shape == (N * Lq, H * 32) and d_out.is_contiguous()
    if d_value is None:
        d_value = torch.zeros(value.shape, dtype=torch.float32, device=value.device)
    if d_proj is None:
        d_proj = torch.empty(proj.shape, dtype=torch.float32, device=value.device)
    assert d_value.dtype == torch.float32 and d_value.shape == value.shape and d_value.is_contiguous()
    assert d_proj.dtype == torch.float32 and d_proj.shape == proj.shape and d_proj.is_contiguous()
    hw, st = _msda_levels(shapes, starts)
    s = _lib.load().opb_ms_deform_attn_bwd(value.data_ptr(), proj.data_ptr(), ref.data_ptr(), d_out.data_ptr(),
                                           d_value.data_ptr(), d_proj.data_ptr(), N, S_in, Lq, H, 32, L, P, ref.shape[1], hw,
                                           st, _stream())
    _lib.check(s, "opb_ms_deform_attn_bwd")
    _count()
    return d_value, d_proj


def gemm_ln(a, w, epi, out, *, ln_mu=None, ln_rstd=None, ln_colsum=None, bias=None, colscale=None, gamma=None,
            resid=None, stats_out=None, out_bf16=None, cta_group=0, workspace=None, ln_partial=None, out_group=0,
            out_group_stride=0, out_row_offset=0, out_group_valid=0, resid_period=0, resid_row_offset=0):
    """GEMM through `opb_gemm_bf16_ex`: fused LayerNorm of the A operand (ln_*), statistics / bf16 side outputs, and the
    row remapping of `gemm`."""
    _need_cuda(a, w, out)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.stride(-1) == 1 and w.stride(1) == 1
    M, Kd = a.shape
    N = w.shape[0]
    args = _lib.GemmArgs()
    args.A, args.lda, args.B, args.ldb = a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0)
    args.M, args.N, args.K, args.epi = M, N, Kd, epi
    args.out, args.ldo = out.data_ptr(), out.stride(-2)
    args.bias, args.colscale, args.gamma, args.resid = _ptr(bias) or None, _ptr(colscale) or None, _ptr(gamma) or None, _ptr(resid) or None
    args.ldr = resid.stride(-2) if resid is not None else 0
    args.ln_mu, args.ln_rstd, args.ln_colsum = _ptr(ln_mu) or None, _ptr(ln_rstd) or None, _ptr(ln_colsum) or None
    args.stats_out = _ptr(stats_out) or None
    args.out_bf16 = _ptr(out_bf16) or None
    args.ldo_bf16 = out_bf16.stride(-2) if out_bf16 is not None else 0
    args.cta_group = cta_group
    args.out_group, args.out_group_stride, args.out_row_offset = out_group, out_group_stride, out_row_offset
    args.out_group_valid, args.resid_period, args.resid_row_offset = out_group_valid, resid_period, resid_row_offset
    if ln_partial is not None:      # (records tensor, parts, dim, eps)
        args.ln_partial, args.ln_parts, args.ln_dim, args.ln_eps = ln_partial[0].data_ptr(), ln_partial[1], ln_partial[2], ln_partial[3]
    if workspace is not None:
        args.workspace, args.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    if PROFILE_HOOK is not None:
        PROFILE_HOOK("gemm_begin", 0.0, None)
    import ctypes as _ct
    st = _lib.load().opb_gemm_bf16_ex(_ct.addressof(args), _stream())
    _lib.check(st, "opb_gemm_bf16_ex")
    _count()
    if PROFILE_HOOK is not None:
        PROFILE_HOOK("gemm", 2.0 * M * N * Kd, (M, N, Kd, epi))
    return out


def row_stats_cast(x, out_bf16, mu, rstd, eps=1e-5):
    rows, dim = x.shape
    st = _lib.load().opb_row_stats_cast(x.data_ptr(), x.stride(0), out_bf16.data_ptr(), out_bf16.stride(0), mu.data_ptr(),
                                        rstd.data_ptr(), rows, dim, eps, _stream())
    _lib.check(st, "opb_row_stats_cast")
    _count()


def ln_stats_finalize(partial, parts, rows, dim, eps, mu, rstd):
    st = _lib.load().opb_ln_stats_finalize(partial.data_ptr(), parts, rows, dim, eps, mu.data_ptr(), rstd.data_ptr(),
                                           _stream())
    _lib.check(st, "opb_ln_stats_finalize")
    _count()


def attention(qkv, bias, key_pad, B, S, H, out=None, lse=None, ln_stats=None):
    """attention, any S (wgmma kernel for S <= 224, mma.sync above).  bias: dense fp32 (H,S,S_pad) shared by the batch, or
    (B,H,S,S_pad) per sample."""
    _need_cuda(qkv, bias, key_pad)
    D = H * 64
    assert qkv.dtype == torch.bfloat16 and qkv.shape == (B * S, 3 * D) and qkv.is_contiguous()
    if out is None:
        out = torch.empty(B * S, D, dtype=torch.bfloat16, device=qkv.device)
    s_pad, bstride = 0, 0
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.shape[-3] == H and bias.shape[-2] == S
        s_pad = bias.shape[-1]
        if bias.dim() == 4:
            assert bias.shape[0] == B
            bstride = H * S * s_pad
    if key_pad is not None:
        assert key_pad.dtype == torch.uint8 and key_pad.shape == (B, S) and key_pad.is_contiguous()
    st = _lib.load().opb_attention_fwd(qkv.data_ptr(), _ptr(bias), _ptr(key_pad), out.data_ptr(), _ptr(lse),
                                       _ptr(ln_stats), B, S, H, s_pad, bstride, _stream())
    _lib.check(st, "opb_attention_fwd")
    _count()
    return out


def layernorm(x, gamma, beta, out, *, rows=None, dim=None, ld_in=None, ld_out=None, eps=1e-5, gelu=False,
              merge_grid_w=0, row_period=0, row_valid=0, out_period=0, out_row_shift=0, group_in=0, group_out=0,
              accumulate=False):
    _need_cuda(x, out)
    if rows is None:
        rows = x.shape[0]
    if dim is None:
        dim = x.shape[-1]
    if ld_in is None:
        ld_in = x.stride(-2)
    if ld_out is None:
        ld_out = out.stride(-2)
    st = _lib.load().opb_layernorm(x.data_ptr(), _dt(x), ld_in, out.data_ptr(), _dt(out), ld_out, _ptr(gamma),
                                   _ptr(beta), rows, dim, eps, int(gelu), merge_grid_w, row_period, row_valid,
                                   out_period, out_row_shift, group_in, group_out, int(accumulate), _stream())
    _lib.check(st, "opb_layernorm")
    _count()
    return out


def grouped_conv1d(x_halo, w, bias, out, rows, groups, c_pad, taps, n_per_group, epi=EPI_STORE_BF16):
    """out[r, g*n+co] = bias + sum_j sum_c x_halo[r+j, g, c] * w[g*n+co, j*c_pad+c]  (see onepeace_b200.h)."""
    _need_cuda(x_halo, w, out)
    assert x_halo.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x_halo.is_contiguous() and w.is_contiguous()
    assert x_halo.numel() >= (rows + taps - 1) * groups * c_pad and w.shape == (groups * n_per_group, taps * c_pad)
    st = _lib.load().opb_grouped_conv1d_bf16(x_halo.data_ptr(), w.data_ptr(), rows, groups, c_pad, taps, n_per_group,
                                             epi, out.data_ptr(), out.stride(-2), _ptr(bias), _stream())
    _lib.check(st, "opb_grouped_conv1d_bf16")
    _count()
    return out


def pack_group_halo(x, out, B, T, x_period, x_row_shift, out_period, halo, dim, group_in, group_out):
    _need_cuda(x, out)
    assert x.dtype == torch.float32 and out.dtype == torch.bfloat16
    st = _lib.load().opb_pack_group_halo(x.data_ptr(), x.stride(-2), out.data_ptr(), B, T, x_period, x_row_shift,
                                         out_period, halo, dim, group_in, group_out, _stream())
    _lib.check(st, "opb_pack_group_halo")
    _count()
    return out


def text_embed(tokens, table, pos, cls, pad_idx=1):
    """-> (x fp32 [B,T+1,D], pad_mask uint8 [B,T+1])"""
    _need_cuda(tokens, table, pos, cls)
    B, T = tokens.shape
    D = table.shape[1]
    assert tokens.dtype == torch.int64 and tokens.is_contiguous() and table.is_contiguous()
    assert pos.dtype == torch.float32 and cls.dtype == torch.float32 and pos.shape[0] >= T + 1
    x = torch.empty(B, T + 1, D, dtype=torch.float32, device=tokens.device)
    pad = torch.empty(B, T + 1, dtype=torch.uint8, device=tokens.device)
    st = _lib.load().opb_text_embed(tokens.data_ptr(), table.data_ptr(), _dt(table), pos.data_ptr(), cls.data_ptr(),
                                    x.data_ptr(), pad.data_ptr(), B, T, D, pad_idx, _stream())
    _lib.check(st, "opb_text_embed")
    _count()
    return x, pad


def image_patchify4(img):
    _need_cuda(img)
    B, C, R, R2 = img.shape
    assert C == 3 and R == R2 and img.is_contiguous()
    out = torch.empty(B * (R // 4) * (R // 4), 48, dtype=torch.bfloat16, device=img.device)
    st = _lib.load().opb_image_patchify4(img.data_ptr(), _dt(img), out.data_ptr(), B, R, _stream())
    _lib.check(st, "opb_image_patchify4")
    _count()
    return out


def cls_row_init(cls, pos0, x):
    """x fp32 [B,S,D]: x[:,0,:] = cls + pos0"""
    _need_cuda(cls, pos0, x)
    B, S, D = x.shape
    st = _lib.load().opb_cls_row_init(cls.data_ptr(), pos0.data_ptr(), x.data_ptr(), S * D, B, D, _stream())
    _lib.check(st, "opb_cls_row_init")
    _count()
    return x


def relpos_bias_build(table, bucket, S, H):
    """table fp32 [NB,H], bucket int64 [R,R] -> fp32 [H,S,s_pad]"""
    _need_cuda(table, bucket)
    assert table.dtype == torch.float32 and table.is_contiguous() and table.shape[1] == H
    assert bucket.dtype == torch.int64 and bucket.stride(1) == 1 and bucket.shape[0] >= S and bucket.shape[1] >= S
    s_pad = (S + 7) // 8 * 8
    bias = torch.empty(H, S, s_pad, dtype=torch.float32, device=table.device)
    st = _lib.load().opb_relpos_bias_build(table.data_ptr(), bucket.data_ptr(), bias.data_ptr(), S, s_pad, H,
                                           bucket.stride(0), _stream())
    _lib.check(st, "opb_relpos_bias_build")
    _count()
    return bias


def audio_frame10(wav, pitch, out):
    _need_cuda(wav, out)
    B, N = wav.shape
    assert wav.is_contiguous()
    st = _lib.load().opb_audio_frame10(wav.data_ptr(), _dt(wav), out.data_ptr(), B, N, pitch, _stream())
    _lib.check(st, "opb_audio_frame10")
    _count()
    return out


def l2_normalize_rows(x, want_bf16=False):
    _need_cuda(x)
    assert x.dtype == torch.float32 and x.stride(1) == 1
    rows, D = x.shape
    y = torch.empty(rows, D, dtype=torch.float32, device=x.device)
    y16 = torch.empty(rows, D, dtype=torch.bfloat16, device=x.device) if want_bf16 else None
    st = _lib.load().opb_l2_normalize_rows(x.data_ptr(), x.stride(0), y.data_ptr(), _ptr(y16), rows, D, _stream())
    _lib.check(st, "opb_l2_normalize_rows")
    _count()
    return (y, y16) if want_bf16 else y


def zero_padded_rows(x, pad_mask):
    _need_cuda(x, pad_mask)
    D = x.shape[-1]
    rows = x.numel() // D
    assert x.dtype == torch.float32 and x.is_contiguous() and pad_mask.dtype == torch.uint8 and pad_mask.numel() == rows
    st = _lib.load().opb_zero_padded_rows(x.data_ptr(), pad_mask.data_ptr(), rows, D, _stream())
    _lib.check(st, "opb_zero_padded_rows")
    _count()
    return x


# ----------------------------------------------------------------------------------------------------
# contrastive head
# ----------------------------------------------------------------------------------------------------
def transpose_bf16(x, rows=None, cols=None):
    """bf16 [rows, cols] view (row pitch x.stride(0)) -> contiguous [cols, rows]"""
    _need_cuda(x)
    assert x.dtype == torch.bfloat16 and x.stride(1) == 1 and x.dim() == 2
    rows = x.shape[0] if rows is None else rows
    cols = x.shape[1] if cols is None else cols
    out = torch.empty(cols, rows, dtype=torch.bfloat16, device=x.device)
    st = _lib.load().opb_transpose_bf16(x.data_ptr(), x.stride(0), out.data_ptr(), rows, cols, _stream())
    _lib.check(st, "opb_transpose_bf16")
    _count()
    return out


def split_bf16x3(xs, sides):
    """fp32 [r_i, d] tensors (1 to 4) -> bf16 [r_i, 3d] splits in ONE launch; side 0 = [hi|hi|lo] (local operand),
    side 1 = [hi|lo|hi] (gathered operand)."""
    import ctypes
    count = len(xs)
    assert 1 <= count <= 4 and len(sides) == count
    d = xs[0].shape[1]
    for x in xs:
        _need_cuda(x)
        assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2 and x.shape[1] == d
    outs = [torch.empty(x.shape[0], 3 * d, dtype=torch.bfloat16, device=x.device) for x in xs]
    px = (ctypes.c_void_p * count)(*[x.data_ptr() for x in xs])
    po = (ctypes.c_void_p * count)(*[o.data_ptr() for o in outs])
    pr = (ctypes.c_int64 * count)(*[x.shape[0] for x in xs])
    ps = (ctypes.c_int * count)(*[int(v) for v in sides])
    st = _lib.load().opb_split_bf16x3(ctypes.cast(px, ctypes.c_void_p), ctypes.cast(po, ctypes.c_void_p),
                                      ctypes.cast(pr, ctypes.c_void_p), ctypes.cast(ps, ctypes.c_void_p), count, d, _stream())
    _lib.check(st, "opb_split_bf16x3")
    _count()
    return outs


_TICKETS = {}


def infonce_forward(pairs, scale, target_offset, eps, n_valid=0, rows=False):
    """InfoNCE forward of one direction, pairs = [(a3, b_all3)], or of both, pairs = [(a3, b_all3), (b3, a_all3)]: one
    LSE_PARTIAL GEMM per direction + one merge / reduce kernel.  a3 bf16 [b,k], b_all3 bf16 [n,k], scale fp32 device scalar.
    n_valid > 0: only the first n_valid rows of b_all3 are classes (the rest is zero padding to n % 8 == 0).
    -> ([row_lse [b] per direction], out3 = {mean row loss over all directions, #correct a->b, #correct b->a (0 for one
    direction)}), and with `rows` also the row losses [dirs * b] and arg-max columns int32 [dirs * b] (direction a, then b)"""
    dirs = len(pairs)
    assert dirs in (1, 2)
    b, k = pairs[0][0].shape
    n = pairs[0][1].shape[0]
    _need_cuda(scale)
    assert scale.dtype == torch.float32
    for x, y in pairs:
        _need_cuda(x, y)
        assert x.dtype == torch.bfloat16 and y.dtype == torch.bfloat16 and x.is_contiguous() and y.is_contiguous()
        assert x.shape == (b, k) and y.shape == (n, k)
    lib = _lib.load()
    dev = pairs[0][0].device
    ws = []
    for x, y in pairs:
        w = torch.empty(lib.opb_infonce_ws_floats(b, n), dtype=torch.float32, device=dev)
        st = lib.opb_infonce_lse_gemm(x.data_ptr(), y.data_ptr(), scale.data_ptr(), b, n, k, target_offset, w.data_ptr(), int(n_valid),
                                      _stream())
        _lib.check(st, "opb_infonce_lse_gemm")
        ws.append(w)
    lse = [torch.empty(b, dtype=torch.float32, device=dev) for _ in pairs]
    loss_ab = torch.empty(dirs * b, dtype=torch.float32, device=dev)
    am_ab = torch.empty(dirs * b, dtype=torch.int32, device=dev)
    out3 = torch.empty(3, dtype=torch.float32, device=dev)
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    if key not in _TICKETS:
        _TICKETS[key] = torch.zeros(1, dtype=torch.int32, device=dev)       # the kernel leaves it at zero
    ws_b, lse_b = (ws[1], lse[1]) if dirs == 2 else (None, None)
    st = lib.opb_infonce_merge_reduce(ws[0].data_ptr(), _ptr(ws_b), b, n, int(n_valid), float(eps), target_offset, lse[0].data_ptr(),
                                      _ptr(lse_b), loss_ab.data_ptr(), am_ab.data_ptr(), out3.data_ptr(), _TICKETS[key].data_ptr(),
                                      _stream())
    _lib.check(st, "opb_infonce_merge_reduce")
    _count(dirs + 1)
    if rows:
        return lse, out3, loss_ab, am_ab
    return lse, out3


def infonce_grad(a_local, b_all, scale, row_lse, target_offset, eps, d, n_valid=0, coef=0.0):
    """-> (grad_a fp32 [b,d], ws_gz) for one direction; a_local/b_all [.,k] (k = d or 3d); b_all is read in place as an
    MN-major operand.  coef = weight of one row's loss (0 -> 1 / (2 b), the two-direction InfoNCE mean)"""
    b, k = a_local.shape
    n = b_all.shape[0]
    dev = a_local.device
    g_ws = torch.empty(b, n, dtype=torch.bfloat16, device=dev)
    ws_gz = torch.empty((n + 255) // 256 * b, dtype=torch.float32, device=dev)
    grad = torch.empty(b, d, dtype=torch.float32, device=dev)
    st = _lib.load().opb_infonce_grad(a_local.data_ptr(), b_all.data_ptr(), scale.data_ptr(),
                                      row_lse.data_ptr(), b, n, d, k, target_offset, eps, g_ws.data_ptr(),
                                      ws_gz.data_ptr(), grad.data_ptr(), int(n_valid), float(coef), _stream())
    _lib.check(st, "opb_infonce_grad")
    _count(2)
    return grad, ws_gz


def infonce_dscale(ws_a, ws_b, b, n):
    out = torch.empty(1, dtype=torch.float32, device=ws_a.device)
    st = _lib.load().opb_infonce_dscale(ws_a.data_ptr(), ws_b.data_ptr(), b, n, out.data_ptr(), _stream())
    _lib.check(st, "opb_infonce_dscale")
    _count()
    return out


# ----------------------------------------------------------------------------------------------------------------
# backward pass
# ----------------------------------------------------------------------------------------------------------------
_BWD_WS = {}


def bwd_ws(dim, device):
    """fp32 scratch for the column-reduction kernels (per device, grown on demand)."""
    need = _lib.load().opb_bwd_ws_floats(int(dim))
    key = (device.index if device.index is not None else torch.cuda.current_device())
    ws = _BWD_WS.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.float32, device=device)
        _BWD_WS[key] = ws
    return ws


def layernorm_bwd(x, dy, gamma, beta, dx, *, eps=1e-5, gelu=False, accumulate=False, dgamma=None, dbeta=None, rows=None,
                  dim=None, ldx=None, ld_dx=None, dy_merge_w=0):
    """x, dy, dx: [rows, dim] (fp32 / bf16, row stride free); dgamma / dbeta fp32 [dim] outputs (optional)."""
    _need_cuda(x, dy, dx)
    rows = x.shape[0] if rows is None else rows
    dim = x.shape[-1] if dim is None else dim
    ws = bwd_ws(dim, x.device) if (dgamma is not None or dbeta is not None) else None
    st = _lib.load().opb_layernorm_bwd(x.data_ptr(), _dt(x), x.stride(-2) if ldx is None else ldx, dy.data_ptr(), _dt(dy),
                                       dy.stride(-2), _ptr(gamma), _ptr(beta), dx.data_ptr(), _dt(dx),
                                       dx.stride(-2) if ld_dx is None else ld_dx, int(accumulate), rows, dim, eps,
                                       int(gelu), dy_merge_w, _ptr(ws), _ptr(dgamma), _ptr(dbeta), _stream())
    _lib.check(st, "opb_layernorm_bwd")
    _count(1 + (dgamma is not None) + (dbeta is not None))
    return dx


def geglu_fwd(gl, u):
    rows, F2 = gl.shape
    st = _lib.load().opb_geglu_fwd(gl.data_ptr(), u.data_ptr(), rows, F2 // 2, _stream())
    _lib.check(st, "opb_geglu_fwd")
    _count()
    return u


def geglu_bwd(gl, du, dgl):
    rows, F2 = gl.shape
    st = _lib.load().opb_geglu_bwd(gl.data_ptr(), du.data_ptr(), dgl.data_ptr(), rows, F2 // 2, _stream())
    _lib.check(st, "opb_geglu_bwd")
    _count()
    return dgl


def gelu_fwd(z, y):
    """y = gelu_erf(z), bf16 [rows, F] (row-contiguous)"""
    rows, F = z.shape
    assert z.is_contiguous() and y.is_contiguous() and y.shape == z.shape
    st = _lib.load().opb_gelu_fwd(z.data_ptr(), y.data_ptr(), rows, F, _stream())
    _lib.check(st, "opb_gelu_fwd")
    _count()
    return y


def gelu_bwd(z, dy, dz):
    """dz = dy * gelu'(z), bf16 [rows, F]"""
    rows, F = z.shape
    assert z.is_contiguous() and dy.is_contiguous() and dz.is_contiguous() and dy.shape == z.shape == dz.shape
    st = _lib.load().opb_gelu_bwd(z.data_ptr(), dy.data_ptr(), dz.data_ptr(), rows, F, _stream())
    _lib.check(st, "opb_gelu_bwd")
    _count()
    return dz


def scale_resid_fwd(x, o, gamma, row_scale, out):
    rows, n = x.shape
    st = _lib.load().opb_scale_resid_fwd(x.data_ptr(), o.data_ptr(), _ptr(gamma), _ptr(row_scale), out.data_ptr(), rows, n,
                                         _stream())
    _lib.check(st, "opb_scale_resid_fwd")
    _count()
    return out


def scale_resid_bwd(dx, o, gamma, row_scale, d_o, dgamma=None, dbias=None, in_period=0, in_valid=0, in_shift=0):
    """d_o bf16 [rows, n] = row_scale * gamma * dx (rows of dx optionally gathered, see onepeace_b200.h)."""
    rows, n = d_o.shape
    ws = bwd_ws(n, dx.device)
    st = _lib.load().opb_scale_resid_bwd(dx.data_ptr(), _ptr(o), _ptr(gamma), _ptr(row_scale), d_o.data_ptr(), ws.data_ptr(),
                                         _ptr(dgamma), _ptr(dbias), rows, n, in_period, in_valid, in_shift, _stream())
    _lib.check(st, "opb_scale_resid_bwd")
    _count(1 + (dgamma is not None) + (dbias is not None))
    return d_o


def colsum(y, out):
    rows, n = y.shape
    ws = bwd_ws(n, y.device)
    st = _lib.load().opb_colsum_bf16(y.data_ptr(), y.stride(0), ws.data_ptr(), out.data_ptr(), rows, n, _stream())
    _lib.check(st, "opb_colsum_bf16")
    _count(2)
    return out


def attention_bwd(qkv, out, d_out, bias, key_pad, lse, dqkv, dbias, B, S, H, q_scale):
    """bias / dbias: dense fp32 (H,S,S_pad) tables shared by the batch, (B,H,S,S_pad) per-sample tables, or None;
    lse fp32 [B,H,S] from `attention(..., lse=)`."""
    delta = torch.empty(B * H * S, dtype=torch.float32, device=qkv.device)
    s_pad = bias.shape[-1] if bias is not None else 0
    bstride = H * S * s_pad if (bias is not None and bias.dim() == 4) else 0
    if dbias is not None:
        assert dbias.shape == bias.shape
    st = _lib.load().opb_attention_bwd(qkv.data_ptr(), out.data_ptr(), d_out.data_ptr(), _ptr(bias), _ptr(key_pad),
                                       lse.data_ptr(), delta.data_ptr(), dqkv.data_ptr(), _ptr(dbias), B, S, H, s_pad,
                                       float(q_scale), bstride, _stream())
    _lib.check(st, "opb_attention_bwd")
    _count(3)
    return dqkv


BIAS_T_KEYS, BIAS_T_Q = 256, 224      # transposed bias tables of the attention backward (csrc/attention_bwd.cu)


def relpos_bias_transpose(bias):
    """dense fp32 (H,S,S_pad) bias -> (H,256,112) half2 words (int32 storage), x log2 e, zero-padded; S <= 224."""
    H, S, s_pad = bias.shape
    out = torch.empty(H, BIAS_T_KEYS, BIAS_T_Q // 2, dtype=torch.int32, device=bias.device)
    st = _lib.load().opb_relpos_bias_transpose(bias.data_ptr(), out.data_ptr(), S, s_pad, H, _stream())
    _lib.check(st, "opb_relpos_bias_transpose")
    _count()
    return out


def relpos_dbias_fold(dbias_t, dbias):
    """dbias fp32 (H,S,S_pad) += transpose of dbias_t fp32 (H,256,224)"""
    H, S, s_pad = dbias.shape
    st = _lib.load().opb_relpos_dbias_fold(dbias_t.data_ptr(), dbias.data_ptr(), S, s_pad, H, _stream())
    _lib.check(st, "opb_relpos_dbias_fold")
    _count()
    return dbias


def relpos_dbias_center(dbias):
    """in place: every row of the dense fp32 (H,S,S_pad) bias gradient gets its mean over the S valid columns subtracted"""
    H, S, s_pad = dbias.shape
    st = _lib.load().opb_relpos_dbias_center(dbias.data_ptr(), S, s_pad, H, _stream())
    _lib.check(st, "opb_relpos_dbias_center")
    _count()
    return dbias


def attention_bwd_t(qkv, out, d_out, bias_t, key_pad, lse, dqkv, dbias_t, B, S, H, q_scale):
    """attention backward with transposed bias tables (relpos_bias_transpose / a zeroed (H,256,224) fp32 dbias_t that
    several layers may share); S <= 224."""
    delta = torch.empty(B * H * S, dtype=torch.float32, device=qkv.device)
    st = _lib.load().opb_attention_bwd_t(qkv.data_ptr(), out.data_ptr(), d_out.data_ptr(), _ptr(bias_t), _ptr(key_pad),
                                         lse.data_ptr(), delta.data_ptr(), dqkv.data_ptr(), _ptr(dbias_t), B, S, H,
                                         float(q_scale), _stream())
    _lib.check(st, "opb_attention_bwd_t")
    _count(2)
    return dqkv


def relpos_bias_bwd(dbias, bucket, dtable, S):
    H, s_pad = dbias.shape[0], dbias.shape[-1]
    st = _lib.load().opb_relpos_bias_bwd(dbias.data_ptr(), bucket.data_ptr(), dtable.data_ptr(), S, s_pad, H, bucket.stride(0),
                                         _stream())
    _lib.check(st, "opb_relpos_bias_bwd")
    _count()
    return dtable


def batch_sum(x, out, B, n, ld, accumulate=False):
    """out[c] (+)= sum_b x[b * ld + c], c < n (x is addressed through its data pointer: pass a view of the first row)"""
    st = _lib.load().opb_batch_sum_f32(x.data_ptr(), ld, out.data_ptr(), B, n, int(accumulate), _stream())
    _lib.check(st, "opb_batch_sum_f32")
    _count()
    return out


def l2_normalize_bwd(x, dy, want_f32=False):
    """x fp32 [rows, D] (the un-normalised rows), dy fp32 -> bf16 dx (and fp32 when asked)"""
    rows, D = x.shape
    dx16 = torch.empty(rows, D, dtype=torch.bfloat16, device=x.device)
    dx32 = torch.empty(rows, D, dtype=torch.float32, device=x.device) if want_f32 else None
    st = _lib.load().opb_l2_normalize_bwd(x.data_ptr(), x.stride(0), dy.data_ptr(), dy.stride(0), _ptr(dx32), dx16.data_ptr(),
                                          rows, D, _stream())
    _lib.check(st, "opb_l2_normalize_bwd")
    _count()
    return (dx16, dx32) if want_f32 else dx16


def text_embed_bwd(dx, tokens, dtable, dpos, dcls, pad_idx=1):
    B, T = tokens.shape
    D = dx.shape[-1]
    st = _lib.load().opb_text_embed_bwd(dx.data_ptr(), tokens.data_ptr(), dtable.data_ptr(), dpos.data_ptr(), dcls.data_ptr(),
                                        B, T, D, pad_idx, _stream())
    _lib.check(st, "opb_text_embed_bwd")
    _count()


def window_gather(x, B, t_in, t_out, stride, kw, pad, groups):
    """bf16 [B*t_in, C] -> [groups, B*t_out, kw*(C/groups)] convolution windows (see onepeace_b200.h)"""
    C = x.shape[1]
    cg = C // groups
    out = torch.empty(groups, B * t_out, kw * cg, dtype=torch.bfloat16, device=x.device)
    st = _lib.load().opb_window_gather(x.data_ptr(), out.data_ptr(), B, t_in, t_out, stride, kw, pad, groups, cg, _stream())
    _lib.check(st, "opb_window_gather")
    _count()
    return out


def window_scatter(dwin, B, t_in, t_out, stride, kw, pad):
    """adjoint of window_gather: bf16 [groups, B*t_out, kw*cg] -> [B*t_in, groups*cg]"""
    groups = dwin.shape[0]
    cg = dwin.shape[2] // kw
    dx = torch.empty(B * t_in, groups * cg, dtype=torch.bfloat16, device=dwin.device)
    st = _lib.load().opb_window_scatter(dwin.data_ptr(), dx.data_ptr(), B, t_in, t_out, stride, kw, pad, groups, cg, _stream())
    _lib.check(st, "opb_window_scatter")
    _count()
    return dx


def topk10_rows(sim, want_values=False):
    """fp32 [R, C] -> int32 [R, 10] column indices of the 10 largest entries per row (descending)"""
    _need_cuda(sim)
    assert sim.dtype == torch.float32 and sim.stride(1) == 1
    R, C = sim.shape
    idx = torch.empty(R, 10, dtype=torch.int32, device=sim.device)
    val = torch.empty(R, 10, dtype=torch.float32, device=sim.device) if want_values else None
    st = _lib.load().opb_topk10_rows(sim.data_ptr(), sim.stride(0), idx.data_ptr(), _ptr(val), R, C, _stream())
    _lib.check(st, "opb_topk10_rows")
    _count()
    return (idx, val) if want_values else idx


def recall_hits(idx, cand_ids, row_ids):
    """-> int32 [3]: rows whose id is among the ids of their top-1 / top-5 / top-10 candidates"""
    hits = torch.zeros(3, dtype=torch.int32, device=idx.device)
    st = _lib.load().opb_recall_hits(idx.data_ptr(), cand_ids.data_ptr(), row_ids.data_ptr(), idx.shape[0], hits.data_ptr(),
                                     _stream())
    _lib.check(st, "opb_recall_hits")
    _count()
    return hits


# ----------------------------------------------------------------------------------------------------------------
# pretraining path: row gathers, general dense relative-position bias
# ----------------------------------------------------------------------------------------------------------------
def row_gather(src, idx, out=None, fill=None, out_dtype=None, add=None):
    """out[r] = (src[idx[r]] if idx[r] >= 0 else fill (fp32 [dim]) / 0) + add[r % period] (add fp32 [period, dim] or None).
    src [n, dim] fp32 / bf16 (row stride free), idx int64 [rows]."""
    _need_cuda(src, idx)
    assert idx.dtype == torch.int64 and idx.is_contiguous() and src.stride(-1) == 1 and src.dim() == 2
    rows, dim = idx.numel(), src.shape[1]
    if out is None:
        out = torch.empty(rows, dim, dtype=out_dtype or src.dtype, device=src.device)
    if rows == 0:
        return out
    assert out.stride(-1) == 1 and (fill is None or (fill.dtype == torch.float32 and fill.is_contiguous()))
    assert add is None or (add.dtype == torch.float32 and add.is_contiguous() and add.shape[-1] == dim)
    st = _lib.load().opb_row_gather(src.data_ptr(), _dt(src), src.stride(0), idx.data_ptr(), _ptr(fill), _ptr(add),
                                    add.numel() // dim if add is not None else 0, out.data_ptr(), _dt(out), out.stride(-2),
                                    rows, dim, _stream())
    _lib.check(st, "opb_row_gather")
    _count()
    return out


def row_scatter_add(dout, idx, dsrc):
    """dsrc[idx[r]] += dout[r] for idx[r] >= 0; dsrc fp32 [n, dim] (caller zero-initialises)."""
    _need_cuda(dout, idx, dsrc)
    assert idx.dtype == torch.int64 and idx.is_contiguous() and dsrc.dtype == torch.float32 and dout.dim() == 2
    rows, dim = idx.numel(), dout.shape[1]
    if rows == 0:
        return dsrc
    st = _lib.load().opb_row_scatter_add(dout.data_ptr(), _dt(dout), dout.stride(0), idx.data_ptr(), dsrc.data_ptr(),
                                         dsrc.stride(-2), rows, dim, _stream())
    _lib.check(st, "opb_row_scatter_add")
    _count()
    return dsrc


def relpos_bias_block(table, bucket, ids, n, lo, bias, S, H):
    """Writes one modality's diagonal block of the dense bias canvas `bias` fp32 [Bb, H, S, s_pad] (Bb = 1 when ids is None):
    bias[bb, h, lo+i, lo+j] = table[bucket[p_i, p_j], h], p = ids[bb] (int64 [Bb, n], -1 = padded slot) or arange(n)."""
    _need_cuda(table, bucket, bias)
    assert table.dtype == torch.float32 and table.is_contiguous() and table.shape[1] == H and bias.is_contiguous()
    assert bucket.dtype == torch.int64 and bucket.stride(1) == 1 and bias.dim() == 4 and bias.shape[1] == H and bias.shape[2] == S
    Bb = bias.shape[0]
    if ids is not None:
        assert ids.dtype == torch.int64 and ids.shape == (Bb, n) and ids.stride(1) == 1
    st = _lib.load().opb_relpos_bias_block(table.data_ptr(), bucket.data_ptr(), bucket.stride(0), _ptr(ids),
                                           ids.stride(0) if ids is not None else 0, Bb, n, lo, bias.data_ptr(), S,
                                           bias.shape[3], H, _stream())
    _lib.check(st, "opb_relpos_bias_block")
    _count()
    return bias


def relpos_bias_block_bwd(dbias, bucket, ids, n, lo, dtable, S, H):
    Bb = dbias.shape[0]
    st = _lib.load().opb_relpos_bias_block_bwd(dbias.data_ptr(), bucket.data_ptr(), bucket.stride(0), _ptr(ids),
                                               ids.stride(0) if ids is not None else 0, Bb, n, lo, dtable.data_ptr(), S,
                                               dbias.shape[3], H, _stream())
    _lib.check(st, "opb_relpos_bias_block_bwd")
    _count()
    return dtable


def ln_fold(weight, ln_w, ln_b, bias, out_w, colsum, bias_out, interleave=0):
    """Folds LayerNorm(ln_w, ln_b) into the following Linear(weight, bias): writes the bf16 operand rows, their column sums and
    the fused bias into (views of) out_w / colsum / bias_out.  weight fp32 / bf16 [N, K]; ln_w / ln_b / bias fp32 or None."""
    _need_cuda(weight, out_w)
    N, Kd = weight.shape
    assert weight.stride(1) == 1 and out_w.dtype == torch.bfloat16 and out_w.stride(-1) == 1
    st = _lib.load().opb_ln_fold(weight.data_ptr(), _dt(weight), weight.stride(0), _ptr(ln_w), _ptr(ln_b), _ptr(bias), N, Kd,
                                 interleave, out_w.data_ptr(), out_w.stride(0), colsum.data_ptr(), bias_out.data_ptr(), _stream())
    _lib.check(st, "opb_ln_fold")
    _count()


def gemm_t(a, b, epi, out, a_mn=False, b_mn=False, bias=None, cta_group=0):
    """out[M, N] = A B^T with MN-major operands: a is [K, M] when a_mn else [M, K]; b is [K, N] when b_mn else [N, K]
    (bf16, unit column stride, free row pitch).  No transposed copies: TMA + UMMA read the row-contracted layout directly."""
    _need_cuda(a, b, out)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.stride(1) == 1 and b.stride(1) == 1
    Kd, M = (a.shape[0], a.shape[1]) if a_mn else (a.shape[1], a.shape[0])
    Kb, N = (b.shape[0], b.shape[1]) if b_mn else (b.shape[1], b.shape[0])
    assert Kd == Kb and out.shape == (M, N)
    st = _lib.load().opb_gemm_bf16_t(a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn), M, N, Kd, epi,
                                     out.data_ptr(), out.stride(0), _ptr(bias), cta_group, _stream())
    _lib.check(st, "opb_gemm_bf16_t")
    _count()
    if PROFILE_HOOK is not None:
        PROFILE_HOOK("gemm", 2.0 * M * N * Kd, (M, N, Kd, epi))
    return out


# ----------------------------------------------------------------------------------------------------------------
# classification head (csrc/classify.cu)
# ----------------------------------------------------------------------------------------------------------------
def attn_pool_fwd(kv, q, key_pad, B, T):
    """kv bf16 [B*T, 2d] (k | v), q fp32 [H, 64], key_pad uint8 [B, T] or None -> (out bf16 [B, d], lse fp32 [B, H])."""
    _need_cuda(kv, q, key_pad)
    d = kv.shape[1] // 2
    assert kv.dtype == torch.bfloat16 and kv.is_contiguous() and kv.shape[0] == B * T
    assert q.dtype == torch.float32 and q.is_contiguous() and q.numel() == d
    if key_pad is not None:
        assert key_pad.dtype == torch.uint8 and key_pad.shape == (B, T) and key_pad.is_contiguous()
    out = torch.empty(B, d, dtype=torch.bfloat16, device=kv.device)
    lse = torch.empty(B, d // 64, dtype=torch.float32, device=kv.device)
    st = _lib.load().opb_attn_pool_fwd(kv.data_ptr(), q.data_ptr(), _ptr(key_pad), out.data_ptr(), lse.data_ptr(), B, T, d,
                                       _stream())
    _lib.check(st, "opb_attn_pool_fwd")
    _count()
    return out, lse


def attn_pool_bwd(kv, q, key_pad, lse, dout, B, T):
    """Adjoint of attn_pool_fwd for dout bf16 [B, d] -> (dkv bf16 [B*T, 2d], dq fp32 [H, 64])."""
    _need_cuda(kv, q, key_pad, lse, dout)
    d = kv.shape[1] // 2
    assert dout.dtype == torch.bfloat16 and dout.is_contiguous() and dout.shape == (B, d)
    assert lse.dtype == torch.float32 and lse.is_contiguous() and lse.shape == (B, d // 64)
    if key_pad is not None:
        assert key_pad.dtype == torch.uint8 and key_pad.shape == (B, T) and key_pad.is_contiguous()
    dkv = torch.empty_like(kv)
    ws = torch.empty(B, d, dtype=torch.float32, device=kv.device)
    dq = torch.empty(d // 64, 64, dtype=torch.float32, device=kv.device)
    st = _lib.load().opb_attn_pool_bwd(kv.data_ptr(), q.data_ptr(), _ptr(key_pad), lse.data_ptr(), dout.data_ptr(), dkv.data_ptr(),
                                       ws.data_ptr(), dq.data_ptr(), B, T, d, _stream())
    _lib.check(st, "opb_attn_pool_bwd")
    _count(2)
    return dkv, dq


LOSS_HARD, LOSS_SOFT, LOSS_MULTI_LABEL, LOSS_HINGE = 0, 1, 2, 3
_LOSS_TICKETS = {}


def classify_loss(logits, n_valid, mode, labels=None, targets=None, eps=0.0, num_choices=1):
    """logits fp32 [rows, >= n_valid] (unit column stride, free row pitch; columns past n_valid are never read) ->
    (row_loss, dlogits fp32 shaped like logits' rows x pitch, row_correct, out2 = {loss sum, n_correct sum})."""
    _need_cuda(logits, labels, targets)
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    rows, ld = logits.shape[0], logits.stride(0)
    dev = logits.device
    if targets is not None:
        assert targets.dtype == torch.float32 and targets.stride(1) == 1
    if labels is not None:
        assert labels.dtype == torch.int64 and labels.is_contiguous()
    n_out = rows // num_choices if mode == LOSS_HINGE else rows
    row_loss = torch.empty(n_out, dtype=torch.float32, device=dev)
    row_correct = torch.empty(n_out, dtype=torch.float32, device=dev)
    dlogits = torch.empty(rows, ld, dtype=torch.float32, device=dev)
    out2 = torch.empty(2, dtype=torch.float32, device=dev)
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    if key not in _LOSS_TICKETS:
        _LOSS_TICKETS[key] = torch.zeros(1, dtype=torch.int32, device=dev)       # the kernel leaves it at zero
    st = _lib.load().opb_classify_loss(logits.data_ptr(), ld, rows, int(n_valid), int(mode), _ptr(labels), _ptr(targets),
                                       targets.stride(0) if targets is not None else 0, float(eps), int(num_choices),
                                       row_loss.data_ptr(), dlogits.data_ptr(), row_correct.data_ptr(), out2.data_ptr(),
                                       _LOSS_TICKETS[key].data_ptr(), _stream())
    _lib.check(st, "opb_classify_loss")
    _count()
    return row_loss, dlogits, row_correct, out2


# ----------------------------------------------------------------------------------------------------------------
# visual grounding (csrc/grounding.cu)
# ----------------------------------------------------------------------------------------------------------------
def refcoco_loss(logits, targets, nsentences):
    """logits fp32 [B, >= 4] (unit column stride, free row pitch ld; columns past 4 are never read), targets [B, 4] ->
    (out fp32 [3] = {loss, L1 part, n_valid}, valid int32 [B], giou fp32 [B], dlogits fp32 [B, ld] = d loss / d logits with
    zero pad columns).  The loss is NaN when no row is valid; dlogits stays finite (the L1 part)."""
    _need_cuda(logits, targets)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    B, ld = logits.shape[0], logits.stride(0)
    dev = logits.device
    t = targets.to(torch.float32).contiguous()
    assert t.shape == (B, 4)
    out = torch.empty(3, dtype=torch.float32, device=dev)
    valid = torch.empty(B, dtype=torch.int32, device=dev)
    giou = torch.empty(B, dtype=torch.float32, device=dev)
    dlogits = torch.empty(B, ld, dtype=torch.float32, device=dev)
    st = _lib.load().opb_refcoco_loss(logits.data_ptr(), ld, t.data_ptr(), B, int(nsentences), out.data_ptr(), valid.data_ptr(),
                                      giou.data_ptr(), dlogits.data_ptr(), _stream())
    _lib.check(st, "opb_refcoco_loss")
    _count()
    return out, valid, giou, dlogits


def iou_acc(hyps, refs, hits, row_hit=None):
    """hits int32 [1] += IoU >= 0.5 hits of hyps / refs fp32 [n, 4] (metrics/iou_acc.py:20-32); asynchronous.  row_hit: optional
    int32 [n] receiving the per-row flag."""
    _need_cuda(hyps, refs, hits, row_hit)
    assert hyps.dtype == torch.float32 and refs.dtype == torch.float32 and hyps.stride(1) == 1 and refs.stride(1) == 1
    assert hyps.shape == refs.shape and hyps.shape[1] == 4
    assert hits.dtype == torch.int32 and hits.numel() >= 1
    if row_hit is not None:
        assert row_hit.dtype == torch.int32 and row_hit.is_contiguous() and row_hit.numel() == hyps.shape[0]
    st = _lib.load().opb_iou_acc(hyps.data_ptr(), hyps.stride(0), refs.data_ptr(), refs.stride(0), hyps.shape[0], hits.data_ptr(),
                                 _ptr(row_hit), _stream())
    _lib.check(st, "opb_iou_acc")
    _count()
    return hits


# ----------------------------------------------------------------------------------------------------------------
# classification evaluation (csrc/metrics.cu)
# ----------------------------------------------------------------------------------------------------------------
def _view2d(x):
    """(dtype tag, row stride, column stride) of a 2-D fp32 / bf16 view, read in place (no copy of padded or strided rows)."""
    assert x.dim() == 2
    return _dt(x), max(x.stride(0), 1), max(x.stride(1), 1)


def argmax_hits(logits, targets, hyp=None, score=None):
    """metrics/accuracy.py:20-25: hyp int64 [n] = torch.argmax(logits, 1) and score fp32 [n] = the row's hit.  logits fp32 / bf16
    [n, C] with any strides; targets int64 labels [n], fp32 labels [n] (compared as torch.eq does) or fp32 soft scores [n, >= C]
    (score = targets[r, hyp]).  Asynchronous."""
    _need_cuda(logits, targets, hyp, score)
    dt, ld, cs = _view2d(logits)
    n, C = logits.shape
    if targets.dim() == 2:
        t = targets if targets.dtype == torch.float32 and targets.stride(1) == 1 else targets.to(torch.float32).contiguous()
        assert t.shape[0] == n and t.shape[1] >= C
        tmode, ldt = 2, max(t.stride(0), 1)
    else:
        assert targets.dim() == 1 and targets.shape[0] == n
        if targets.dtype == torch.int64:
            t, tmode = targets.contiguous(), 0
        elif targets.is_floating_point() or targets.dtype == torch.bool:
            t, tmode = targets.to(torch.float32).contiguous(), 1
        else:
            t, tmode = targets.to(torch.int64).contiguous(), 0
        ldt = 0
    dev = logits.device
    hyp = torch.empty(n, dtype=torch.int64, device=dev) if hyp is None else hyp
    score = torch.empty(n, dtype=torch.float32, device=dev) if score is None else score
    assert hyp.dtype == torch.int64 and hyp.is_contiguous() and hyp.numel() >= n
    assert score.dtype == torch.float32 and score.is_contiguous() and score.numel() >= n
    st = _lib.load().opb_argmax_hits(logits.data_ptr(), dt, ld, cs, n, C, t.data_ptr(), tmode, ldt, hyp.data_ptr(),
                                     score.data_ptr(), _stream())
    _lib.check(st, "opb_argmax_hits")
    _count()
    return hyp, score


def sum_f64(x, out=None):
    """fp64 [1] = sum of x fp32 [n] in a fixed order (bit-identical on every run)."""
    _need_cuda(x, out)
    assert x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty(1, dtype=torch.float64, device=x.device) if out is None else out
    st = _lib.load().opb_sum_f64(x.data_ptr(), x.numel(), out.data_ptr(), _stream())
    _lib.check(st, "opb_sum_f64")
    _count()
    return out


def sigmoid_pack(logits, targets, probs, labels, row_offset, flags):
    """metrics/map.py:20-23 + the sigmoid of :34: probs[row_offset + r] = torch.sigmoid(float(logits[r])) bit for bit, labels
    uint8 = (targets == 1), flags int32 [2] += (targets outside {0, 1}, NaN probabilities).  logits fp32 / bf16 [n, C], any
    strides; targets fp32 [n, C]; probs fp32 / labels uint8 [>= row_offset + n, C] contiguous.  Asynchronous."""
    _need_cuda(logits, targets, probs, labels, flags)
    dt, ld, cs = _view2d(logits)
    n, C = logits.shape
    t = targets if targets.dtype == torch.float32 and targets.stride(1) == 1 else targets.to(torch.float32).contiguous()
    assert t.shape == (n, C)
    assert probs.dtype == torch.float32 and probs.is_contiguous() and probs.shape[1] == C and probs.shape[0] >= row_offset + n
    assert labels.dtype == torch.uint8 and labels.is_contiguous() and labels.shape == probs.shape
    assert flags.dtype == torch.int32 and flags.numel() >= 2
    st = _lib.load().opb_sigmoid_pack(logits.data_ptr(), dt, ld, cs, t.data_ptr(), max(t.stride(0), 1), n, C, probs.data_ptr(),
                                      labels.data_ptr(), row_offset, flags.data_ptr(), _stream())
    _lib.check(st, "opb_sigmoid_pack")
    _count()


def average_precision(probs, labels):
    """sklearn.metrics.average_precision_score(labels, probs, average=None) and its mean: probs fp32 [N, C] in [0, 1], labels
    uint8 [N, C] -> (ap fp64 [C], mean fp64 [1], npos int64 [C]); ap is 0 for a class without positives."""
    _need_cuda(probs, labels)
    assert probs.dtype == torch.float32 and probs.is_contiguous() and labels.dtype == torch.uint8 and labels.is_contiguous()
    assert probs.dim() == 2 and labels.shape == probs.shape
    N, C = probs.shape
    lib = _lib.load()
    nbytes = lib.opb_average_precision_ws_bytes(N, C)
    if nbytes < 0:
        raise RuntimeError(f"opb_average_precision: shape {N} x {C} is outside 1 <= N < 2^24, 1 <= C <= 4096, N * C < 2^31")
    dev = probs.device
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    ap = torch.empty(C, dtype=torch.float64, device=dev)
    mean = torch.empty(1, dtype=torch.float64, device=dev)
    npos = torch.empty(C, dtype=torch.int64, device=dev)
    st = lib.opb_average_precision(probs.data_ptr(), labels.data_ptr(), N, C, ws.data_ptr(), nbytes, ap.data_ptr(),
                                   mean.data_ptr(), npos.data_ptr(), _stream())
    _lib.check(st, "opb_average_precision")
    _count(4 + 3 * ((31 + max(C - 1, 0).bit_length() + 7) // 8))
    return ap, mean, npos


# ----------------------------------------------------------------------------------------------------------------
# pooled head of OnePeaceViT (csrc/vit_head.cu)
# ----------------------------------------------------------------------------------------------------------------
def _check_rows3(x, name):
    """(B, S, d, row pitch) of an fp32 [B, S, d] view whose rows are d contiguous floats at one pitch."""
    if x.dtype != torch.float32 or x.dim() != 3 or x.stride(2) != 1 or x.stride(0) != x.shape[1] * x.stride(1):
        raise ValueError(f"{name}: fp32 [B, S, d] with unit column stride and one row pitch expected")
    return x.shape[0], x.shape[1], x.shape[2], x.stride(1)


def token_mean_ln_fwd(x, gamma, beta, eps):
    """x fp32 [B, S, d] (any row pitch) -> (y bf16 [B, d], m fp32 [B, d], mean fp32 [B], rstd fp32 [B]):
    y = LayerNorm(x[:, 1:].mean(1)) with gamma / beta fp32 [d] (models_vit.py:431-434, global_pool=True)."""
    _need_cuda(x, gamma, beta)
    B, S, d, ld = _check_rows3(x, "token_mean_ln_fwd")
    for t in (gamma, beta):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != d:
            raise ValueError("token_mean_ln_fwd: gamma / beta must be contiguous fp32 [d]")
    lib = _lib.load()
    n_ws = lib.opb_token_mean_ln_ws_floats(B, S, d)
    if n_ws < 0:
        raise ValueError(f"token_mean_ln_fwd: unsupported shape B={B}, S={S}, d={d}")
    dev = x.device
    ws = torch.empty(n_ws, dtype=torch.float32, device=dev)
    m = torch.empty(B, d, dtype=torch.float32, device=dev)
    y = torch.empty(B, d, dtype=torch.bfloat16, device=dev)
    mean = torch.empty(B, dtype=torch.float32, device=dev)
    rstd = torch.empty(B, dtype=torch.float32, device=dev)
    st = lib.opb_token_mean_ln_fwd(x.data_ptr(), ld, B, S, d, gamma.data_ptr(), beta.data_ptr(), float(eps), ws.data_ptr(), n_ws,
                                   m.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), _stream())
    _lib.check(st, "opb_token_mean_ln_fwd")
    _count(2)
    return y, m, mean, rstd


def token_mean_ln_bwd(dy, m, mean, rstd, gamma, dx):
    """Adjoint of token_mean_ln_fwd for dy fp32 [B, d]: writes dx fp32 [B, S, d] (any row pitch; every row, the CLS row as
    zeros) and returns (dgamma fp32 [d], dbeta fp32 [d])."""
    _need_cuda(dy, m, mean, rstd, gamma, dx)
    B, S, d, ld = _check_rows3(dx, "token_mean_ln_bwd")
    for t, shape in ((dy, (B, d)), (m, (B, d)), (mean, (B,)), (rstd, (B,)), (gamma, (d,))):
        if t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != shape:
            raise ValueError(f"token_mean_ln_bwd: contiguous fp32 operands of shape {shape} expected, got {tuple(t.shape)}")
    dev = dy.device
    dgamma = torch.empty(d, dtype=torch.float32, device=dev)
    dbeta = torch.empty(d, dtype=torch.float32, device=dev)
    ws = torch.empty(B, d, dtype=torch.float32, device=dev)
    st = _lib.load().opb_token_mean_ln_bwd(dy.data_ptr(), m.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(), B, S, d,
                                           dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(), dx.data_ptr(), ld, _stream())
    _lib.check(st, "opb_token_mean_ln_bwd")
    _count(2)
    return dgamma, dbeta
