"""Multi-scale deformable attention of the segmentation recipe (one_peace_vision/seg/ops/modules/ms_deform_attn.py), the
operator under the ViT-Adapter's injectors and extractors and the Mask2Former pixel decoder.

``MSDeformAttn`` keeps the reference module's constructor, submodules (``sampling_offsets``, ``attention_weights``,
``value_proj``, ``output_proj``: names, shapes, registration order and initialisation), ``im2col_step`` and ``forward``
signature, and runs as one autograd node:

    input_flatten -> value_proj (GEMM, bf16 out)                                 value [N * S_in, H * 32]
    query -> [sampling_offsets | attention_weights] (one GEMM, fp32 out)        proj  [N * Lq, 3 * H * L * P]
    -> opb_ms_deform_attn_fwd (soft-max, locations, bilinear taps, weighted sum; csrc/ms_deform_attn.cu)
    -> output_proj (GEMM, fp32 out)

The backward is opb_ms_deform_attn_bwd between the adjoints of the three GEMMs.  Only what the recipes use is built: 32
channels per head, at most 4 levels and 8 points, reference points of the (x, y) form without a gradient, no padding mask.
Anything else raises ``NotImplementedError`` before a kernel runs.
"""
import math

import torch
import torch.nn as nn

from .. import kernels as K
from ..autograd import _dw, _dx, _pad8
from ..components import PackCache, bf16, f32

_HEAD_DIM = 32


def _host_ints(x):
    """A tensor (on any device: one host read) or a nested sequence of ints -> flat list of Python ints."""
    return [int(v) for v in torch.as_tensor(x).reshape(-1).tolist()]


def level_layout(input_spatial_shapes, input_level_start_index, n_levels, len_in):
    """Host copies of the level shapes [(H_l, W_l)] and start rows, checked as the reference module checks them:
    sum H_l W_l == Len_in, and the start rows are the running sums."""
    hw = _host_ints(input_spatial_shapes)
    if len(hw) != 2 * n_levels:
        raise ValueError(f"input_spatial_shapes must hold {n_levels} (H, W) pairs, got {len(hw) // 2}")
    shapes = [(hw[2 * i], hw[2 * i + 1]) for i in range(n_levels)]
    if any(h <= 0 or w <= 0 for h, w in shapes):
        raise ValueError(f"level shapes must be positive, got {shapes}")
    if sum(h * w for h, w in shapes) != len_in:
        raise ValueError(f"sum of H_l * W_l over the levels {shapes} is not Len_in = {len_in}")
    starts = _host_ints(input_level_start_index)
    want = [sum(h * w for h, w in shapes[:i]) for i in range(n_levels)]
    if starts != want:
        raise ValueError(f"input_level_start_index {starts} is not the running sum {want} of the level sizes")
    return shapes, starts


def msda_params(m):
    """The eight parameters in the order MSDeformAttnFn takes them."""
    return [m.sampling_offsets.weight, m.sampling_offsets.bias, m.attention_weights.weight, m.attention_weights.bias,
            m.value_proj.weight, m.value_proj.bias, m.output_proj.weight, m.output_proj.bias]


def msda_pack(m, cache):
    """bf16 GEMM weights and fp32 biases; the offset and logit projections as one weight whose rows are zero-padded to a
    multiple of 8 (the GEMM's N % 8 == 0)."""
    ps = msda_params(m)

    def build():
        sw, sb, aw, ab, vw, vb, ow, ob = ps
        n = sw.shape[0] + aw.shape[0]
        wp = torch.zeros(_pad8(n), sw.shape[1], dtype=torch.bfloat16, device=sw.device)
        wp[:n].copy_(torch.cat([sw.detach(), aw.detach()], 0))
        bp = torch.zeros(_pad8(n), dtype=torch.float32, device=sw.device)
        bp[:n].copy_(torch.cat([sb.detach(), ab.detach()], 0))
        return dict(wp=wp, bp=bp, n_proj=n, wv=bf16(vw), bv=f32(vb), wo=bf16(ow), bo=f32(ob))
    return cache.get(ps, build)


def msda_forward(pk, q, x, ref, shapes, starts, N, Lq, H, P, out, epi, **epilogue):
    """value_proj, the fused offset / logit projection, the core and output_proj: q bf16 [N * Lq, d], x bf16 [N * S_in, d]
    -> (value, proj, core).  output_proj writes `out` through epilogue `epi` with bias bo and the GEMM options `epilogue`
    (e.g. the in-place residual of the segmentation backbone's injectors and extractors)."""
    dev = q.device
    value = K.gemm(x, pk["wv"], K.EPI_STORE_BF16, torch.empty(x.shape[0], pk["wv"].shape[0], dtype=torch.bfloat16, device=dev),
                   bias=pk["bv"])
    proj = K.gemm(q, pk["wp"], K.EPI_STORE_F32, torch.empty(N * Lq, pk["wp"].shape[0], dtype=torch.float32, device=dev),
                  bias=pk["bp"])
    if proj.shape[1] != pk["n_proj"]:
        proj = proj[:, :pk["n_proj"]].contiguous()
    core = K.ms_deform_attn_fwd(value, proj, ref, shapes, starts, N, Lq, H, P)
    K.gemm(core, pk["wo"], epi, out, bias=pk["bo"], **epilogue)
    return value, proj, core


class MSDeformAttnFn(torch.autograd.Function):
    """(query [N, Lq, d], input_flatten [N, S_in, d]) -> output [N, Lq, d] in the query's dtype.  meta = (pack, reference
    points fp32 [N * Lq, L_ref, 2], level shapes, start rows, n_heads, n_points); then the eight msda_params."""

    @staticmethod
    def forward(ctx, meta, query, input_flatten, *params):
        pk, ref, shapes, starts, H, P = meta
        N, Lq, d = query.shape
        S_in = input_flatten.shape[1]
        dev = query.device
        q = query.reshape(N * Lq, d).to(torch.bfloat16).contiguous()
        x = input_flatten.reshape(N * S_in, d).to(torch.bfloat16).contiguous()
        y = torch.empty(N * Lq, d, dtype=torch.float32, device=dev)
        value, proj, core = msda_forward(pk, q, x, ref, shapes, starts, N, Lq, H, P, y, K.EPI_STORE_F32)
        ctx.meta = (pk, ref, shapes, starts, H, P, N, Lq, S_in, d)
        ctx.saved = (q, x, value, proj, core)
        ctx.dtypes = [p.dtype for p in params]
        ctx.in_dtypes = (query.dtype, input_flatten.dtype)
        return y.view(N, Lq, d).to(query.dtype)

    @staticmethod
    def backward(ctx, dy):
        pk, ref, shapes, starts, H, P, N, Lq, S_in, d = ctx.meta
        q, x, value, proj, core = ctx.saved
        dev = dy.device

        def g32(n):
            return torch.empty(n, dtype=torch.float32, device=dev)
        dyb = dy.reshape(N * Lq, d).to(torch.bfloat16).contiguous()
        gp = ctx.needs_input_grad[3:]
        dbo = K.colsum(dyb, g32(d)) if gp[7] else None
        dWo = _dw(dyb, core, torch.float32) if gp[6] else None
        dcore = _dx(dyb, pk["wo"], core.shape[1])
        d_value, d_proj = K.ms_deform_attn_bwd(value, proj, ref, dcore, shapes, starts, N, Lq, H, P)
        dvb = d_value.to(torch.bfloat16)
        dbv = K.colsum(dvb, g32(dvb.shape[1])) if gp[5] else None
        dWv = _dw(dvb, x, torch.float32) if gp[4] else None
        dx = _dx(dvb, pk["wv"], d, out=torch.empty(N * S_in, d, dtype=torch.float32, device=dev)) \
            if ctx.needs_input_grad[2] else None
        n, n_pad = pk["n_proj"], pk["wp"].shape[0]
        dpb = torch.zeros(N * Lq, n_pad, dtype=torch.bfloat16, device=dev)
        dpb[:, :n].copy_(d_proj)
        n_off = 2 * n // 3
        dbp = K.colsum(dpb, g32(n_pad))[:n] if gp[1] or gp[3] else None
        dWp = _dw(dpb, q, torch.float32)[:n] if gp[0] or gp[2] else None
        dq = _dx(dpb, pk["wp"], d, out=torch.empty(N * Lq, d, dtype=torch.float32, device=dev)) \
            if ctx.needs_input_grad[1] else None
        grads = [dWp[:n_off] if gp[0] else None, dbp[:n_off] if gp[1] else None,
                 dWp[n_off:] if gp[2] else None, dbp[n_off:] if gp[3] else None, dWv, dbv, dWo, dbo]
        out = [None if g is None else g.to(dt) for g, dt in zip(grads, ctx.dtypes)]
        ctx.saved = None
        dq = None if dq is None else dq.view(N, Lq, d).to(ctx.in_dtypes[0])
        dx = None if dx is None else dx.view(N, S_in, d).to(ctx.in_dtypes[1])
        return (None, dq, dx, *out)


class MSDeformAttn(nn.Module):
    """Multi-scale deformable attention (seg/ops/modules/ms_deform_attn.py) on the sm_90a kernels; see the module
    docstring for what is built."""

    def __init__(self, d_model=256, n_levels=4, n_heads=8, n_points=4, ratio=1.0):
        super().__init__()
        if d_model % n_heads != 0:
            raise ValueError(f"d_model must be divisible by n_heads, but got {d_model} and {n_heads}")
        self.im2col_step = 64
        self.d_model = d_model
        self.n_levels = n_levels
        self.n_heads = n_heads
        self.n_points = n_points
        self.ratio = ratio
        self.sampling_offsets = nn.Linear(d_model, n_heads * n_levels * n_points * 2)
        self.attention_weights = nn.Linear(d_model, n_heads * n_levels * n_points)
        self.value_proj = nn.Linear(d_model, int(d_model * ratio))
        self.output_proj = nn.Linear(int(d_model * ratio), d_model)
        self._reset_parameters()
        self._pack = PackCache()

    def _reset_parameters(self):
        """Zero offset weights with the head-direction grid as their bias: head h points along angle 2 pi h / n_heads,
        scaled so its larger coordinate is 1, times p + 1 for point p on every level.  Zero logits (uniform weights),
        Xavier value and output projections with zero biases."""
        H, L, P = self.n_heads, self.n_levels, self.n_points
        nn.init.constant_(self.sampling_offsets.weight.data, 0.0)
        theta = torch.arange(H, dtype=torch.float32) * (2.0 * math.pi / H)
        direction = torch.stack([theta.cos(), theta.sin()], -1)
        direction = direction / direction.abs().max(-1, keepdim=True)[0]
        scale = torch.arange(1, P + 1, dtype=torch.float32).view(1, 1, P, 1)
        grid = direction.view(H, 1, 1, 2).repeat(1, L, P, 1) * scale
        with torch.no_grad():
            self.sampling_offsets.bias = nn.Parameter(grid.view(-1))
        nn.init.constant_(self.attention_weights.weight.data, 0.0)
        nn.init.constant_(self.attention_weights.bias.data, 0.0)
        nn.init.xavier_uniform_(self.value_proj.weight.data)
        nn.init.constant_(self.value_proj.bias.data, 0.0)
        nn.init.xavier_uniform_(self.output_proj.weight.data)
        nn.init.constant_(self.output_proj.bias.data, 0.0)

    def _refuse(self, query, reference_points, input_flatten, input_padding_mask):
        if input_padding_mask is not None:
            raise NotImplementedError("MSDeformAttn: input_padding_mask is not supported (no recipe passes one)")
        if reference_points.shape[-1] == 4:
            raise NotImplementedError("MSDeformAttn: reference boxes (last dim 4) are not supported")
        if reference_points.shape[-1] != 2:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {reference_points.shape[-1]} instead.")
        dv = int(self.d_model * self.ratio)
        if dv % self.n_heads != 0 or dv // self.n_heads != _HEAD_DIM:
            raise NotImplementedError(f"MSDeformAttn: d_model * ratio / n_heads = {dv / self.n_heads:g}; only "
                                      f"{_HEAD_DIM} channels per head are built")
        if self.n_levels > 4 or self.n_points > 8:
            raise NotImplementedError(f"MSDeformAttn: n_levels = {self.n_levels}, n_points = {self.n_points}; at most 4 "
                                      f"levels and 8 points are built")
        if reference_points.requires_grad:
            raise NotImplementedError("MSDeformAttn: no gradient of the reference points is built")
        for name, t in (("query", query), ("reference_points", reference_points), ("input_flatten", input_flatten)):
            if t.dtype not in (torch.float32, torch.bfloat16):
                raise NotImplementedError(f"MSDeformAttn: {name} dtype {t.dtype}; only float32 and bfloat16 are built")

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None):
        """query [N, Lq, d_model], reference_points [N, Lq, n_levels or 1, 2] in [0, 1] (x, y), input_flatten
        [N, sum H_l W_l, d_model], input_spatial_shapes [(H_l, W_l)] and input_level_start_index (tensors or sequences)
        -> [N, Lq, d_model] in the query's dtype."""
        self._refuse(query, reference_points, input_flatten, input_padding_mask)
        N, Lq, _ = query.shape
        _, len_in, _ = input_flatten.shape
        shapes, starts = level_layout(input_spatial_shapes, input_level_start_index, self.n_levels, len_in)
        if reference_points.dim() != 4 or tuple(reference_points.shape[:2]) != (N, Lq) \
                or reference_points.shape[2] not in (1, self.n_levels):
            raise ValueError(f"reference_points must be [N, Lq, 1 or n_levels, 2], got {tuple(reference_points.shape)}")
        ref = reference_points.detach().reshape(N * Lq, reference_points.shape[2], 2).to(torch.float32).contiguous()
        pk = msda_pack(self, self._pack)
        meta = (pk, ref, shapes, starts, self.n_heads, self.n_points)
        return MSDeformAttnFn.apply(meta, query, input_flatten, *msda_params(self))
