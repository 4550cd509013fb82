"""fp64 reference of the multi-scale deformable attention core (csrc/ms_deform_attn.cu) as direct bilinear sums over the
four taps of each sample, not grid_sample, and per-element error bounds derived from the kernel's arithmetic.

Layouts as opb_ms_deform_attn_fwd: value [N * S_in, H * 32], proj [N * Lq, 3 * H * L * P] = [offsets (h, l, p, xy) |
logits (h, l * P + p)], ref [N * Lq, L_ref, 2].  Everything is computed in fp64 from the operands the kernel reads (the
bf16 value and d_out already rounded, fp32 proj and ref).

Bounds (u = 2^-24, fp32 unit roundoff), each the sum of
  - location: px = (ref + off / W) * W - 0.5 takes 4 fp32 roundings, |d px| <= 4u (W |ref| + |off| + |px| + 1), and moves
    the sample by at most |d px| * |v_right - v_left| per channel (the same for y with the vertical tap differences).
    Contract cases keep every sample >= 1e-3 pixel from a cell crossing, so the taps are the kernel's;
  - soft-max: exp, the (z - max) subtraction, the L * P-term sum and the division give |d a| <= a u (|z - max| + L P + 4);
  - accumulation: each output channel is a sum of L * P * 4 products (bilinear weights times taps, times a), accumulated in
    fp32 sequentially per lane group and by a shuffle tree: <= (L P + 8) u times the sum of the absolute terms.  d_value
    is scattered with fp32 atomics in any order: (count + 4) u times the sum of its absolute terms, count the number of
    contributions to the element;
  - bf16 output rounding: 2^-8 |out| (assert_within's u_out).
"""
import torch

U32 = 2.0 ** -24
HD = 32


def _split(proj, N, Lq, H, L, P):
    p = proj.double().view(N, Lq, 3 * H * L * P)
    off = p[..., :2 * H * L * P].reshape(N, Lq, H, L, P, 2)
    logit = p[..., 2 * H * L * P:].reshape(N, Lq, H, L * P)
    return off, logit


def _softmax(logit, L, P, mistake):
    N, Lq, H, _ = logit.shape
    if mistake == "softmax_per_level":
        return torch.softmax(logit.view(N, Lq, H, L, P), -1).view(N, Lq, H, L * P)
    return torch.softmax(logit, -1)


def geometry(proj, ref, shapes, N, Lq, H, P, mistake=None, left=False):
    """Soft-max weights a [N, Lq, H, L, P] and pixel coordinates px, py [N, Lq, H, L, P] (align_corners = False), with the
    inputs of the bounds: logits z and their row max, offsets."""
    L = len(shapes)
    off, logit = _split(proj, N, Lq, H, L, P)
    a = _softmax(logit, L, P, mistake).view(N, Lq, H, L, P)
    r = ref.double().view(N, Lq, -1, 2)
    r = r.expand(N, Lq, L, 2) if r.shape[2] == 1 else r
    Hs = torch.tensor([h for h, _ in shapes], dtype=torch.float64, device=proj.device).view(1, 1, 1, L, 1)
    Ws = torch.tensor([w for _, w in shapes], dtype=torch.float64, device=proj.device).view(1, 1, 1, L, 1)
    nx, ny = (Hs, Ws) if mistake == "swap_norm" else (Ws, Hs)
    locx = r[:, :, None, :, None, 0] + off[..., 0] / nx
    locy = r[:, :, None, :, None, 1] + off[..., 1] / ny
    if mistake == "align_corners":
        px, py = locx * (Ws - 1), locy * (Hs - 1)
    else:
        px, py = locx * Ws - 0.5, locy * Hs - 0.5
    return dict(a=a, px=px, py=py, off=off, z=logit.view(N, Lq, H, L, P), zmax=logit.max(-1).values, r=r, Ws=Ws, Hs=Hs)


def _taps(geo, shapes, starts, S_in, mistake, left):
    """For each of the 4 taps (y0 x0, y0 x1, y1 x0, y1 x1): flat value row index [N, Lq, H, L, P], weight, validity."""
    L = len(shapes)
    px, py = geo["px"], geo["py"]
    if left:
        x0, y0 = torch.ceil(px) - 1, torch.ceil(py) - 1
    else:
        x0, y0 = torch.floor(px), torch.floor(py)
    lx, ly = px - x0, py - y0
    Ws, Hs = geo["Ws"], geo["Hs"]
    st = list(starts)
    if mistake == "start_off_by_one":
        st = [st[(l - 1) % L] for l in range(L)]
    St = torch.tensor(st, dtype=torch.float64, device=px.device).view(1, 1, 1, L, 1)
    out = []
    for dy in (0, 1):
        for dx in (0, 1):
            xi, yi = x0 + dx, y0 + dy
            w = (ly if dy else 1 - ly) * (lx if dx else 1 - lx)
            valid = (xi >= 0) & (xi <= Ws - 1) & (yi >= 0) & (yi <= Hs - 1)
            if mistake == "clamp":
                xi, yi = xi.clamp(min=0), yi.clamp(min=0)
                xi, yi = torch.minimum(xi, Ws - 1), torch.minimum(yi, Hs - 1)
                valid = torch.ones_like(valid)
            row = (St + yi * Ws + xi).clamp(0, S_in - 1).long() % S_in
            out.append((row, w, valid, dx, dy))
    return out, lx, ly


def _gather(value, rows, N, S_in, H):
    """value [N * S_in, H * 32] -> the rows' head slices [N, Lq, H, L, P, 32]."""
    v = value.double().view(N, S_in, H, HD)
    n_idx = torch.arange(N, device=rows.device).view(N, 1, 1, 1, 1).expand_as(rows)
    h_idx = torch.arange(H, device=rows.device).view(1, 1, H, 1, 1).expand_as(rows)
    return v[n_idx, rows, h_idx]


def forward(value, proj, ref, shapes, starts, N, Lq, H, P, mistake=None, left=False, with_bound=False):
    """-> out fp64 [N * Lq, H * 32] (and its error bound without the output rounding when with_bound)."""
    S_in = value.shape[0] // N
    geo = geometry(proj, ref, shapes, N, Lq, H, P, mistake)
    taps, lx, ly = _taps(geo, shapes, starts, S_in, mistake, left)
    vals = [_gather(value, row, N, S_in, H) * valid[..., None] for row, _, valid, _, _ in taps]
    s = sum(w[..., None] * v for (_, w, _, _, _), v in zip(taps, vals))
    a = geo["a"]
    out = (a[..., None] * s).sum((3, 4)).reshape(N * Lq, H * HD)
    if not with_bound:
        return out
    return out, _fwd_bound(geo, taps, vals, s, lx, ly, N, Lq, H, P, len(shapes))


def _loc_err(geo):
    ex = 4 * U32 * (geo["Ws"] * geo["r"][:, :, None, :, None, 0].abs() + geo["off"][..., 0].abs() + geo["px"].abs() + 1)
    ey = 4 * U32 * (geo["Hs"] * geo["r"][:, :, None, :, None, 1].abs() + geo["off"][..., 1].abs() + geo["py"].abs() + 1)
    return ex, ey


def _softmax_err(geo, L, P):
    return geo["a"] * U32 * ((geo["z"] - geo["zmax"][..., None, None]).abs() + L * P + 4)


def _diffs(vals):
    gx = torch.maximum((vals[1] - vals[0]).abs(), (vals[3] - vals[2]).abs())
    gy = torch.maximum((vals[2] - vals[0]).abs(), (vals[3] - vals[1]).abs())
    return gx, gy


def _fwd_bound(geo, taps, vals, s, lx, ly, N, Lq, H, P, L):
    a = geo["a"][..., None]
    ex, ey = _loc_err(geo)
    gx, gy = _diffs(vals)
    da = _softmax_err(geo, L, P)[..., None]
    absterm = sum(w[..., None] * v.abs() for (_, w, _, _, _), v in zip(taps, vals))
    e = a * (ex[..., None] * gx + ey[..., None] * gy) + da * s.abs() + (L * P + 8) * U32 * a * absterm
    return e.sum((3, 4)).reshape(N * Lq, H * HD)


def backward(value, proj, ref, d_out, shapes, starts, N, Lq, H, P, left=False, with_bound=False, acc=None):
    """-> (d_value fp64 [N * S_in, H * 32], d_proj fp64 [N * Lq, 3 * H * L * P]) and, when with_bound, their bounds.
    acc: a dict shared by calls over consecutive query-row chunks of one N = 1 problem; d_value and its bound are then
    those of all the chunks so far (the bound's contribution count included)."""
    S_in = value.shape[0] // N
    L = len(shapes)
    geo = geometry(proj, ref, shapes, N, Lq, H, P)
    taps, lx, ly = _taps(geo, shapes, starts, S_in, None, left)
    vals = [_gather(value, row, N, S_in, H) * valid[..., None] for row, _, valid, _, _ in taps]
    s = sum(w[..., None] * v for (_, w, _, _, _), v in zip(taps, vals))
    a = geo["a"]
    g = d_out.double().view(N, Lq, H, 1, 1, HD)
    dA = (g * s).sum(-1)
    # d sample / d px and / d py inside the cell
    sx = (1 - ly)[..., None] * (vals[1] - vals[0]) + ly[..., None] * (vals[3] - vals[2])
    sy = (1 - lx)[..., None] * (vals[2] - vals[0]) + lx[..., None] * (vals[3] - vals[1])
    gX, gY = (g * sx).sum(-1), (g * sy).sum(-1)
    sad = (a * dA).sum((3, 4), keepdim=True)
    dlogit = a * (dA - sad)
    d_off = torch.stack([a * gX, a * gY], -1)
    d_proj = torch.cat([d_off.reshape(N, Lq, -1), dlogit.reshape(N, Lq, -1)], -1).reshape(N * Lq, 3 * H * L * P)
    dev = value.device
    if acc is None:
        acc = {}
    if not acc:
        z = dict(dtype=torch.float64, device=dev)
        acc.update(dv=torch.zeros(N, S_in, H, HD, **z), cnt=torch.zeros(N, S_in, H, **z), ev=torch.zeros(N, S_in, H, HD, **z),
                   absdv=torch.zeros(N, S_in, H, HD, **z))
    dv, cnt = acc["dv"], acc["cnt"]
    n_idx = torch.arange(N, device=dev).view(N, 1, 1, 1, 1).expand_as(a)
    h_idx = torch.arange(H, device=dev).view(1, 1, H, 1, 1).expand_as(a)
    for row, w, valid, _, _ in taps:
        c = (a * w * valid)[..., None] * g
        dv.index_put_((n_idx.reshape(-1), row.reshape(-1), h_idx.reshape(-1)), c.reshape(-1, HD), accumulate=True)
        cnt.index_put_((n_idx.reshape(-1), row.reshape(-1), h_idx.reshape(-1)), valid.double().reshape(-1), accumulate=True)
    d_value = dv.reshape(N * S_in, H * HD)
    if not with_bound:
        return d_value, d_proj
    # ---- bounds ----
    ex, ey = _loc_err(geo)
    da = _softmax_err(geo, L, P)
    ga = g.abs()
    gx, gy = _diffs(vals)
    absv = sum(w[..., None] * v.abs() for (_, w, _, _, _), v in zip(taps, vals))
    absx = (1 - ly)[..., None] * (vals[1].abs() + vals[0].abs()) + ly[..., None] * (vals[3].abs() + vals[2].abs())
    absy = (1 - lx)[..., None] * (vals[2].abs() + vals[0].abs()) + lx[..., None] * (vals[3].abs() + vals[1].abs())
    # gX moves with py (and gY with px) inside a cell; per-channel sums of 32 terms in fp32
    e_gX = (ga * (ey[..., None] * 2 * gx)).sum(-1) + 48 * U32 * (ga * absx).sum(-1)
    e_gY = (ga * (ex[..., None] * 2 * gy)).sum(-1) + 48 * U32 * (ga * absy).sum(-1)
    b_off = torch.stack([a * e_gX + da * gX.abs() + 4 * U32 * (a * gX).abs(),
                         a * e_gY + da * gY.abs() + 4 * U32 * (a * gY).abs()], -1)
    e_dA = (ga * (ex[..., None] * gx + ey[..., None] * gy)).sum(-1) + (48 + 8) * U32 * (ga * absv).sum(-1)
    e_sad = (da * dA.abs() + a * e_dA).sum((3, 4), keepdim=True) + (L * P + 2) * U32 * (a * dA.abs()).sum((3, 4), keepdim=True)
    b_logit = da * (dA - sad).abs() + a * (e_dA + e_sad) + 3 * U32 * a * (dA.abs() + sad.abs())
    b_proj = torch.cat([b_off.reshape(N, Lq, -1), b_logit.reshape(N, Lq, -1)], -1).reshape(N * Lq, 3 * H * L * P)
    bv, absdv = acc["ev"], acc["absdv"]
    for row, w, valid, _, _ in taps:
        idx = (n_idx.reshape(-1), row.reshape(-1), h_idx.reshape(-1))
        e = ((da * w + a * (ex + ey + 4 * U32)) * valid)[..., None] * ga
        bv.index_put_(idx, e.reshape(-1, HD), accumulate=True)
        absdv.index_put_(idx, ((a * w * valid)[..., None] * ga).reshape(-1, HD), accumulate=True)
    bv = bv + (cnt[..., None] + 4) * U32 * absdv
    return d_value, d_proj, bv.reshape(N * S_in, H * HD), b_proj


def contract_case(N, Lq, H, shapes, P, L_ref, off_scale, seed, device="cpu"):
    """Seeded kernel operands (value bf16, proj / ref fp32, d_out bf16) with every sample >= 1e-3 pixel from a cell crossing
    (and from the -1 / W edges of the inside test): offsets that land closer are moved by 5e-3 pixel."""
    g = torch.Generator().manual_seed(seed)
    L = len(shapes)
    S_in = sum(h * w for h, w in shapes)
    starts = [sum(h * w for h, w in shapes[:i]) for i in range(L)]
    value = torch.randn(N * S_in, H * HD, generator=g).to(torch.bfloat16)
    ref = (torch.rand(N * Lq, L_ref, 2, generator=g) * 0.9 + 0.05).float()
    off = (torch.randn(N * Lq, H, L, P, 2, generator=g) * off_scale).float()
    logit = (torch.randn(N * Lq, H, L * P, generator=g) * 2).float()
    for _ in range(4):
        proj = torch.cat([off.reshape(N * Lq, -1), logit.reshape(N * Lq, -1)], 1).contiguous()
        geo = geometry(proj, ref, shapes, N, Lq, H, P)
        fx = geo["px"] - torch.floor(geo["px"])
        fy = geo["py"] - torch.floor(geo["py"])
        near_x = (torch.minimum(fx, 1 - fx) < 1e-3).reshape(N * Lq, H, L, P)
        near_y = (torch.minimum(fy, 1 - fy) < 1e-3).reshape(N * Lq, H, L, P)
        if not (near_x.any() or near_y.any()):
            break
        off[..., 0] += 5e-3 * near_x
        off[..., 1] += 5e-3 * near_y
    proj = torch.cat([off.reshape(N * Lq, -1), logit.reshape(N * Lq, -1)], 1).contiguous()
    d_out = torch.randn(N * Lq, H * HD, generator=g).to(torch.bfloat16)
    return dict(value=value.to(device), proj=proj.to(device), ref=ref.to(device), d_out=d_out.to(device), shapes=shapes,
                starts=starts, N=N, Lq=Lq, H=H, P=P)
