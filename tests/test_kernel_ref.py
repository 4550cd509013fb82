"""CPU: the fp64 reference and per-element bounds of tests/kernel_ref.py.  A correct kernel, emulated here in fp32 (bf16
operands, fp32 matmul, the epilogue and the LayerNorm statistics in fp32 as the kernel evaluates them; for attention the
blocked online soft-max and the recomputing backward), must pass the bounds; each of the subtle mistakes a GEMM, InfoNCE
or attention kernel can make must fail them.  The exact kernels (top-10 ranking, transpose, row gather, block bias) are
ported or emulated and must equal their references bit for bit, and their planted mistakes must not."""
import struct

import numpy as np
import pytest
import torch

import kernel_ref as R

M, K_DIM, N, PARTS = 256, 1000, 512, 8      # two 128-row panels, two 256-column tiles, 16 k-blocks (the last one partial)


def _records(x, parts):
    """[parts, M, 2] (sum, sum of squares) records of equal column slices of x (as the producing kernel writes them)"""
    s = x.view(x.shape[0], parts, -1)
    return torch.stack([s.sum(2), (s * s).sum(2)], 2).transpose(0, 1).contiguous()


@pytest.fixture(scope="module")
def data():
    g = torch.Generator().manual_seed(5)
    # rows differ in scale and offset by a few percent only, so a row given its neighbour's statistics is off by about as
    # much as a slightly wrong rstd
    x = torch.randn(M, K_DIM, generator=g) * (1 + 0.01 * torch.randn(M, 1, generator=g)) + 0.01 * torch.randn(M, 1, generator=g)
    w = (torch.randn(N, K_DIM, generator=g) * 0.05).bfloat16()
    return dict(
        x=x, a=x.bfloat16(), rec=_records(x, PARTS), w=w,
        colsum=w.float().sum(1), bias=0.02 * torch.randn(N, generator=g),
        colscale=torch.rand(N, generator=g) + 0.5, gamma=torch.randn(N, generator=g), resid=torch.randn(M, N, generator=g))


def emulate(d, epi, mutation=None, k_used=K_DIM, parts_used=PARTS):
    """what a correct kernel computes, in fp32, with an optional mistake"""
    acc = d["a"][:, :k_used].float() @ d["w"][:, :k_used].float().t()
    rec = d["rec"]
    s1 = torch.zeros(M)
    s2 = torch.zeros(M)
    for p in range(parts_used):               # record order, fp32
        s1 = s1 + rec[p, :, 0]
        s2 = s2 + rec[p, :, 1]
    mu = s1 / K_DIM
    rstd = torch.rsqrt((s2 / K_DIM - mu * mu).clamp_min(0) + 1e-5)
    colsum, bias = d["colsum"].clone(), d["bias"].clone()
    if mutation == "row_plus_8":              # fragment row r + 8's statistics used for row r, in the second 128-row tile
        r = torch.arange(128, 256)
        src = torch.where(r % 16 < 8, r + 8, r)
        mu[r], rstd[r] = mu[src].clone(), rstd[src].clone()
    if mutation == "col_shift_8":             # the second 256-column tile reads its colsum / bias slices 8 columns late
        colsum[256:512] = torch.roll(d["colsum"][256:512], -8)
        bias[256:512] = torch.roll(d["bias"][256:512], -8)
    x = rstd[:, None] * (acc - mu[:, None] * colsum) + bias
    if epi == R.EPI_STORE_F32:
        return x
    if epi == R.EPI_STORE_BF16:
        return (x * d["colscale"]).bfloat16()
    if epi == R.EPI_GELU_BF16:
        return torch.nn.functional.gelu(x * d["colscale"]).bfloat16()
    if epi == R.EPI_RESID_F32:
        y = d["resid"] + d["gamma"] * x
        t = y.view(M, N // 256, 256)
        return y, torch.stack([t.sum(2), (t * t).sum(2)], 2).transpose(0, 1)
    if epi == R.EPI_GEGLU_BF16:
        z = x.view(M, N // 256, 2, 128)
        u = (torch.nn.functional.gelu(z[:, :, 0]) * z[:, :, 1]).reshape(M, N // 2)
        t = u.view(M, N // 256, 128)
        st = torch.stack([t.sum(2), (t * t).sum(2)], 2).transpose(0, 1)
        return u.bfloat16(), torch.stack([st, torch.zeros_like(st)], 1).reshape(N // 128, M, 2)
    raise ValueError(epi)


def reference(d, epi, **kw):
    extra = dict(colscale=d["colscale"]) if epi in (R.EPI_STORE_BF16, R.EPI_GELU_BF16) else {}
    if epi == R.EPI_RESID_F32:
        extra = dict(gamma=d["gamma"], resid=d["resid"], stats=True)
    if epi == R.EPI_GEGLU_BF16:
        extra = dict(stats=True)
    return R.gemm_ref(d["a"], d["w"], epi, ln_colsum=d["colsum"], bias=d["bias"], ln_partial=(d["rec"], PARTS, K_DIM, 1e-5),
                      **extra, **kw)


@pytest.mark.parametrize("epi,dt", [(R.EPI_STORE_F32, torch.float32), (R.EPI_STORE_BF16, torch.bfloat16),
                                    (R.EPI_GELU_BF16, torch.bfloat16), (R.EPI_RESID_F32, torch.float32),
                                    (R.EPI_GEGLU_BF16, torch.bfloat16)])
def test_correct_emulation_passes(data, epi, dt):
    ref = reference(data, epi)
    got = emulate(data, epi)
    if isinstance(got, tuple):
        got, st = got
        R.assert_within(st, ref.stats, ref.stats_mag, R.TAU, torch.float32, extra=ref.stats_extra, what="stats")
    R.assert_within(got, ref.y, ref.mag, R.TAU, dt, extra=ref.extra)


@pytest.mark.parametrize("mutation", ["row_plus_8", "col_shift_8", "last_k_block", "parts_minus_1"])
def test_mutated_gemm_fails(data, mutation):
    kw = {}
    if mutation == "last_k_block":
        kw["k_used"] = K_DIM // 64 * 64           # the partial 16th k-block (40 columns) dropped
    if mutation == "parts_minus_1":
        kw["parts_used"] = PARTS - 1
    ref = reference(data, R.EPI_STORE_F32)
    got = emulate(data, R.EPI_STORE_F32, mutation if not kw else None, **kw)
    with pytest.raises(AssertionError, match="outside the bound"):
        R.assert_within(got, ref.y, ref.mag, R.TAU, torch.float32, extra=ref.extra)


def test_mutated_row_stats_fail_after_bf16_rounding(data):
    """the wrong-fragment-row mistake is still caught behind a bf16 output's rounding"""
    ref = reference(data, R.EPI_STORE_BF16)
    with pytest.raises(AssertionError, match="outside the bound"):
        R.assert_within(emulate(data, R.EPI_STORE_BF16, "row_plus_8"), ref.y, ref.mag, R.TAU, torch.bfloat16, extra=ref.extra)


def _split(x):
    hi = x.bfloat16()
    return hi, (x - hi.float()).bfloat16()


def emulate_infonce_loss(xa, xb, scale, target_offset, eps, eps_den):
    """fp32 InfoNCE row losses from the bf16x3 split operands, label smoothing eps_i = eps / eps_den"""
    (ah, al), (bh, bl) = _split(xa), _split(xb)
    z = scale * (ah.float() @ bh.float().t() + ah.float() @ bl.float().t() + al.float() @ bh.float().t())
    lse = torch.logsumexp(z, 1)
    n = xb.shape[0]
    eps_i = eps / eps_den
    rows = torch.arange(xa.shape[0])
    zt = z[rows, rows + target_offset]
    return (1 - eps - eps_i) * (lse - zt) + eps_i * (n * lse - z.sum(1)), lse


def test_infonce_label_smoothing_denominator():
    """eps_i = eps / (n - 1) passes the loss bound, eps / n fails it"""
    g = torch.Generator().manual_seed(9)
    b, n, d, off, eps, scale = 64, 300, 256, 128, 0.1, 5.0
    xb = torch.nn.functional.normalize(torch.randn(n, d, generator=g), dim=1)
    xa = torch.nn.functional.normalize(xb[off:off + b] + 0.5 * torch.randn(b, d, generator=g), dim=1)
    ref = R.infonce_ref(xa, xb, scale, off, eps)
    loss, lse = emulate_infonce_loss(xa, xb, scale, off, eps, n - 1)
    R.assert_within(lse, ref.lse, ref.dlse, 1.0, torch.float32, what="lse")
    R.assert_within(loss, ref.loss, ref.dloss, 1.0, torch.float32, what="loss")
    bad, _ = emulate_infonce_loss(xa, xb, scale, off, eps, n)
    with pytest.raises(AssertionError, match="outside the bound"):
        R.assert_within(bad, ref.loss, ref.dloss, 1.0, torch.float32, what="loss")


def test_canary_helpers():
    out, buf = R.canary_out((5, 16), ldo_extra=8, rows_before=2, rows_after=3, dtype=torch.bfloat16, device="cpu")
    assert out.stride(0) == 24 and out.shape == (5, 16)
    out.fill_(1.0)
    R.assert_canary(buf, out)
    buf[1, 0] = 0.0                            # a write one row before the view
    with pytest.raises(AssertionError, match="outside the logical output"):
        R.assert_canary(buf, out)
    buf[1, 0] = float("nan")
    out[1, 16 - 1] = 2.0
    buf[3, 16] = 0.0                           # a write into the pitch padding of row 1
    with pytest.raises(AssertionError, match="outside the logical output"):
        R.assert_canary(buf, out)
    buf[3, 16] = float("nan")
    written = torch.ones(5, 16, dtype=torch.bool)
    written[3] = False                         # a skipped row must stay NaN ...
    with pytest.raises(AssertionError, match="outside the logical output"):
        R.assert_canary(buf, out, written=written)
    out[3] = float("nan")
    R.assert_canary(buf, out, written=written)
    out32, buf32 = R.canary_out((4, 8), ldo_extra=8, dtype=torch.float32, device="cpu")
    out32[:3] = 0.0                            # ... and a row that should have been written must not
    with pytest.raises(AssertionError, match="not finite"):
        R.assert_canary(buf32, out32)


# ----------------------------------------------------------------------------------------------------------------------
# convolutions lowered onto the GEMM
# ----------------------------------------------------------------------------------------------------------------------
CG, CPAD, CN, CTAPS, CGROUPS, CROWS = 96, 128, 96, 19, 3, 150     # the audio positional conv's group geometry (two 64-channel
                                                                    # k-blocks per tap), three groups
OV_C, OV_KW, OV_M = 64, 3, 100                                      # overlapping rows: K = 3 C read at a pitch of 2 C


@pytest.fixture(scope="module")
def conv():
    g = torch.Generator().manual_seed(13)
    x = torch.zeros(CROWS + CTAPS - 1, CGROUPS, CPAD)
    x[:, :, :CG] = torch.randn(CROWS + CTAPS - 1, CGROUPS, CG, generator=g)
    w = torch.zeros(CGROUPS * CN, CTAPS, CPAD)
    w[:, :, :CG] = torch.randn(CGROUPS * CN, CTAPS, CG, generator=g) * 0.05
    K = OV_KW * OV_C
    return dict(x=x.bfloat16(), w=w.view(CGROUPS * CN, CTAPS * CPAD).bfloat16(), bias=torch.randn(CGROUPS * CN, generator=g),
                flat=torch.randn(OV_M * K, generator=g).bfloat16(), w_ov=(torch.randn(128, K, generator=g) * 0.05).bfloat16())


def emulate_grouped_conv(c, mutation=None):
    """fp32 grouped sliding-window conv as a correct kernel computes it, with an optional mistake.  Rows past the operand, a
    group past the last and weight rows past groups * n read as zero (the tensor maps zero-fill them)."""
    X = c["x"].float()
    X = torch.cat([X, torch.zeros(2, CGROUPS, CPAD)], 0)
    X = torch.cat([X, torch.zeros(X.shape[0], 1, CPAD)], 1)
    W = torch.cat([c["w"].float(), torch.zeros(CGROUPS * 256, CTAPS * CPAD)], 0)
    bias = torch.cat([c["bias"], torch.zeros(CN)])
    r, j = torch.arange(CROWS)[:, None], torch.arange(CTAPS)[None, :]
    src = r + j
    if mutation == "tap_shift":                   # window one tap late
        src = r + j + 1
    if mutation == "taps_reversed":
        src = r + (CTAPS - 1 - j)
    out = []
    for g in range(CGROUPS):
        A = X[src, g + 1 if mutation == "group_c0" else g]          # [rows, taps, c_pad]; group_c0: the next group's channels
        if mutation == "kin_swapped":             # the two 64-channel k-blocks of every tap exchanged
            A = A.view(CROWS, CTAPS, CPAD // 64, 64).flip(2)
        A = A.reshape(CROWS, CTAPS * CPAD)
        w0 = g * 256 if mutation == "b_group_rows" else g * CN      # b_group_rows: a whole 256-row tile per group
        b0 = (g + 1) * CN if mutation == "bias_neighbour" else g * CN
        out.append(A @ W[w0:w0 + CN].t() + bias[b0:b0 + CN])
    return torch.cat(out, 1)


def conv_ref(c, epi=R.EPI_STORE_F32):
    return R.grouped_window_ref(c["x"], c["w"], CROWS, CGROUPS, CPAD, CTAPS, CN, epi, bias=c["bias"])


def overlap_ref(c):
    K = OV_KW * OV_C
    return R.gemm_ref(c["flat"].as_strided((OV_M, K), (2 * OV_C, 1)), c["w_ov"], R.EPI_STORE_F32)


def emulate_overlap(c, mutation=None):
    K = OV_KW * OV_C
    pitch = K if mutation == "pitch_K" else 2 * OV_C
    return c["flat"].float().as_strided((OV_M, K), (pitch, 1)) @ c["w_ov"].float().t()


def test_window_matrix_is_conv1d():
    """the references are Conv1d: grouped, k = 19, padding 9 on a halo'd buffer, and k = 3, stride 2 on overlapping rows"""
    g = torch.Generator().manual_seed(17)
    B, T, G, cg, cpad, kp = 2, 30, 3, 8, 64, 19
    halo = kp // 2
    x, w, b = torch.randn(B, T, G * cg, generator=g), torch.randn(G * cg, cg, kp, generator=g), torch.randn(G * cg, generator=g)
    buf = torch.zeros(B, T + 2 * halo, G, cpad, dtype=torch.float64)
    buf[:, halo:halo + T, :, :cg] = x.double().view(B, T, G, cg)
    wp = torch.zeros(G * cg, kp, cpad, dtype=torch.float64)
    wp[:, :, :cg] = w.double().permute(0, 2, 1)
    rows = B * (T + 2 * halo)
    buf = torch.cat([buf.view(rows, G, cpad), torch.zeros(kp - 1, G, cpad, dtype=torch.float64)])
    got = R.grouped_window_ref(buf, wp.view(G * cg, kp * cpad), rows, G, cpad, kp, cg, R.EPI_STORE_F32, bias=b).y
    want = torch.nn.functional.conv1d(x.double().transpose(1, 2), w.double(), b.double(), padding=halo, groups=G)
    torch.testing.assert_close(got.view(B, T + 2 * halo, G * cg)[:, :T], want.transpose(1, 2), rtol=1e-12, atol=1e-12)
    C, T_in = 16, 41
    T_out = (T_in - 3) // 2 + 1
    xs, ws = torch.randn(T_in, C, generator=g, dtype=torch.float64), torch.randn(32, C, 3, generator=g, dtype=torch.float64)
    got = R.gemm_ref(xs.view(-1).as_strided((T_out, 3 * C), (2 * C, 1)), ws.permute(0, 2, 1).reshape(32, 3 * C),
                     R.EPI_STORE_F32).y
    want = torch.nn.functional.conv1d(xs.t()[None], ws, stride=2)[0].t()
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("epi,dt", [(R.EPI_STORE_F32, torch.float32), (R.EPI_STORE_BF16, torch.bfloat16)])
def test_conv_emulation_passes(conv, epi, dt):
    ref = conv_ref(conv, epi)
    got = emulate_grouped_conv(conv)
    r = R.assert_within(got.to(dt), ref.y, ref.mag, R.TAU, dt, extra=ref.extra)
    print(f"grouped window {dt}: {r:.3g} of the bound")
    ov = overlap_ref(conv)
    r = R.assert_within(emulate_overlap(conv), ov.y, ov.mag, R.TAU, torch.float32, extra=ov.extra)
    print(f"overlapping rows: {r:.3g} of the bound")


CONV_MUTATIONS = ["tap_shift", "taps_reversed", "kin_swapped", "group_c0", "b_group_rows", "bias_neighbour", "pitch_K"]


@pytest.mark.parametrize("mutation", CONV_MUTATIONS)
def test_mutated_conv_fails(conv, mutation):
    """each mistake of the grouped sliding window or the overlapping view lands outside the fp32 bound (run with -s to
    see by how much)"""
    if mutation == "pitch_K":
        ref, got = overlap_ref(conv), emulate_overlap(conv, mutation)
    else:
        ref, got = conv_ref(conv), emulate_grouped_conv(conv, mutation)
    print(f"{mutation}: {_ratio(got, ref.y, R.TAU * ref.mag + ref.extra, torch.float32):.3g} x the bound")
    with pytest.raises(AssertionError, match="outside the bound"):
        R.assert_within(got, ref.y, ref.mag, R.TAU, torch.float32, extra=ref.extra)


# ----------------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------------
AB, AS, AH = 2, 197, 2              # S = 197: three full 64-key blocks and a partial one of 5 keys
PAD_FROM = (195, 127)               # first padded key per sample: odd, so a pair (even live key, odd padded key) straddles
                                    # each edge; sample 0 keeps three live keys in the last block, sample 1's padding
                                    # covers the whole third 64-key block and the fourth
SPLIT = 60                          # two-segment LUT: segments [0, 60) and [60, 197)
Q_SCALE = 0.125
LOG2E, LN2 = 1.4426950408889634, 0.69314718055994531


@pytest.fixture(scope="module")
def att():
    g = torch.Generator().manual_seed(11)
    B, S, H = AB, AS, AH
    kp = torch.zeros(B, S, dtype=torch.uint8)
    for b, p in enumerate(PAD_FROM):
        kp[b, p:] = 1
    s1, s2 = SPLIT, S - SPLIT
    return dict(
        qkv=(torch.randn(B * S, 3 * H * 64, generator=g) * 0.3).bfloat16(), kp=kp,
        bias=torch.randn(H, S, S, generator=g), bias_ps=torch.randn(B, H, S, S, generator=g),
        d_out=(torch.randn(B * S, H * 64, generator=g) * 0.5).bfloat16(), dbias0=0.01 * torch.randn(H, S, S, generator=g),
        # two-segment LUT form: per segment a Toeplitz LUT (code difference i - j), the second segment's row codes shifted
        # past the first segment's LUT
        lut=torch.randn(H, (2 * s1 - 1) + (2 * s2 - 1), generator=g),
        code_row=torch.cat([torch.arange(s1) + s1 - 1, torch.arange(s2) + s2 - 1 + 2 * s1 - 1]),
        code_col=torch.cat([torch.arange(s1), torch.arange(s2)]))


def lut_dense(d, mutation=None):
    """the (H,S,S) bias the two-segment LUT form encodes, as the kernel gathers it"""
    S = AS
    col = d["code_col"].clone()
    if mutation == "seg_code_col_off_by_one":       # the first key of the second segment reads the previous key's code
        col[SPLIT] = col[SPLIT - 1]
    i, j = torch.arange(S)[:, None], torch.arange(S)[None, :]
    t = d["lut"][:, (d["code_row"][i] - col[j]).clamp(0, d["lut"].shape[1] - 1)]
    if mutation == "seg_cross_not_zeroed":
        return t
    return torch.where((i < SPLIT) == (j < SPLIT), t, torch.zeros_like(t))


def half_table(bias, mutation=None):
    """the bias the transposed-table backward adds: fp16(b log2 e) ln 2, evaluated in fp32"""
    t = (bias * LOG2E).half().float() * LN2
    if mutation == "half2_pair_swapped":            # query rows q and q + 1 of each half2 word exchanged
        S = t.shape[-2]
        src = torch.arange(S) ^ 1
        t = torch.where((src < S)[:, None], t[..., src.clamp(max=S - 1), :], torch.zeros_like(t))
    return t


def _f32_qkv(qkv):
    t = qkv.float().view(AB, AS, 3, AH, 64).permute(2, 0, 3, 1, 4)
    return t[0], t[1], t[2]


def emulate_attention_fwd(qkv, bias, kp, mutation=None):
    """fp32 emulation of a correct forward kernel: 64-key blocks, online soft-max with a running max, bf16 P in P.V with
    the denominator summed from the unrounded values, lse = m + log l.  bias: (1 or B, H, S, S)."""
    B, S, H = AB, AS, AH
    q, k, v = _f32_qkv(qkv)
    nb = (S + 63) // 64
    grow = lambda t: torch.nn.functional.pad(t, (0, 0, 0, nb * 64 - S))
    k, v = grow(k), grow(v)
    b = torch.nn.functional.pad(bias, (0, nb * 64 - S))
    keys = torch.arange(nb * 64)
    kpad = torch.nn.functional.pad(kp.bool(), (0, nb * 64 - S))
    dead = (keys >= S)[None, :] | kpad
    if mutation == "key_S_live":                     # the key == S of the partial last block taken as live
        dead[:, S] = False
    if mutation == "dead_pair":                      # the odd key of a pair masked with its even partner's pad flag
        dead = (keys >= S)[None, :] | kpad[:, keys & ~1]
    if mutation == "bias_cols_shifted_2":            # one key block reads its bias two columns late
        b = b.clone()
        b[..., 64:128] = torch.nn.functional.pad(bias, (0, nb * 64 + 2 - S))[..., 66:130]
    dead = dead.view(B, 1, 1, -1)
    m = torch.full((B, H, S), float("-inf"))
    l = torch.zeros(B, H, S)
    o = torch.zeros(B, H, S, 64)
    for kb in range(nb):
        sl = slice(kb * 64, kb * 64 + 64)
        s = (q @ k[..., sl, :].transpose(-1, -2) + b[..., sl]).masked_fill(dead[..., sl], float("-inf"))
        mn = torch.maximum(m, s.amax(-1))
        base = torch.where(mn == float("-inf"), torch.zeros_like(mn), mn)
        corr = (m - base).exp()
        m_prev, m = m, mn
        p = (s - base[..., None]).exp()
        l = l * (1.0 if mutation == "no_rescale_l" and kb == 1 else corr) + p.sum(-1)
        o = o * (1.0 if mutation == "no_rescale_o" and kb == 1 else corr[..., None]) + p.bfloat16().float() @ v[..., sl, :]
    lse = (m_prev if mutation == "lse_previous_max" else m) + l.log()
    of = o / l[..., None]
    st = torch.stack([of.sum(-1), (of * of).sum(-1)], -1).permute(1, 0, 2, 3).reshape(H, B * S, 2)
    return R.heads_to_rows(of, B, S, H).bfloat16(), lse, st


def emulate_attention_bwd(qkv, out, d_out, lse, bias, kp, mutation=None):
    """fp32 emulation of a correct backward: P recomputed from the given lse, bf16 P and dS in the products, fp32 dS
    returned for the bias gradient"""
    B, S, H = AB, AS, AH
    q, k, v = _f32_qkv(qkv)
    do = d_out.float().view(B, S, H, 64).permute(0, 2, 1, 3)
    o = out.float().view(B, S, H, 64).permute(0, 2, 1, 3)
    L = lse.view(B, H, S)
    dl = (do * o).sum(-1)
    if mutation == "row_g_reads_g8":                 # rows g of each 16-row fragment read row g + 8's lse and delta
        r = torch.arange(S)
        src = torch.where(r % 16 < 8, (r + 8).clamp(max=S - 1), r)
        L, dl = L[..., src], dl[..., src]
    s = (q @ k.transpose(-1, -2) + bias).masked_fill(kp.bool().view(B, 1, 1, S), float("-inf"))
    p = (s - L[..., None]).exp()
    ds = p * (do @ v.transpose(-1, -2) - dl[..., None])
    dv = p.bfloat16().float().transpose(-1, -2) @ do
    dq = (ds.bfloat16().float() @ k) * (1.0 if mutation == "dq_without_q_scale" else Q_SCALE)
    dk = ds.bfloat16().float().transpose(-1, -2) @ q
    rows = lambda t: R.heads_to_rows(t, B, S, H)
    return torch.cat([rows(dq), rows(dk), rows(dv)], 1).bfloat16(), ds


FWD_FORMS = {"key_S_live": "dense", "dead_pair": "dense", "bias_cols_shifted_2": "dense", "no_rescale_o": "dense",
             "no_rescale_l": "dense", "lse_previous_max": "dense", "sample_1_reads_sample_0": "per_sample",
             "seg_cross_not_zeroed": "two_segment", "seg_code_col_off_by_one": "two_segment"}
BWD_FORMS = {"row_g_reads_g8": "dense", "dq_without_q_scale": "dense", "half2_pair_swapped": "transposed",
             "dbias_t_launch_lost": "transposed", "fold_swaps_query_and_key": "transposed"}


def attention_outputs(d, form, mutation=None):
    """{name: (got, ref, bound, dtype)} for the emulated kernel (with an optional mistake) against the references"""
    B, S, H = AB, AS, AH
    bias = {"dense": d["bias"], "transposed": d["bias"], "per_sample": d["bias_ps"], "two_segment": lut_dense(d)}[form]
    seen = bias
    if mutation == "sample_1_reads_sample_0":
        seen = torch.stack([bias[0], bias[0]])
    if form == "two_segment":
        seen = lut_dense(d, mutation)
    seen = seen if seen.dim() == 4 else seen[None]
    out, lse, st = emulate_attention_fwd(d["qkv"], seen, d["kp"], mutation)
    fr = R.attention_ref(d["qkv"], bias, d["kp"], B, S, H)
    res = {"out": (out, fr.out, fr.out_err, torch.bfloat16), "lse": (lse, fr.lse, fr.dlse, torch.float32),
           "ln_stats": (st, fr.stats, fr.stats_err, torch.float32)}
    if form not in ("dense", "per_sample", "transposed") or mutation in FWD_FORMS:
        return res
    # the backward runs on the forward's outputs, as in training
    out, lse, _ = emulate_attention_fwd(d["qkv"], bias if bias.dim() == 4 else bias[None], d["kp"])
    eps_b = R.EPS_B_HALF if form == "transposed" else None
    bseen = half_table(bias, mutation) if form == "transposed" else bias
    dqkv, ds = emulate_attention_bwd(d["qkv"], out, d["d_out"], lse, bseen, d["kp"], mutation)
    br = R.attention_bwd_ref(d["qkv"], out, d["d_out"], lse, bias, d["kp"], B, S, H, Q_SCALE, eps_b=eps_b)
    res["dqkv"] = (dqkv, br.dqkv, br.dqkv_err, torch.bfloat16)
    if form == "per_sample":
        db, dbe = R.dbias_ref(br, d["dbias0"][None].expand(B, H, S, S), per_sample=True)
        res["dbias"] = (d["dbias0"] + ds, db, dbe, torch.float32)
    elif form == "dense":
        db, dbe = R.dbias_ref(br, d["dbias0"])
        res["dbias"] = (d["dbias0"] + ds.sum(0), db, dbe, torch.float32)
    else:
        # two launches accumulate into the transposed table, which is folded onto dbias and centred
        launches = 1 if mutation == "dbias_t_launch_lost" else 2
        acc = torch.zeros(H, S, S)
        for _ in range(launches):
            acc = acc + ds.sum(0)
        if mutation == "fold_swaps_query_and_key":
            acc = acc.transpose(-1, -2)
        got = d["dbias0"] + acc
        got = got - got.sum(-1, keepdim=True) / S
        db, dbe = R.center_ref(*R.dbias_ref(br, d["dbias0"], launches=2))
        res["dbias"] = (got, db, dbe, torch.float32)
    return res


def _ratio(got, ref, bound, dt):
    """largest |got - ref| / bound (the fraction of the bound used; inf for a NaN)"""
    err = (got.double() - ref.double()).abs()
    tol = bound + (2.0 ** -8 * ref.double().abs() if dt == torch.bfloat16 else 0.0)
    return torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / tol), nan=float("inf")).max().item()


@pytest.mark.parametrize("form", ["dense", "per_sample", "two_segment", "transposed"])
def test_attention_emulation_passes(att, form):
    for name, (got, ref, bound, dt) in attention_outputs(att, form).items():
        R.assert_within(got, ref, bound, 1.0, dt, what=f"{form} {name}")


@pytest.mark.parametrize("mutation", list(FWD_FORMS) + list(BWD_FORMS))
def test_attention_mutation_fails(att, mutation):
    """each mistake exceeds the bound at least ten-fold on at least one output (run with -s to see the factors)"""
    form = FWD_FORMS.get(mutation) or BWD_FORMS[mutation]
    ratios = {name: _ratio(*v) for name, v in attention_outputs(att, form, mutation).items()}
    name = max(ratios, key=ratios.get)
    print(f"{mutation}: {name} exceeds its bound {ratios[name]:.3g}-fold")
    assert ratios[name] >= 10, ratios


# ----------------------------------------------------------------------------------------------------------------------
# row kernels
# ----------------------------------------------------------------------------------------------------------------------
def _f32(t):
    return t.float().double()


def _c(v):
    return float(torch.tensor(v, dtype=torch.float32))


def fast_erf(x, d_rcp=0.0, d_ex2=0.0):
    """fp32 port of common.cuh fast_erf (fp64 arithmetic rounded to fp32 after each operation, an fma rounded once);
    d_rcp / d_ex2: relative errors of rcp.approx / ex2.approx"""
    x = x.double()
    ax = x.abs()
    t = _f32(_f32(1.0 / _f32(_c(0.3275911) * ax + 1.0)) * (1 + d_rcp))
    p = _f32(_c(1.061405429) * t + _c(-1.453152027))
    for c in (1.421413741, -0.284496736, 0.254829592):
        p = _f32(p * t + _c(c))
    p = _f32(p * t)
    e = _f32(_f32(torch.exp2(_f32(_f32(_c(-1.4426950408889634) * ax) * ax))) * (1 + d_ex2))
    return _f32(1.0 - p * e).copysign(x)


def gelu_erf(x, **k):
    x = x.double()
    return _f32(_f32(0.5 * x) * _f32(1.0 + fast_erf(_f32(x * _c(0.70710678118654752440)), **k)))


def gelu_grad(z, d_exp=0, **k):
    """d_exp = +-1: __expf off by its documented limit, 2 + floor(1.173 |x|) ulps"""
    z = z.double()
    cdf = _f32(0.5 * _f32(1.0 + fast_erf(_f32(z * _c(0.70710678118654752)), **k)))
    arg = _f32(_f32(-0.5 * z) * z)
    e = _f32(_f32(torch.exp(arg)) * (1 + d_exp * (2 + torch.floor(1.173 * arg.abs())) * 2.0 ** -23))
    return _f32(cdf + z * _f32(_c(0.3989422804014327) * e))


def test_gelu_constants():
    """the erf / gelu / gelu' allowances of kernel_ref hold for the fp32 port with every approximation at its limit"""
    z = _f32(torch.linspace(-10, 10, 200001, dtype=torch.float64))
    phi = torch.exp(-0.5 * z * z) / (2 * torch.pi) ** 0.5
    Phi = 0.5 * (1 + torch.special.erf(z / 2 ** 0.5))
    worst = [0.0, 0.0, 0.0]
    for dr in (-2.0 ** -23, 0.0, 2.0 ** -23):
        for de in (-2.0 ** -22, 0.0, 2.0 ** -22):
            worst[0] = max(worst[0], (fast_erf(z, d_rcp=dr, d_ex2=de) - torch.special.erf(z)).abs().max().item())
            worst[1] = max(worst[1], ((gelu_erf(z, d_rcp=dr, d_ex2=de) - z * Phi).abs() / z.abs().clamp_min(1e-30)).max().item())
            for dx in (-1, 1):
                worst[2] = max(worst[2], (gelu_grad(z, d_exp=dx, d_rcp=dr, d_ex2=de) - (Phi + z * phi)).abs().max().item())
    print(f"erf {worst[0]:.3g} of {R.ERF_ABS:.3g}, gelu / |x| {worst[1]:.3g} of {R.GELU_REL:.3g}, "
          f"gelu' {worst[2]:.3g} of {R.GELU_GRAD_ABS:.3g}")
    assert worst[0] <= R.ERF_ABS and worst[1] <= R.GELU_REL and worst[2] <= R.GELU_GRAD_ABS


LN_ROWS, LN_DIM = 300, 256          # 300 CTAs of one row each: a parts % 128 tail of 44 records


def _ln_rows(g, rows, dim):
    """N(0, 1) rows, then stress rows: |mean| / std ~ 10^3, an outlier in column 0, constant rows and var << eps"""
    x = torch.randn(rows, dim, generator=g) * (1 + 0.3 * torch.rand(rows, 1, generator=g))
    x[-8:-4] = 1000.0 + torch.randn(4, dim, generator=g)
    x[-4, 0] += 40.0
    x[-3] = 0.75
    x[-2] = 0.3 + 1e-4 * torch.randn(dim, generator=g)
    return x


@pytest.fixture(scope="module")
def rowk():
    g = torch.Generator().manual_seed(21)
    x = _ln_rows(g, LN_ROWS, LN_DIM)
    d = dict(x=x, dy=torch.randn(LN_ROWS, LN_DIM, generator=g), gamma=1 + 0.3 * torch.randn(LN_DIM, generator=g),
             beta=0.3 * torch.randn(LN_DIM, generator=g))
    # gelu inputs up to |z| = 8: a wide gamma
    d["gamma_gelu"] = 3 * torch.randn(LN_DIM, generator=g)
    return d


def _partials(terms, grid):
    """column sums of terms [rows, n] as the kernel forms them: row r in CTA r % grid (fp32, in row order), then
    partial_reduce_kernel: 32 lanes each over records p = lane (mod 32), lanes summed in order"""
    rows = terms.shape[0]
    part = torch.zeros(grid, terms.shape[1])
    for r in range(rows):
        part[r % grid] += terms[r]
    lanes = torch.zeros(32, terms.shape[1])
    for p in range(grid):
        lanes[p % 32] += part[p]
    tot = torch.zeros(terms.shape[1])
    for k in range(32):
        tot += lanes[k]
    return tot, part


def emulate_ln_bwd(d, gelu=False, mutation=None):
    """fp32 layernorm_bwd: the plain path reduces once about K = x[row][0]; the gelu path runs two-pass statistics"""
    X, G = d["x"].float(), d["dy"].float()
    g = d["gamma_gelu"] if gelu else d["gamma"]
    n = X.shape[1]
    if gelu:
        mean = X.sum(1, keepdim=True) / n
        xc = X - mean
        rstd = torch.rsqrt((xc * xc).sum(1, keepdim=True) / n + 1e-5)
        xh = xc * rstd
        Gp = (G.double() * gelu_grad(xh.double() * g.double() + d["beta"].double())).float()
        gy = Gp * g
        m1, m2 = gy.sum(1, keepdim=True) / n, (gy * xh).sum(1, keepdim=True) / n
    else:
        Gp = G
        K = torch.zeros_like(X[:, :1]) if mutation == "unshifted_var" else X[:, :1]
        xs = X - K
        ms = xs.sum(1, keepdim=True) / n
        rstd = torch.rsqrt(((xs * xs).sum(1, keepdim=True) / n - ms * ms).clamp_min(0) + 1e-5)
        if mutation == "neighbour_row_stats":             # every row reads the statistics of the row after it
            mean = torch.roll(K + ms, -1, 0)
            rstd = torch.roll(rstd, -1, 0)
            xs, ms = X - mean, torch.zeros_like(ms)
        gy = G * g
        m1 = gy.sum(1, keepdim=True) / n
        m2 = rstd * ((gy * xs).sum(1, keepdim=True) - ms * gy.sum(1, keepdim=True)) / n
        xh = (xs - ms) * rstd
        if mutation == "gamma_after_sums":                 # row sums of dy, then times gamma
            m1 = g * G.sum(1, keepdim=True) / n
            m2 = g * rstd * ((G * xs).sum(1, keepdim=True) - ms * G.sum(1, keepdim=True)) / n
    if mutation == "drop_xhat_term":
        m2 = torch.zeros_like(m2)
    dx = rstd * (gy - m1 - xh * m2)
    grid = min(X.shape[0], 132 * 8)
    dgamma, part = _partials(Gp * xh, grid)
    dbeta, partb = _partials(Gp, grid)
    if mutation == "last_partial_dropped":              # the reduction's tail loop stops one record early
        dgamma, dbeta = dgamma - part[-1], dbeta - partb[-1]
    return dx, dgamma, dbeta


def ln_bwd_outputs(d, gelu=False, mutation=None):
    dx, dg, db = emulate_ln_bwd(d, gelu, mutation)
    r = R.layernorm_bwd_ref(d["x"], d["dy"], d["gamma_gelu"] if gelu else d["gamma"], d["beta"], 1e-5, gelu=gelu)
    return {"dx": (dx.bfloat16(), r.dx, r.dx_err, torch.bfloat16), "dx_f32": (dx, r.dx, r.dx_err, torch.float32),
            "dgamma": (dg, r.dgamma, r.dgamma_err, torch.float32), "dbeta": (db, r.dbeta, r.dbeta_err, torch.float32)}


MERGE_W = 8                        # two images of an 8 x 8 grid, merged 2 x 2


def emulate_ln_fwd(d, mutation=None):
    """fp32 layernorm forward (two-pass statistics, fast_erf GELU) with the pixel-merge scatter, output [rows / 4, 4 dim]"""
    X = d["x"][:2 * MERGE_W * MERGE_W].float()
    n = X.shape[1]
    mean = X.sum(1, keepdim=True) / n
    xc = X - mean
    rstd = torch.rsqrt((xc * xc).sum(1, keepdim=True) / n + 1e-5)
    y = (xc * rstd * d["gamma_gelu"] + d["beta"]).double()
    y = gelu_erf(y).float()
    rows = torch.arange(X.shape[0])
    if mutation == "merge_xy_swapped":
        w = MERGE_W
        rows = (rows // (w * w)) * w * w + (rows % w) * w + (rows // w) % w
    orow, col, _ = R.ln_layout(X.shape[0], n, merge_grid_w=MERGE_W)
    out = torch.zeros(X.shape[0] // 4, 4 * n)
    out[orow[rows][:, None], col[rows]] = y
    return out


def ln_fwd_outputs(d, mutation=None):
    X = d["x"][:2 * MERGE_W * MERGE_W]
    r = R.layernorm_ref(X, d["gamma_gelu"], d["beta"], 1e-5, gelu=True)
    orow, col, _ = R.ln_layout(X.shape[0], X.shape[1], merge_grid_w=MERGE_W)
    ref = torch.zeros(X.shape[0] // 4, 4 * X.shape[1], dtype=torch.float64)
    err = torch.zeros_like(ref)
    ref[orow[:, None], col] = r.y
    err[orow[:, None], col] = r.err
    got = emulate_ln_fwd(d, mutation)
    return {"y": (got.bfloat16(), ref, err, torch.bfloat16), "y_f32": (got, ref, err, torch.float32)}


SR_B, SR_S = 3, 197                 # image adapter: 196 token rows behind the CLS slot of every sample


@pytest.fixture(scope="module")
def sres():
    g = torch.Generator().manual_seed(23)
    n = 64
    rows = SR_B * (SR_S - 1)
    rs = (torch.rand(SR_B * SR_S, generator=g) < 0.7).float() / 0.7      # drop-path keep mask / keep prob, per dx row
    return dict(dx=torch.randn(SR_B * SR_S, n, generator=g), o=torch.randn(rows, n, generator=g).bfloat16(),
                gamma=torch.randn(n, generator=g), rs_long=rs, rows=rows)


def sres_outputs(d, mutation=None):
    rows = d["rows"]
    idx = R.scale_resid_rows(rows, SR_S, SR_S - 1, 1)
    rs = d["rs_long"][:rows]
    got_idx = idx - 1 if mutation == "in_shift_off_by_one" else idx
    got_rs = d["rs_long"][idx] if mutation == "row_scale_by_input_row" else rs
    dd = got_rs[:, None] * d["dx"][got_idx] * d["gamma"]
    dg, _ = _partials(got_rs[:, None] * d["dx"][got_idx] * d["o"].float(), min(rows, 1056))
    db, _ = _partials(dd, min(rows, 1056))
    r = R.scale_resid_bwd_ref(d["dx"][idx], d["o"], d["gamma"], rs)
    return {"d_o": (dd.bfloat16(), r.d_o, r.d_o_err, torch.bfloat16), "dgamma": (dg, r.dgamma, r.dgamma_err, torch.float32),
            "dbias": (db, r.dbias, r.dbias_err, torch.float32)}


def misc_outputs(mutation=None):
    """l2_normalize_bwd, text_embed_bwd, geglu fwd / bwd and ln_fold, each emulated in fp32"""
    g = torch.Generator().manual_seed(29)
    res = {}
    x, dy = torch.randn(40, 96, generator=g) * 3, torch.randn(40, 96, generator=g)
    nrm = torch.sqrt((x * x).sum(1, keepdim=True))
    inv = 1.0 / nrm
    k = (x * dy).sum(1, keepdim=True) * inv * inv * inv
    v = dy * inv - (0.0 if mutation == "l2_no_projection" else x * k)
    ref, bnd = R.l2_normalize_bwd_ref(x, dy)
    res["l2_dx"] = (v, ref, bnd, torch.float32)
    # text_embed_bwd: B = 4 texts of T = 12 tokens, pad id 1 at the end of three of them; vocabulary of 9 (many duplicates)
    B, T, D, V = 4, 12, 32, 9
    tok = torch.randint(2, V, (B, T), generator=g)
    for b, p in enumerate((12, 7, 3, 10)):
        tok[b, p:] = 1
    dxe = torch.randn(B, T + 1, D, generator=g)
    t0, p0, c0 = torch.randn(V, D, generator=g), torch.randn(T + 1, D, generator=g), torch.randn(D, generator=g)
    live = (tok != 1) | (mutation == "pad_not_skipped")
    dt, dp = t0.clone(), p0.clone()
    bi, si = live.nonzero(as_tuple=True)
    dt.index_add_(0, tok[bi, si], dxe[bi, si + 1])
    dp.index_add_(0, si + 1, dxe[bi, si + 1])
    dp[0] += dxe[:, 0].sum(0)
    ok = (tok != 1)
    bi, si = ok.nonzero(as_tuple=True)
    res["dtable"] = (dt, *R.scatter_ref(t0, tok[bi, si], dxe[bi, si + 1]), torch.float32)
    dest = torch.cat([torch.zeros(B, dtype=torch.long), si + 1])
    res["dpos"] = (dp, *R.scatter_ref(p0, dest, torch.cat([dxe[:, 0], dxe[bi, si + 1]])), torch.float32)
    # geglu
    gl = (torch.randn(64, 2 * 128, generator=g) * 3).bfloat16()
    du = torch.randn(64, 128, generator=g).bfloat16()
    a, b = gl.double()[:, :128], gl.double()[:, 128:]
    if mutation == "geglu_halves_swapped":
        a, b = b, a
    u = (gelu_erf(a) * b).float()
    res["geglu_u"] = (u.bfloat16(), *R.geglu_ref(gl), torch.bfloat16)
    dgl = torch.cat([_f32(_f32(du.double() * b) * gelu_grad(a)), _f32(du.double() * gelu_erf(a))], 1).float()
    res["geglu_dgl"] = (dgl.bfloat16(), *R.geglu_bwd_ref(gl, du), torch.bfloat16)
    # ln_fold with the GeGLU interleave: 256 weight rows (two 128-row halves of wi_0), K = 200
    W = torch.randn(256, 200, generator=g) * 0.05
    lw, lb, bias = 1 + 0.2 * torch.randn(200, generator=g), 0.1 * torch.randn(200, generator=g), torch.randn(256, generator=g)
    f = R.ln_fold_ref(W, lw, lb, bias, interleave=1)
    wg = (W * lw).bfloat16()
    dest = f.rows + (128 if mutation == "interleave_wi1_first" else 0)
    buf_cs, buf_b = torch.zeros(512), torch.zeros(512)
    buf_cs[dest] = wg.float().sum(1)
    buf_b[dest] = (W * lb).sum(1) + bias
    res["fold_wg"] = (wg.float(), f.wg.double(), torch.zeros(256, 200, dtype=torch.float64), torch.float32)
    res["fold_colsum"] = (buf_cs[f.rows], f.colsum, f.colsum_err, torch.float32)
    res["fold_bias"] = (buf_b[f.rows], f.bias, f.bias_err, torch.float32)
    return res


ROW_MUTATIONS = {
    "neighbour_row_stats": "ln_bwd", "drop_xhat_term": "ln_bwd", "gamma_after_sums": "ln_bwd", "unshifted_var": "ln_bwd",
    "last_partial_dropped": "ln_bwd", "merge_xy_swapped": "ln_fwd", "in_shift_off_by_one": "sres",
    "row_scale_by_input_row": "sres", "l2_no_projection": "misc", "pad_not_skipped": "misc",
    "geglu_halves_swapped": "misc", "interleave_wi1_first": "misc"}


def row_outputs(kind, rowk, sres, mutation=None):
    if kind == "ln_bwd":
        return ln_bwd_outputs(rowk, False, mutation)
    if kind == "ln_bwd_gelu":
        return ln_bwd_outputs(rowk, True, mutation)
    if kind == "ln_fwd":
        return ln_fwd_outputs(rowk, mutation)
    if kind == "sres":
        return sres_outputs(sres, mutation)
    return misc_outputs(mutation)


@pytest.mark.parametrize("kind", ["ln_bwd", "ln_bwd_gelu", "ln_fwd", "sres", "misc"])
def test_row_emulation_passes(rowk, sres, kind):
    for name, (got, ref, bound, dt) in row_outputs(kind, rowk, sres).items():
        r = R.assert_within(got, ref, bound, 1.0, dt, what=f"{kind} {name}")
        print(f"{kind} {name}: {r:.3g} of the bound")


@pytest.mark.parametrize("mutation", list(ROW_MUTATIONS))
def test_row_mutation_fails(rowk, sres, mutation):
    """each mistake exceeds the bound at least ten-fold on at least one output (run with -s to see the factors)"""
    ratios = {name: _ratio(*v) for name, v in row_outputs(ROW_MUTATIONS[mutation], rowk, sres, mutation).items()}
    name = max(ratios, key=ratios.get)
    print(f"{mutation}: {name} exceeds its bound {ratios[name]:.3g}-fold")
    assert ratios[name] >= 10, ratios


# ----------------------------------------------------------------------------------------------------------------------
# optimizer
# ----------------------------------------------------------------------------------------------------------------------
OPT_BETAS, OPT_EPS, OPT_GS = (0.9, 0.98), 1e-8, 0.37
# (lr, wd) per param group: lr = 1e-2 with wd = 0.05 puts the order of decay and update above u |p|; a layer-decayed
# group (lr_scale 0.5) and a no-decay group
OPT_GROUPS = [(1e-2, 0.05), (0.5 * 1e-3, 0.05), (1e-3, 0.0)]
# (param group, step count t after the step, parameter kind): "f32", "bf16" (no master copy), "master" (bf16 + fp32 master)
OPT_TENSORS = [(0, 1, "f32"), (1, 2, "bf16"), (2, 10, "master"), (0, 1000, "f32"), (0, 2, "bf16"), (1, 10, "f32"),
               (2, 1, "bf16"), (0, 10, "master")]
OPT_N = 4096


def _opt_state(t, n, band, g):
    """m, v as a step count of t - 1 leaves them: zero at t = 1, else moments of gradients of the same scale"""
    if t == 1:
        return torch.zeros(n), torch.zeros(n)
    b1, b2 = OPT_BETAS
    scale = torch.where(band, 1e-7, 0.3)
    h1, h2 = torch.randn(n, generator=g) * scale, torch.randn(n, generator=g) * scale
    return (1 - b1 ** (t - 1)) * h1, (1 - b2 ** (t - 1)) * h2 * h2


@pytest.fixture(scope="module")
def opt():
    """every 4th gradient in a band 1e-9 <= |g| <= 1e-6 (sqrt(v) comparable to eps), every 16th gradient and state zero"""
    g = torch.Generator().manual_seed(11)
    tensors = []
    for gi, t, kind in OPT_TENSORS:
        i = torch.arange(OPT_N)
        band = i % 4 == 1
        grad = torch.randn(OPT_N, generator=g) * 0.3
        grad[band] = torch.sign(grad[band]) * 10.0 ** (-9 + 3 * torch.rand(int(band.sum()), generator=g))
        m, v = _opt_state(t, OPT_N, band, g)
        zero = i % 16 == 3
        grad[zero], m[zero], v[zero] = 0.0, 0.0, 0.0
        p = torch.randn(OPT_N, generator=g)
        if kind != "f32":
            p = p.bfloat16().float()
        tensors.append(dict(group=gi, t=t, kind=kind, p=p, g=grad, m=m, v=v))
    vgroups = list(dict.fromkeys((T["group"], T["t"]) for T in tensors))
    return dict(tensors=tensors, vgroups=vgroups)


def _bits_trunc_bf16(x):
    """bf16 by truncation (the mistake): drop the low 16 bits of the fp32 pattern"""
    return (x.view(torch.int32) & -65536).view(torch.float32).bfloat16()


def emulate_adam(d, mutation=None):
    """fp32 emulation of adam_multi_kernel in ``adam_math``'s order of operations, optionally with one planted mistake.
    -> per tensor (m', v', fp32 p' (None for bf16 without a master copy), bf16 p' (None for fp32))"""
    f = lambda x: torch.tensor(float(x), dtype=torch.float32)
    b1, b2 = OPT_BETAS[::-1] if mutation == "betas_swapped" else OPT_BETAS
    b1f, b2f, epsf, gs = f(b1), f(b2), f(OPT_EPS), f(OPT_GS)
    out = []
    for T in d["tensors"]:
        lr, wd = OPT_GROUPS[T["group"]]
        t = T["t"]
        vg = d["vgroups"].index((T["group"], t))
        if mutation == "bias_corr_t_minus_1" and t > 1:          # (at t = 1 the lagging count gives 0 / 0)
            t = t - 1
        if mutation == "bias_corr_neighbour_group":
            t = d["vgroups"][(vg + 1) % len(d["vgroups"])][1]
        bc = R.bias_correction(t, OPT_BETAS)
        p, m, v = T["p"].clone(), T["m"].clone(), T["v"].clone()
        x = T["g"] * gs
        lr_wd = f(wd) * f(lr)
        if mutation == "wd_into_g":
            x = x + f(wd) * p
        m = m * b1f + x * (1 - b1f)
        xv = T["g"] if mutation == "grad_scale_m_only" else x
        v = v * b2f + ((1 - b2f) * xv) * xv
        step = f(lr) * f(bc)
        if mutation == "eps_after_bias_correction":          # torch AdamW: lr m_hat / (sqrt(v_hat) + eps)
            q = (m / f(1 - b1 ** t)) / (torch.sqrt(v / f(1 - b2 ** t)) + epsf)
            step = f(lr)
        else:
            q = m / (torch.sqrt(v) + epsf)
        decay = lr_wd != 0 and mutation != "wd_into_g"
        if decay and mutation != "wd_after_update":
            p = p + p * -lr_wd
        p = p + -step * q
        if decay and mutation == "wd_after_update":
            p = p + p * -lr_wd
        p16 = None if T["kind"] == "f32" else (_bits_trunc_bf16(p) if mutation == "bf16_truncated" else p.bfloat16())
        out.append((m, v, None if T["kind"] == "bf16" else p, p16))
    return out


def adam_outputs(d, mutation=None):
    """{name: (got, ref, bound)} for every output of every tensor; a bf16 parameter without a master copy appears as its
    distance outside the allowed interval [bf16_rn(p' - dp'), bf16_rn(p' + dp')] against a bound of dp'"""
    res = {}
    for k, (T, (m, v, p32, p16)) in enumerate(zip(d["tensors"], emulate_adam(d, mutation))):
        lr, wd = OPT_GROUPS[T["group"]]
        r = R.adam_ref(T["p"], T["g"], T["m"], T["v"], t=T["t"], lr=lr, wd=wd, betas=OPT_BETAS, eps=OPT_EPS,
                       grad_scale=OPT_GS)
        res[f"t{k} m"] = (m, r.m, r.m_err)
        res[f"t{k} v"] = (v, r.v, r.v_err)
        if p32 is not None:
            res[f"t{k} p"] = (p32, r.p, r.p_err)
        if T["kind"] == "master":
            res[f"t{k} p16 == bf16(master)"] = (p16.double(), p32.bfloat16().double(), torch.zeros(OPT_N, dtype=torch.float64))
        if T["kind"] == "bf16":
            lo, hi = (r.p - r.p_err).bfloat16().double(), (r.p + r.p_err).bfloat16().double()
            gd = p16.double()
            res[f"t{k} p16"] = ((gd - hi).clamp_min(0) + (lo - gd).clamp_min(0), torch.zeros_like(gd), r.p_err)
    return res


def test_adam_reference_is_python_adam(opt):
    """adam_ref in fp64 is oracle/restated.adam_step (the reference's python Adam) run in fp64"""
    import restated
    for T in opt["tensors"]:
        lr, wd = OPT_GROUPS[T["group"]]
        r = R.adam_ref(T["p"], T["g"], T["m"], T["v"], t=T["t"], lr=lr, wd=wd, betas=OPT_BETAS, eps=OPT_EPS,
                       grad_scale=OPT_GS)
        p, m, v = T["p"].double(), T["m"].double(), T["v"].double()
        restated.adam_step(p, T["g"].double() * OPT_GS, m, v, T["t"], lr, *OPT_BETAS, OPT_EPS, wd)
        for got, want in ((p, r.p), (m, r.m), (v, r.v)):
            torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-15)


def test_adam_emulation_passes(opt):
    for name, (got, ref, bound) in adam_outputs(opt).items():
        r = R.assert_within(got, ref, bound, 1.0, torch.float32, what=name)
        print(f"adam {name}: {r:.3g} of the bound")
    for T, (_, _, _, p16) in zip(opt["tensors"], emulate_adam(opt)):
        if T["kind"] == "bf16":
            lr, wd = OPT_GROUPS[T["group"]]
            r = R.adam_ref(T["p"], T["g"], T["m"], T["v"], t=T["t"], lr=lr, wd=wd, betas=OPT_BETAS, eps=OPT_EPS,
                           grad_scale=OPT_GS)
            amb = R.bf16_param_check(p16, r.p, r.p_err)
            assert amb < OPT_N // 100, amb       # the either-neighbour band is a few elements, not a percentage


ADAM_MUTATIONS = ["bias_corr_t_minus_1", "bias_corr_neighbour_group", "eps_after_bias_correction", "wd_after_update",
                  "wd_into_g", "grad_scale_m_only", "betas_swapped", "bf16_truncated"]


@pytest.mark.parametrize("mutation", ADAM_MUTATIONS)
def test_adam_mutation_fails(opt, mutation):
    """each mistake exceeds the bound at least ten-fold on at least one output (run with -s to see the factors)"""
    outs = adam_outputs(opt, mutation)
    ratios = {name: _ratio(got, ref, bound, torch.float32) for name, (got, ref, bound) in outs.items()}
    name = max(ratios, key=ratios.get)
    assert ratios[name] >= 10, ratios
    # the factor printed leaves out elements whose bound is 0 (exact results, e.g. zero state), where any error is infinite
    finite = {n: _ratio(got[bound > 0], ref[bound > 0], bound[bound > 0], torch.float32)
              for n, (got, ref, bound) in outs.items() if (bound > 0).any()}
    name = max(finite, key=finite.get)
    print(f"{mutation}: {name} exceeds its bound {finite[name]:.3g}-fold")


# gradient norm: 1100 tiny tensors, then a two-chunk tensor with a 1000-element tail chunk and a bf16-valued one, so that
# 1105 chunks > 1056 CTAs and the last CTAs' second chunks are the big ones
@pytest.fixture(scope="module")
def norm_grads():
    g = torch.Generator().manual_seed(12)
    sizes = (torch.randint(1, 200, (1100,), generator=g)).tolist() + [2 * R.ADAM_CHUNK + 1000, R.ADAM_CHUNK + 5]
    grads = [torch.randn(n, generator=g) * (0.1 + torch.rand(1, generator=g)) for n in sizes]
    grads[-1] = grads[-1].bfloat16().float()
    return grads


def emulate_grad_norm(grads, mf, max_norm, mutation=None):
    """fp32 emulation of grad_sumsq_kernel (per-thread order, shuffle tree, warp partials) and grad_norm_finalize_kernel"""
    chunks = R.norm_chunks([x.numel() for x in grads])
    grid = min(len(chunks), R.NORM_GRID_CAP)
    acc = torch.zeros(grid, 256)
    for c, (ti, off, n) in enumerate(chunks):
        if mutation == "second_chunk_dropped" and c >= grid:
            continue
        if mutation == "tail_chunk_dropped" and n < R.ADAM_CHUNK and grads[ti].numel() > R.ADAM_CHUNK:
            continue
        x = grads[ti][off:off + n]
        if n == R.ADAM_CHUNK:            # vector path: per thread 8 loads of 4 elements, ((a + b) + c) + d added per load
            sq = (x * x).view(8, 256, 4)
            terms = torch.zeros(256, 32)
            terms[:, ::4] = (((sq[..., 0] + sq[..., 1]) + sq[..., 2]) + sq[..., 3]).t()
        else:                            # scalar path: thread t adds elements t, t + 256, ...
            terms = torch.nn.functional.pad(x * x, (0, R.ADAM_CHUNK - n)).view(32, 256).t()
        b = c % grid
        for j in range(32):
            acc[b] = acc[b] + terms[:, j]
    w = acc.view(grid, 8, 32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, :, torch.arange(32) ^ o]
    part = torch.zeros(grid)
    for k in range(8):
        part = part + w[:, k, 0]
    s = float(part.double().sum())
    mff = torch.tensor(1.0 if mutation == "no_multiply_factor" else mf, dtype=torch.float32)
    norm = mff * torch.tensor(s ** 0.5, dtype=torch.float32)
    r = torch.tensor(max_norm, dtype=torch.float32) / (norm + torch.tensor(1e-6, dtype=torch.float32))
    coef = torch.where(r >= 1, torch.ones(()), r) if max_norm > 0 else torch.ones(())
    return norm, torch.tensor(mf, dtype=torch.float32) * coef


NORM_MUTATIONS = ["second_chunk_dropped", "tail_chunk_dropped", "no_multiply_factor"]


def norm_outputs(grads, mutation=None):
    mf = 0.37
    ref0 = R.grad_norm_ref(grads, mf)
    ref = R.grad_norm_ref(grads, mf, 0.5 * ref0.norm)          # clips to half
    norm, scale = emulate_grad_norm(grads, mf, 0.5 * ref0.norm, mutation)
    d = lambda x: torch.tensor([x], dtype=torch.float64)
    return ref, {"norm": (norm.reshape(1), d(ref.norm), d(ref.norm_err)), "scale": (scale.reshape(1), d(ref.scale), d(ref.scale_err))}


def test_grad_norm_emulation_passes(norm_grads):
    ref, outs = norm_outputs(norm_grads)
    assert ref.n_chunks == 1105 and ref.grid == 1056 and ref.depth == 1 + 64 + 13
    for name, (got, want, bound) in outs.items():
        r = R.assert_within(got, want, bound, 1.0, torch.float32, what=name)
        print(f"grad norm {name}: {r:.3g} of the bound")


@pytest.mark.parametrize("mutation", NORM_MUTATIONS)
def test_grad_norm_mutation_fails(norm_grads, mutation):
    _, outs = norm_outputs(norm_grads, mutation)
    ratios = {name: _ratio(got, want, bound, torch.float32) for name, (got, want, bound) in outs.items()}
    name = max(ratios, key=ratios.get)
    print(f"{mutation}: {name} exceeds its bound {ratios[name]:.3g}-fold")
    assert ratios[name] >= 10, ratios


def test_clip_scale_keeps_nan_and_zeroes_inf():
    """the reference of out[1]: a NaN norm gives a NaN scale (clamp(max=1) keeps it), an infinite one a zero scale"""
    import math
    assert math.isnan(R.clip_scale_ref(float("nan"), 0.0, 1.0, 1.0)[0])
    assert R.clip_scale_ref(float("inf"), 0.0, 0.5, 1.0)[0] == 0.0
    assert R.clip_scale_ref(3.0, 0.0, 0.5, 0.0) == (0.5, 0.0)


# ----------------------------------------------------------------------------------------------------------------------
# embedding, gather, transpose and ranking kernels
# ----------------------------------------------------------------------------------------------------------------------
def _key32(x):
    """order key of one fp32 value (``order_key`` of csrc/recall.cu)"""
    if x != x:
        return 0xFFFFFFFF
    if x == 0:
        return 0x80000000
    u = struct.unpack("<I", struct.pack("<f", x))[0]
    return (~u & 0xFFFFFFFF) if u >> 31 else u | 0x80000000


def topk10_warp(flat, ld, rows, C, mutation=None):
    """Python port of ``topk_rows_kernel`` on a flat fp32 buffer of row pitch ld: 32 lane lists of strided columns, then 10
    arg-max merge rounds.  Mutations: 'strict_gt_neg_inf' (float lists initialised to -inf, an entry inserted only when
    strictly greater than the last one: the rule before the total order), 'ties_to_larger_index', 'ignore_ld'."""
    vals, none = flat.tolist(), 0x7FFFFFFF
    out = []
    for r in range(rows):
        base = r * (C if mutation == "ignore_ld" else ld)
        lanes = []
        for lane in range(32):
            if mutation == "strict_gt_neg_inf":
                t = [(float("-inf"), -none)] * 10                  # (value, -column): larger is better
                for c in range(lane, C, 32):
                    x = vals[base + c]
                    if x > t[9][0]:
                        t[9] = (x, -c)
                        for i in range(9, 0, -1):
                            if t[i][0] > t[i - 1][0]:
                                t[i], t[i - 1] = t[i - 1], t[i]
            else:
                t = [0] * 10
                for c in range(lane, C, 32):
                    low, k = (c if mutation == "ties_to_larger_index" else ~c & 0xFFFFFFFF), _key32(vals[base + c])
                    if k > t[9] >> 32 or (mutation == "ties_to_larger_index" and k == t[9] >> 32):
                        t[9] = k << 32 | low
                        for i in range(9, 0, -1):
                            if t[i] > t[i - 1]:
                                t[i], t[i - 1] = t[i - 1], t[i]
            lanes.append(t)
        row = []
        for _ in range(10):
            if mutation == "strict_gt_neg_inf":
                best = max(lanes, key=lambda t: (t[0][0], t[0][1]))[0]
                row.append(-1 if best[1] == -none else -best[1])
                if best[1] != -none:
                    w = next(t for t in lanes if t[0] == best)
                    w[:] = w[1:] + [(float("-inf"), -none)]
                continue
            best = max(t[0] for t in lanes)
            low = best & 0xFFFFFFFF
            row.append(-1 if best == 0 else (low if mutation == "ties_to_larger_index" else ~low & 0xFFFFFFFF))
            if best:
                w = next(t for t in lanes if t[0] == best)
                w[:] = w[1:] + [0]
        out.append(row)
    return torch.tensor(out, dtype=torch.int32)


def _topk_rows(C, ld):
    """rows for the top-10 port, in a buffer of pitch ld whose gap holds NaN (which would rank first if read): ties within a
    lane (columns c and c + 32) and across lanes, -inf, NaN of both signs, signed zeros, an all-equal row, an all -inf row,
    an all-NaN row, fewer than 10 entries above -inf"""
    g = torch.Generator().manual_seed(C)
    x = torch.tensor([-1.0, 0.0, 0.5, 2.0])[torch.randint(0, 4, (14, C), generator=g)]
    if C > 32:
        x[0, 32:] = x[0, :C - 32].clone()                                # column c + 32 equals column c: a tie within a lane
    x[1] = 0.5
    x[2] = float("-inf")
    x[3] = float("nan")
    x[4] = float("-inf")
    x[4, ::9] = 1.0
    x[5, ::3] = float("-inf")
    x[5, 1::4] = float("nan")
    x[6, ::2] = -0.0
    x[6, 1::3] = float("-inf")
    x[7].view(torch.int32)[::4] = 0xFFC00001 - 2 ** 32            # negative NaN
    x[8, ::2] = float("inf")
    buf = torch.full((x.shape[0], ld), float("nan"))
    buf[:, :C] = x
    return x, buf.view(-1)


@pytest.mark.parametrize("C", [1, 7, 10, 31, 33, 70])
def test_topk10_port_is_the_total_order(C):
    x, flat = _topk_rows(C, C + 3)
    want = R.topk10_ref(x)[0]
    assert torch.equal(topk10_warp(flat, C + 3, x.shape[0], C), want)
    finite = torch.isfinite(x).all(1)
    tv, ti = x[finite].topk(min(10, C), dim=1, sorted=True)
    assert torch.equal(R.topk10_ref(x)[1][finite][:, :min(10, C)], tv)


def test_topk10_reference_ranks_like_torch():
    """NaN first, then values, -inf like any other value, ties by the smaller column: torch.sort(stable) on the CPU"""
    x = torch.tensor([[1.0, float("nan"), float("-inf"), 2.0, float("-inf"), 0.5, 2.0, float("nan"), -0.0, 0.0, -1.0, 0.5]])
    i, v = R.topk10_ref(x)
    s = torch.sort(x, dim=1, descending=True, stable=True).indices[:, :10]
    assert i.tolist() == [[1, 7, 3, 6, 0, 5, 11, 8, 9, 10]] and torch.equal(i.long(), s)
    assert torch.isnan(v[0, :2]).all() and v[0, 2:].tolist() == [2.0, 2.0, 1.0, 0.5, 0.5, -0.0, 0.0, -1.0]
    i3, v3 = R.topk10_ref(x[:, :3])
    assert i3.tolist() == [[1, 0, 2] + [-1] * 7] and v3[0, 3:].eq(float("-inf")).all()


@pytest.mark.parametrize("mutation", ["strict_gt_neg_inf", "ties_to_larger_index", "ignore_ld"])
def test_topk10_mutation_fails(mutation):
    """each mistake returns a wrong column on some rows; the earlier strict-> rule exactly on the rows holding -inf or NaN
    (run with -s to see the counts)"""
    C = 70
    x, flat = _topk_rows(C, C + 3)
    want = R.topk10_ref(x)[0]
    bad = (topk10_warp(flat, C + 3, x.shape[0], C, mutation) != want).any(1)
    print(f"{mutation}: {int(bad.sum())} of {x.shape[0]} rows wrong")
    assert bad.sum() >= 3
    if mutation == "strict_gt_neg_inf":
        special = (torch.isnan(x) | (x == float("-inf"))).any(1)
        assert torch.equal(bad, special & bad) and bad[[2, 3, 4]].all()


def emulate_l2_normalize(x, mutation=None):
    """``l2_normalize_kernel`` in fp32: 256 threads, thread t adds x[c]^2 for c = t, t + 256, ...; a butterfly over each
    warp; lane 0 of warp 0 adds the 8 warp partials in order; y = x * (1 / max(sqrt(s), 1e-12)).  Mutations: 'no_clamp',
    'sum_in_bf16' (squares and partial sums rounded to bf16)."""
    rows, D = x.shape
    xs = x.float()
    sq = torch.nn.functional.pad(xs * xs, (0, (-D) % 256)).view(rows, -1, 256)
    rnd = (lambda t: t.bfloat16().float()) if mutation == "sum_in_bf16" else (lambda t: t)
    part = torch.zeros(rows, 256)
    for s in range(sq.shape[1]):
        part = rnd(part + rnd(sq[:, s]))
    w = part.view(rows, 8, 32)
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        w = rnd(w + w[:, :, lane ^ o])
    tot = torch.zeros(rows)
    for i in range(8):
        tot = rnd(tot + w[:, i, 0])
    nrm = torch.sqrt(tot)
    inv = 1.0 / (nrm if mutation == "no_clamp" else torch.clamp_min(nrm, float(np.float32(1e-12))))
    return xs * inv[:, None]


def _l2_rows(D):
    g = torch.Generator().manual_seed(D)
    x = torch.randn(8, D, generator=g) * (0.5 + torch.rand(8, 1, generator=g))
    x[1] *= 1e6
    x[2] *= 1e-6
    x[3] = 0.0
    x[4] *= 1e-15
    x[5] = 0.0
    x[5, D // 2] = 3.7
    return x


@pytest.mark.parametrize("D", [1, 31, 257, 1536, 4096])
def test_l2_normalize_emulation_passes(D):
    x = _l2_rows(D)
    y = emulate_l2_normalize(x)
    ref, bound = R.l2_normalize_ref(x)
    r = R.assert_within(y, ref, bound, 1.0, torch.float32, what=f"l2_normalize D={D}")
    print(f"l2_normalize D={D}: {r:.3g} of the bound")
    assert y[3].eq(0).all() and not torch.isnan(y).any()


@pytest.mark.parametrize("mutation", ["no_clamp", "sum_in_bf16"])
def test_l2_normalize_mutation_fails(mutation):
    x = _l2_rows(1536)
    ref, bound = R.l2_normalize_ref(x)
    r = _ratio(emulate_l2_normalize(x, mutation), ref, bound, torch.float32)
    print(f"{mutation}: exceeds its bound {r:.3g}-fold")
    assert r >= 10


def emulate_transpose(x, mutation=None):
    """``transpose_bf16_vec_kernel``: 64 x 64 tiles staged in shared memory as tile[col][row]; 'tile_swapped' writes the
    staged tile back as tile[row][col]"""
    rows, cols = x.shape
    out = torch.empty(cols, rows, dtype=x.dtype)
    for r0 in range(0, rows, 64):
        for c0 in range(0, cols, 64):
            blk = x[r0:r0 + 64, c0:c0 + 64]
            tile = torch.zeros(64, 64, dtype=x.dtype)
            tile[:blk.shape[1], :blk.shape[0]] = blk.t()
            if mutation == "tile_swapped":
                tile = tile.t()
            out[c0:c0 + 64, r0:r0 + 64] = tile[:min(64, cols - c0), :min(64, rows - r0)]
    return out


def emulate_row_gather(src, idx, fill, add, out_dtype, mutation=None):
    """``row_gather_kernel`` row by row; 'add_period_off_by_one' takes the addend row r % (period - 1)"""
    period = add.shape[0] - (1 if mutation == "add_period_off_by_one" else 0)
    rows = []
    for r, s in enumerate(idx.tolist()):
        v = src[s].float() if s >= 0 else fill
        rows.append(v + add[r % period])
    return torch.stack(rows).to(out_dtype)


def emulate_bias_block(table, bucket, ids, n, lo, canvas, mutation=None):
    """``relpos_bias_block_kernel`` on the flat canvas; 'cols_without_lo' writes block row i at columns j instead of lo + j,
    'pad_id_to_0' maps -1 ids to 0 instead of n - 1"""
    out = canvas.clone()
    Bb, H, S, s_pad = canvas.shape
    flat = out.view(-1)
    fix = 0 if mutation == "pad_id_to_0" else n - 1
    for bb in range(Bb):
        p = [fix if q < 0 else q for q in ids[bb].tolist()]
        for i in range(n):
            base = (bb * H * S + lo + i) * s_pad + (0 if mutation == "cols_without_lo" else lo)
            for j in range(n):
                for h in range(H):
                    flat[base + h * S * s_pad + j] = table[bucket[p[i], p[j]], h]
    return out


def _exact_cases(mutation=None):
    """(got, want) pairs of the exact kernels' emulations"""
    g = torch.Generator().manual_seed(31)
    x = torch.randn(130, 200, generator=g).bfloat16()
    src = torch.randn(40, 12, generator=g).bfloat16()
    idx = torch.randint(-1, 40, (23,), generator=g)
    fill, add = torch.randn(12, generator=g), torch.randn(5, 12, generator=g)
    table, bucket = torch.randn(50, 3, generator=g), torch.randint(0, 50, (30, 30), generator=g)
    ids = torch.randint(0, 30, (2, 9), generator=g)
    ids[:, -2:] = -1
    canvas = torch.full((2, 3, 14, 16), float("nan"))
    return {"transpose": (emulate_transpose(x, mutation), R.transpose_ref(x)),
            "row_gather": (emulate_row_gather(src, idx, fill, add, torch.bfloat16, mutation),
                           R.row_gather_ref(src, idx, torch.bfloat16, fill, add)),
            "bias_block": (emulate_bias_block(table, bucket, ids, 9, 4, canvas, mutation),
                           R.relpos_bias_block_ref(table, bucket, ids, 9, 4, canvas)[0])}


def _same_bits(a, b):
    it = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    return a.shape == b.shape and torch.equal(a.view(it), b.view(it))


def test_exact_emulations_match_references():
    for name, (got, want) in _exact_cases().items():
        assert _same_bits(got, want), name


@pytest.mark.parametrize("mutation,kernel", [("tile_swapped", "transpose"), ("add_period_off_by_one", "row_gather"),
                                             ("cols_without_lo", "bias_block"), ("pad_id_to_0", "bias_block")])
def test_exact_mutation_fails(mutation, kernel):
    got, want = _exact_cases(mutation)[kernel]
    assert not _same_bits(got, want), mutation


def test_topk_within_and_recall_bounds():
    """an fp32 similarity ranked by the total order passes ``topk_within`` against the fp64 one, and its Recall@k lies within
    the near-tie rows; a list with its 1st and 10th entries swapped, or with the 11th entry in place of the 10th where the
    gap is wide, fails"""
    g = torch.Generator().manual_seed(37)
    a = torch.nn.functional.normalize(torch.randn(60, 64, generator=g), dim=1)
    b = torch.nn.functional.normalize(torch.randn(90, 64, generator=g), dim=1)
    b[1] = b[0] + 1e-7                                             # near-duplicate candidates
    z = a.double() @ b.double().t()
    dz = R.Z_TAU * (a.double().abs() @ b.double().abs().t())
    sim = a @ b.t()
    idx = R.topk10_ref(sim)[0]
    assert R.topk_within(z, dz, idx).all()
    cand, own = torch.randint(0, 30, (90,), generator=g), torch.randint(0, 30, (60,), generator=g)
    hits, near = R.recall_ref(z, dz, cand, own)
    got = R.recall_hits_ref(idx, cand, own)
    assert all(abs(x - y) <= n for x, y, n in zip(got, hits, near))
    swapped = idx.clone()
    swapped[:, [0, 9]] = swapped[:, [9, 0]]
    assert not R.topk_within(z, dz, swapped).any()
    full = z.topk(11, dim=1).indices
    wide = (z.gather(1, full[:, 9:10]) - z.gather(1, full[:, 10:11]) > 1e-3).squeeze(1)
    eleventh = idx.clone().long()
    eleventh[:, 9] = full[:, 10]
    assert not R.topk_within(z, dz, eleventh)[wide].any() and wide.sum() > 30
    dup = idx.clone()
    dup[:, 9] = dup[:, 8]
    assert not R.topk_within(z, dz, dup).any()
