"""CPU: the fp64 reference and per-element bounds of tests/kernel_ref.py.  A correct kernel, emulated here in fp32 (bf16
operands, fp32 matmul, the epilogue and the LayerNorm statistics in fp32 as the kernel evaluates them; for attention the
blocked online soft-max and the recomputing backward), must pass the bounds; each of the subtle mistakes a GEMM, InfoNCE
or attention kernel can make must fail them."""
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
