"""GPU: every sm_90a kernel through the C-ABI vs a plain PyTorch fp32 reference of the same op.
Tolerances are stated per test: operands are bf16 (8 mantissa bits), accumulation fp32."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


def relerr(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-9)).item()


def interleave_geglu(w0, w1):
    """[F,d],[F,d] -> bf16 [2F,d] where each 256-row GEMM tile holds 128 rows of wi_0 followed by the matching
    128 rows of wi_1, so the epilogue can form gelu(a) * b inside one accumulator tile."""
    F_, d = w0.shape
    assert F_ % 128 == 0, "ffn_embed_dim must be a multiple of 128"
    return torch.stack([w0.bfloat16().view(F_ // 128, 128, d), w1.bfloat16().view(F_ // 128, 128, d)], dim=1).reshape(2 * F_, d).contiguous()


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,Kd", [(128, 256, 64), (1000, 384, 48), (1576, 1536, 1536), (12608, 4608, 1536), (37, 768, 256)])
def test_gemm_store(K, cg, M, N, Kd):
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = (torch.randn(M, Kd, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    cs = torch.rand(N, device="cuda", generator=g) + 0.5
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    K.gemm(a, w, K.EPI_STORE_BF16, out, bias=bias, colscale=cs, cta_group=cg)
    want = (a.float() @ w.float().t() + bias) * cs
    assert relerr(out, want) < 6e-3          # bf16 output rounding: 2^-9 relative
    out32 = torch.empty(M, N, device="cuda", dtype=torch.float32)
    K.gemm(a, w, K.EPI_STORE_F32, out32, bias=bias, cta_group=cg)
    assert relerr(out32, a.float() @ w.float().t() + bias) < 1e-5   # fp32 accumulate of exact bf16 products


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M", [1000, 136])           # 136: the small-batch text rows (8 x 17), one partial row panel
def test_gemm_geglu_and_residual(K, cg, M):
    d, F = 256, 1024
    g = torch.Generator(device="cuda").manual_seed(7)
    h = (torch.randn(M, d, device="cuda", generator=g)).bfloat16()
    w0 = (torch.randn(F, d, device="cuda", generator=g) * 0.05)
    w1 = (torch.randn(F, d, device="cuda", generator=g) * 0.05)
    w01 = interleave_geglu(w0, w1)
    u = torch.empty(M, F, device="cuda", dtype=torch.bfloat16)
    K.gemm(h, w01, K.EPI_GEGLU_BF16, u, cta_group=cg)
    want = torch.nn.functional.gelu(h.float() @ w0.bfloat16().float().t()) * (h.float() @ w1.bfloat16().float().t())
    assert relerr(u, want) < 6e-3
    w2 = (torch.randn(d, F, device="cuda", generator=g) * 0.05).bfloat16()
    b2 = torch.randn(d, device="cuda", generator=g)
    gamma = torch.randn(d, device="cuda", generator=g)
    x = torch.randn(M, d, device="cuda", generator=g)
    x0 = x.clone()
    K.gemm(u, w2, K.EPI_RESID_F32, x, bias=b2, gamma=gamma, resid=x, cta_group=cg)
    want = x0 + gamma * (u.float() @ w2.float().t() + b2)
    assert relerr(x, want) < 1e-5


def test_gemm_row_remap_and_broadcast_residual(K):
    B, P, d, Kd = 3, 196, 256, 256
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn(B * P, Kd, device="cuda", generator=g).bfloat16()
    w = (torch.randn(d, Kd, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(d, device="cuda", generator=g)
    pos = torch.randn(P + 1, d, device="cuda", generator=g)
    x = torch.full((B, P + 1, d), 7.0, device="cuda")
    K.gemm(a, w, K.EPI_RESID_F32, x.view(B * (P + 1), d), bias=bias, resid=pos, out_group=P, out_group_stride=P + 1,
           out_row_offset=1, resid_period=P, resid_row_offset=1)
    want = (a.float() @ w.float().t() + bias).view(B, P, d) + pos[1:]
    assert relerr(x[:, 1:], want) < 1e-5
    assert torch.all(x[:, 0] == 7.0)       # CLS slot untouched


@pytest.mark.parametrize("B,S,H,use_bias,use_pad", [(2, 17, 4, True, True), (2, 64, 4, False, False),
                                                     (3, 197, 24, True, False), (2, 500, 4, True, True), (1, 750, 2, True, True)])
def test_attention(K, B, S, H, use_bias, use_pad):
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(S)
    qkv = (torch.randn(B * S, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
    s_pad = (S + 7) // 8 * 8
    bias = None
    if use_bias:
        bias = torch.zeros(H, S, s_pad, device="cuda")
        bias[:, :, :S] = torch.randn(H, S, S, device="cuda", generator=g)
    kp = None
    if use_pad:
        kp = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
        for b in range(B):
            kp[b, S - 1 - 3 * b:] = 1
    out = K.attention(qkv, bias, kp, B, S, H)
    q, k, v = qkv.float().view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    sc = q @ k.transpose(-1, -2)
    if bias is not None:
        sc = sc + bias[None, :, :, :S]
    if kp is not None:
        sc = sc.masked_fill(kp.bool()[:, None, None, :], float("-inf"))
    want = (sc.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * S, D)
    assert relerr(out, want) < 8e-3          # probabilities and output are rounded to bf16


@pytest.mark.parametrize("rows,dim,in_dt,out_dt,affine,gelu,merge", [
    (1000, 1536, torch.float32, torch.bfloat16, True, False, 0), (300, 6144, torch.bfloat16, torch.bfloat16, True, False, 0),
    (77, 256, torch.float32, torch.bfloat16, True, False, 0), (2 * 56 * 56, 384, torch.bfloat16, torch.bfloat16, True, True, 56),
    (999, 512, torch.bfloat16, torch.bfloat16, True, True, 0), (50, 1536, torch.bfloat16, torch.float32, False, True, 0),
    (64, 64, torch.bfloat16, torch.bfloat16, True, True, 8)])
def test_layernorm(K, rows, dim, in_dt, out_dt, affine, gelu, merge):
    g = torch.Generator(device="cuda").manual_seed(rows)
    x = (torch.randn(rows, dim, device="cuda", generator=g) * 2 + 0.5).to(in_dt)
    gm = torch.randn(dim, device="cuda", generator=g) if affine else None
    bt = torch.randn(dim, device="cuda", generator=g) if affine else None
    out = torch.zeros(rows // 4, dim * 4, device="cuda", dtype=out_dt) if merge else torch.empty(rows, dim, device="cuda", dtype=out_dt)
    K.layernorm(x, gm, bt, out, rows=rows, dim=dim, gelu=gelu, merge_grid_w=merge)
    want = torch.nn.functional.layer_norm(x.float(), (dim,), gm, bt, 1e-5)
    if gelu:
        want = torch.nn.functional.gelu(want)
    if merge:
        w = merge
        want = want.view(rows // (w * w), w // 2, 2, w // 2, 2, dim).permute(0, 1, 3, 2, 4, 5).reshape(rows // 4, 4 * dim)
    assert relerr(out, want) < (1e-5 if out_dt == torch.float32 else 6e-3)


def test_text_embed_and_relpos_bias(K):
    import restated as R
    B, T, D, H = 5, 9, 256, 4
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(4, 1000, (B, T), generator=g)
    tok[1, -2:] = 1
    tok[3, -4:] = 1
    table = torch.randn(1000, D, generator=g)
    pos = torch.randn(514, D, generator=g)
    cls = torch.randn(D, generator=g)
    x, pad = K.text_embed(tok.cuda(), table.cuda(), pos.cuda(), cls.cuda(), 1)
    want = torch.cat([cls.expand(B, 1, D), table[tok]], 1) + pos[: T + 1]
    wpad = torch.zeros(B, T + 1, dtype=torch.bool)
    wpad[:, 1:] = tok.eq(1)
    want = want * (~wpad).unsqueeze(-1)
    assert torch.equal(pad.bool().cpu(), wpad)
    assert torch.equal(x.cpu(), want)                       # pure gather + one fp32 add: bit exact
    bucket = R.make_token_bucket_position(256)
    tab = torch.randn(514, H, generator=g)
    bias = K.relpos_bias_build(tab.cuda(), bucket.cuda(), T + 1, H)
    assert torch.equal(bias[:, :, : T + 1].cpu(), R.rel_pos_bias(tab, bucket, T + 1))
    assert torch.all(bias[:, :, T + 1:] == 0)


def test_patchify_and_l2norm(K):
    g = torch.Generator().manual_seed(1)
    img = torch.randn(2, 3, 32, 32, generator=g)
    a = K.image_patchify4(img.cuda())
    want = img.view(2, 3, 8, 4, 8, 4).permute(0, 2, 4, 1, 3, 5).reshape(2 * 64, 48).bfloat16()
    assert torch.equal(a.cpu(), want)
    x = torch.randn(7, 300, generator=g)
    y, y16 = K.l2_normalize_rows(x.cuda(), want_bf16=True)
    torch.testing.assert_close(y.cpu(), torch.nn.functional.normalize(x, dim=1), atol=1e-6, rtol=1e-6)
    assert relerr(y16, y) < 4e-3


def test_layernorm_remap_group_pad_and_accumulate(K):
    B, Tp, T, d, cg, cpad, halo = 2, 30, 21, 96, 24, 64, 4
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.randn(B * Tp, d, device="cuda", generator=g).bfloat16()
    out = torch.zeros(B * Tp, (d // cg) * cpad, dtype=torch.bfloat16, device="cuda")
    K.layernorm(x, None, None, out, rows=B * Tp, dim=d, gelu=True, row_period=Tp, row_valid=T, out_period=Tp,
                out_row_shift=halo, group_in=cg, group_out=cpad)
    want = torch.nn.functional.gelu(torch.nn.functional.layer_norm(x.float(), (d,)))
    o = out.view(B, Tp, d // cg, cpad)
    assert relerr(o[:, halo:halo + T, :, :cg].reshape(B, T, d), want.view(B, Tp, d)[:, :T]) < 6e-3
    assert torch.all(o[:, :halo] == 0) and torch.all(o[:, halo + T:] == 0) and torch.all(o[..., cg:] == 0)
    acc = torch.ones(B, T + 1, d, device="cuda")
    K.layernorm(x, None, None, acc.view(B * (T + 1), d), rows=B * Tp, dim=d, gelu=True, row_period=Tp, row_valid=T,
                out_period=T + 1, out_row_shift=1, accumulate=True)
    assert relerr(acc[:, 1:], 1 + want.view(B, Tp, d)[:, :T]) < 1e-5 and torch.all(acc[:, 0] == 1)


@pytest.mark.parametrize("cg", [1, 2])
def test_gemm_fused_layernorm_and_stats(K, cg):
    """LN(x) W^T + b computed as rstd*(acc - mu*colsum) + bias' on un-normalised bf16 rows, plus the (sum, sumsq)
    side output and bf16 copy of the RESID epilogue (fused-LN chain of the encoder layer)."""
    from one_peace_b200.transformer.transformer_layer import TransformerEncoderLayer as L
    M, d, N = 777, 512, 768
    g = torch.Generator(device="cuda").manual_seed(21)
    x = torch.randn(M, d, device="cuda", generator=g) * 1.5 + 0.3
    lw = 1 + 0.2 * torch.randn(d, device="cuda", generator=g)
    lb = 0.1 * torch.randn(d, device="cuda", generator=g)
    W = torch.randn(N, d, device="cuda", generator=g) * 0.05
    b = torch.randn(N, device="cuda", generator=g)
    xb = torch.empty(M, d, dtype=torch.bfloat16, device="cuda")
    mu = torch.empty(M, device="cuda"); rstd = torch.empty(M, device="cuda")
    K.row_stats_cast(x, xb, mu, rstd)
    torch.testing.assert_close(mu, x.mean(1), atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(rstd, (x.var(1, unbiased=False) + 1e-5).rsqrt(), atol=1e-5, rtol=1e-4)
    class _LN:      # stand-in for nn.LayerNorm: the fold reads .weight / .bias
        def __init__(self, w, b_):
            self.weight, self.bias = w, b_
    wg, colsum, dd = L._fold([W], _LN(lw, lb), [b])
    # the one-pass fold kernel (csrc/pack.cu) equals the torch formulation
    wg_t = (W * lw[None, :]).to(torch.bfloat16)
    assert torch.equal(wg, wg_t)
    torch.testing.assert_close(colsum, wg_t.float().sum(1), atol=1e-4, rtol=1e-5)
    torch.testing.assert_close(dd, W @ lb + b, atol=1e-4, rtol=1e-5)
    out = torch.empty(M, N, dtype=torch.float32, device="cuda")
    K.gemm_ln(xb, wg, K.EPI_STORE_F32, out, ln_mu=mu, ln_rstd=rstd, ln_colsum=colsum, bias=dd, cta_group=cg)
    want = torch.nn.functional.linear(torch.nn.functional.layer_norm(x, (d,), lw, lb), W, b)
    assert relerr(out, want) < 8e-3
    # RESID epilogue with statistics + bf16 copy
    gamma = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    y = res.clone()
    part = torch.zeros(((N + 255) // 256) * M * 2, device="cuda")
    yb = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    K.gemm_ln(xb, wg, K.EPI_RESID_F32, y, ln_mu=mu, ln_rstd=rstd, ln_colsum=colsum, bias=dd, gamma=gamma, resid=y,
              stats_out=part, out_bf16=yb, cta_group=cg)
    assert relerr(y, res + gamma * want) < 8e-3
    assert torch.equal(yb, y.bfloat16())
    m2 = torch.empty(M, device="cuda"); r2 = torch.empty(M, device="cuda")
    K.ln_stats_finalize(part, (N + 255) // 256, M, N, 1e-5, m2, r2)
    torch.testing.assert_close(m2, y.mean(1), atol=1e-4, rtol=1e-4)
    torch.testing.assert_close(r2, (y.var(1, unbiased=False) + 1e-5).rsqrt(), atol=1e-4, rtol=1e-3)
    # consumer reduces the partial records itself (no finalize launch): LN(y) W2^T via ln_partial
    W2 = torch.randn(640, N, device="cuda", generator=g) * 0.05
    lw2 = 1 + 0.2 * torch.randn(N, device="cuda", generator=g)
    lb2 = 0.1 * torch.randn(N, device="cuda", generator=g)
    b2 = torch.randn(640, device="cuda", generator=g)
    wg2, cs2, dd2 = L._fold([W2], _LN(lw2, lb2), [b2])
    want2 = torch.nn.functional.linear(torch.nn.functional.layer_norm(yb.float(), (N,), lw2, lb2), W2, b2)
    for epi, dt in ((K.EPI_STORE_F32, torch.float32), (K.EPI_STORE_BF16, torch.bfloat16)):
        o_arr = torch.empty(M, 640, dtype=dt, device="cuda")
        o_par = torch.empty(M, 640, dtype=dt, device="cuda")
        K.gemm_ln(yb, wg2, epi, o_arr, ln_mu=m2, ln_rstd=r2, ln_colsum=cs2, bias=dd2, cta_group=cg)
        K.gemm_ln(yb, wg2, epi, o_par, ln_partial=(part, (N + 255) // 256, N, 1e-5), ln_colsum=cs2, bias=dd2, cta_group=cg)
        assert relerr(o_par, want2) < 1e-2
        assert relerr(o_par, o_arr) < 1e-5


def test_attention_ln_stats(K):
    B, S, H = 2, 70, 4
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv = (torch.randn(B * S, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
    part = torch.zeros(H * B * S * 2, device="cuda")
    out = K.attention(qkv, None, None, B, S, H, ln_stats=part)
    mu = torch.empty(B * S, device="cuda"); rstd = torch.empty(B * S, device="cuda")
    K.ln_stats_finalize(part, H, B * S, D, 1e-5, mu, rstd)
    o = out.float()
    torch.testing.assert_close(mu, o.mean(1), atol=2e-3, rtol=1e-2)      # stats are of the pre-rounding fp32 rows
    torch.testing.assert_close(rstd, (o.var(1, unbiased=False) + 1e-5).rsqrt(), atol=0, rtol=1e-2)


@pytest.mark.parametrize("kind,B,S,H,use_pad", [("text", 3, 17, 4, True), ("text", 2, 72, 4, True), ("image", 3, 197, 24, False),
                                                 ("image", 2, 257, 4, False), ("text", 2, 384, 2, True), ("text", 5, 128, 4, False),
                                                 ("text", 2, 750, 3, True), ("text", 3, 500, 2, False), ("text", 1, 768, 2, True),
                                                 ("text", 2, 385, 2, True)])
def test_attention_tc(K, kind, B, S, H, use_pad):
    """attention with the LUT-form relative-position bias vs a plain fp32 reference on the dense bias.   The shapes cover
    S <= 224, S <= 384 and 384 < S <= 768 (the 10-15 s audio sequences, whose buckets are the 1-D text scheme,
    adapter/audio.py:20-32), with and without padded keys."""
    import numpy as np
    import restated as R
    from one_peace_b200 import relpos
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(S + H)
    qkv = (torch.randn(B * S, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
    if kind == "text":
        bucket = R.make_token_bucket_position(256)[:S, :S]
        codes = relpos.text_codes(S)
        ntab = 514
    else:
        w = int(round((S - 1) ** 0.5))
        bucket = R.make_image_bucket_position(w)
        codes = relpos.image_codes(S, w)
        ntab = (2 * w - 1) ** 2 + 3
    table = torch.randn(ntab, H, device="cuda", generator=g)
    li = relpos.build_lut_index(bucket.numpy(), codes)
    assert li is not None
    lut_idx, crow, ccol = (torch.from_numpy(a).cuda() for a in li)
    rp = K.RelPosBias(lut=K.relpos_lut_build(table, lut_idx), code_row=crow, code_col=ccol)
    dense = table[bucket.cuda()].permute(2, 0, 1)                     # (H,S,S)
    assert torch.equal(rp.lut[:, (crow[:S, None] - ccol[None, :S]).long()], dense)
    kp = None
    if use_pad:
        kp = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
        for b in range(B):
            kp[b, S - 1 - 2 * b:] = 1
    part = torch.zeros(H * B * S * 2, device="cuda")
    lse = torch.empty(B * H * S, device="cuda")
    out = K.attention_tc(qkv, rp, kp, B, S, H, ln_stats=part, lse=lse)
    q, k, v = qkv.float().view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    sc = q @ k.transpose(-1, -2) + dense[None]
    if kp is not None:
        sc = sc.masked_fill(kp.bool()[:, None, None, :], float("-inf"))
    want = (sc.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * S, D)
    assert relerr(out, want) < 8e-3
    # log-sum-exp per (batch, head, query), consumed by the attention backward
    torch.testing.assert_close(lse.view(B, H, S), torch.logsumexp(sc, dim=-1), atol=2e-3, rtol=1e-4)
    mu = torch.empty(B * S, device="cuda"); rstd = torch.empty(B * S, device="cuda")
    K.ln_stats_finalize(part, H, B * S, D, 1e-5, mu, rstd)
    torch.testing.assert_close(mu, out.float().mean(1), atol=2e-3, rtol=1e-2)


@pytest.mark.parametrize("M,d,N", [(136, 1536, 1536), (136, 6144, 1536), (40, 1024, 256), (255, 512, 512)])
def test_gemm_resid_small_m_splitk(K, M, d, N):
    """M <= 256 (a few texts): with a workspace the fp32-residual GEMM splits its K range over the idle SMs and the split
    epilogue kernel finishes it (gemm_bf16 small-M mode); result, bf16 copy and LN statistics must match the plain schedule."""
    g = torch.Generator(device="cuda").manual_seed(M + d)
    a = (torch.randn(M, d, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, d, device="cuda", generator=g) * 0.05).bfloat16()
    mu = torch.randn(M, device="cuda", generator=g) * 0.1
    rs = torch.rand(M, device="cuda", generator=g) + 0.5
    cs = torch.randn(N, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    n_t = (N + 255) // 256
    outs = []
    for use_ws in (False, True):
        y = res.clone()
        yb = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        part = torch.zeros(n_t * M * 2, device="cuda")
        wsb = torch.empty(16 * 256 * N, device="cuda") if use_ws else None          # fp32 [M rounded up to 128, N] slabs, one per piece
        K.gemm_ln(a, w, K.EPI_RESID_F32, y, ln_mu=mu, ln_rstd=rs, ln_colsum=cs, bias=bias, gamma=gamma, resid=y,
                  stats_out=part, out_bf16=yb, workspace=wsb)
        outs.append((y, yb, part))
    want = res + gamma * (rs[:, None] * (a.float() @ w.float().t() - mu[:, None] * cs) + bias)
    for y, yb, part in outs:
        assert relerr(y, want) < 1e-4
        assert torch.equal(yb, y.bfloat16())
    torch.testing.assert_close(outs[1][2].view(n_t, M, 2), outs[0][2].view(n_t, M, 2), atol=2e-2, rtol=1e-4)


@pytest.mark.parametrize("M,d,N", [(136, 1536, 4608), (17, 1024, 768)])
def test_gemm_store_small_m_splitk(K, M, d, N):
    """the q/k/v projection of a small batch (bf16 store epilogue with fused LayerNorm, bias and column scale): with a workspace
    its K range is split over the idle SMs and the split epilogue kernel applies the epilogue; must match the plain schedule."""
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = (torch.randn(M, d, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, d, device="cuda", generator=g) * 0.05).bfloat16()
    mu = torch.randn(M, device="cuda", generator=g) * 0.1
    rs = torch.rand(M, device="cuda", generator=g) + 0.5
    cs = torch.randn(N, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    scale = torch.rand(N, device="cuda", generator=g) + 0.5
    outs = []
    for use_ws in (False, True):
        y = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        wsb = torch.empty(16 * 256 * 1536, device="cuda") if use_ws else None
        K.gemm_ln(a, w, K.EPI_STORE_BF16, y, ln_mu=mu, ln_rstd=rs, ln_colsum=cs, bias=bias, colscale=scale, workspace=wsb)
        outs.append(y)
    want = (rs[:, None] * (a.float() @ w.float().t() - mu[:, None] * cs) + bias) * scale
    for y in outs:
        assert relerr(y, want) < 8e-3
    assert relerr(outs[1], outs[0]) < 8e-3


def test_gemm_resid_m_tail_splitk(K):
    """M = 49 * 256 + 64 rows, N = 1536, K = 3072, with a workspace: a large M keeps the tiled schedule (the workspace only
    serves M <= 256), and the partially filled last row of tiles must match the fp32 reference and the path without it."""
    M, d, N = 49 * 256 + 64, 3072, 1536
    g = torch.Generator(device="cuda").manual_seed(33)
    a = (torch.randn(M, d, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, d, device="cuda", generator=g) * 0.05).bfloat16()
    mu = torch.randn(M, device="cuda", generator=g) * 0.1
    rs = torch.rand(M, device="cuda", generator=g) + 0.5
    cs = torch.randn(N, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    outs = []
    for use_ws in (False, True):
        y = res.clone()
        yb = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        part = torch.zeros(6 * M * 2, device="cuda")
        wsb = torch.empty(16 * 256 * N, device="cuda") if use_ws else None          # fp32 [M rounded up to 128, N] slabs, one per piece
        K.gemm_ln(a, w, K.EPI_RESID_F32, y, ln_mu=mu, ln_rstd=rs, ln_colsum=cs, bias=bias, gamma=gamma, resid=y,
                  stats_out=part, out_bf16=yb, workspace=wsb)
        outs.append((y, yb, part))
    want = res + gamma * (rs[:, None] * (a.float() @ w.float().t() - mu[:, None] * cs) + bias)
    for y, yb, part in outs:
        assert relerr(y, want) < 1e-4
        assert torch.equal(yb, y.bfloat16())
    assert relerr(outs[1][0], outs[0][0]) < 1e-5
    p0 = outs[0][2].view(6, M, 2); p1 = outs[1][2].view(6, M, 2)
    torch.testing.assert_close(p1, p0, atol=2e-2, rtol=1e-4)
    # same GEMM with the A-row statistics given as 96 partial records (the GeGLU -> fc2 hand-over): the GEMM epilogue
    # reduces them per row itself; must equal the run on the finalized (mu, rstd) arrays
    parts, dim = 96, 6144
    rec = torch.rand(parts, M, 2, device="cuda", generator=g)
    rec[..., 0] = (rec[..., 0] - 0.5) * 8
    rec[..., 1] = rec[..., 1] * 400 + 64
    m2 = torch.empty(M, device="cuda"); r2 = torch.empty(M, device="cuda")
    K.ln_stats_finalize(rec.view(-1), parts, M, dim, 1e-5, m2, r2)
    res2 = []
    for kw in (dict(ln_mu=m2, ln_rstd=r2), dict(ln_partial=(rec.view(-1), parts, dim, 1e-5))):
        y = res.clone()
        K.gemm_ln(a, w, K.EPI_RESID_F32, y, ln_colsum=cs, bias=bias, gamma=gamma, resid=y, workspace=torch.empty(16 * 256 * N, device="cuda"), **kw)
        res2.append(y)
    assert relerr(res2[1], res2[0]) < 1e-5


def test_topk10_rows_and_recall_hits(K):
    g = torch.Generator(device="cuda").manual_seed(77)
    sim = torch.randn(37, 1003, device="cuda", generator=g)
    idx, val = K.topk10_rows(sim, want_values=True)
    tv, ti = sim.topk(10, dim=1)
    assert torch.equal(val, tv) and torch.equal(idx.long(), ti)
    # strided rows (a column-sliced view) and a row with fewer than 10 columns
    wide = torch.randn(5, 64, device="cuda", generator=g)
    idx2 = K.topk10_rows(wide[:, :7])
    assert torch.equal(idx2[:, :7].long(), wide[:, :7].topk(7, dim=1).indices) and torch.all(idx2[:, 7:] == -1)
    cand = torch.randint(0, 50, (1003,), device="cuda", generator=g)
    own = torch.randint(0, 50, (37,), device="cuda", generator=g)
    hits = K.recall_hits(idx, cand, own)
    pred = cand[ti]
    want = [int(pred[:, :r].eq(own[:, None]).any(1).sum()) for r in (1, 5, 10)]
    assert hits.tolist() == want


def test_recall_metric_vs_reference_golden(K, golden_dir):
    """metrics/recall.py protocol through the sm_90a kernels vs the eval_log of the reference's own Recall class."""
    import os
    import synth
    from one_peace_b200.metrics import Recall
    for c in torch.load(os.path.join(golden_dir, "recall.pt"), weights_only=False):
        img, txt, img_ids, txt_ids = synth.retrieval_set(c["n_img"], c["cap"], c["d"], c["seed"], c["noise"])
        rec = Recall()
        rec.initialize(txt_ids.cuda(), txt.cuda())
        for lo in range(0, c["n_img"], 16):
            rec.compute(img_ids[lo:lo + 16].cuda(), img[lo:lo + 16].cuda())
        log = rec.merge_results(output_predict=True)
        for k in ("txt_r1", "txt_r5", "txt_r10", "txt_r_mean", "img_r1", "img_r5", "img_r10", "img_r_mean", "r_mean"):
            assert abs(log[k] - c["log"][k]) < 1e-9, (k, log[k], c["log"][k])
        assert log["img_count"] == c["log"]["img_count"] and log["txt_count"] == c["log"]["txt_count"]
        assert log["predict_txt"] == c["log"]["predict_txt"] and log["predict_img"] == c["log"]["predict_img"]


# ----------------------------------------------------------------------------------------------------------------
# pretraining-path kernels (csrc/gather.cu, attention segment / per-sample bias, DCL form of the InfoNCE epilogues)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sdt,odt", [(torch.float32, torch.float32), (torch.float32, torch.bfloat16),
                                     (torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32)])
def test_row_gather_and_scatter_add(K, sdt, odt):
    g = torch.Generator(device="cuda").manual_seed(11)
    n, dim, rows = 57, 264, 91
    src = torch.randn(n, dim, device="cuda", generator=g).to(sdt)
    idx = torch.randint(-1, n, (rows,), device="cuda", generator=g)
    fill = torch.randn(dim, device="cuda", generator=g)
    out = K.row_gather(src, idx, fill=fill, out_dtype=odt)
    want = torch.where((idx >= 0)[:, None], src.float()[idx.clamp_min(0)], fill[None]).to(odt)
    assert torch.equal(out, want)                                       # a pure copy: bit-exact
    out0 = K.row_gather(src, idx, out_dtype=odt)
    assert torch.equal(out0[idx < 0], torch.zeros_like(out0[idx < 0]))
    # strided source view (rows of a wider matrix)
    wide = torch.randn(n, dim + 24, device="cuda", generator=g).to(sdt)
    assert torch.equal(K.row_gather(wide[:, 8:8 + dim], idx.clamp_min(0), out_dtype=sdt), wide[:, 8:8 + dim][idx.clamp_min(0)])
    # adjoint (duplicates accumulate)
    dout = torch.randn(rows, dim, device="cuda", generator=g).to(odt)
    dsrc = torch.zeros(n, dim, device="cuda")
    K.row_scatter_add(dout, idx, dsrc)
    ref = torch.zeros(n, dim, device="cuda").index_add_(0, idx[idx >= 0], dout.float()[idx >= 0])
    torch.testing.assert_close(dsrc, ref, atol=1e-5, rtol=1e-5)


def test_relpos_bias_block_with_ids_and_adjoint(K):
    """bias gather of gather_features (adapter/text.py:96-101) + block-diagonal placement (transformer_encoder.py:148-158)."""
    g = torch.Generator(device="cuda").manual_seed(12)
    H, n_full, B, n1, n2 = 4, 40, 3, 9, 13
    S = n1 + n2
    s_pad = (S + 7) // 8 * 8
    bucket = torch.randint(0, 50, (n_full, n_full), device="cuda", generator=g)
    t1 = torch.randn(50, H, device="cuda", generator=g)
    t2 = torch.randn(50, H, device="cuda", generator=g)
    ids1 = torch.stack([torch.randperm(n_full, device="cuda", generator=g)[:n1].sort().values for _ in range(B)])
    ids1[1, -2:] = -1
    bias = torch.zeros(B, H, S, s_pad, device="cuda")
    K.relpos_bias_block(t1, bucket, ids1, n1, 0, bias, S, H)
    bias_shared = torch.zeros(1, H, S, s_pad, device="cuda")
    K.relpos_bias_block(t2, bucket, None, n2, n1, bias_shared, S, H)
    pos = ids1.masked_fill(ids1.eq(-1), n1 - 1)
    full = t1[bucket].permute(2, 0, 1)[None].expand(B, -1, -1, -1)                                   # (B,H,n_full,n_full)
    want1 = full.gather(2, pos[:, None, :, None].expand(-1, H, -1, n_full)).gather(3, pos[:, None, None, :].expand(-1, H, n1, -1))
    assert torch.equal(bias[:, :, :n1, :n1], want1)
    assert torch.count_nonzero(bias[:, :, n1:]) == 0 and torch.count_nonzero(bias[:, :, :, n1:]) == 0
    assert torch.equal(bias_shared[0, :, n1:S, n1:S], t2[bucket[:n2, :n2]].permute(2, 0, 1))
    dbias = torch.randn(B, H, S, s_pad, device="cuda", generator=g)
    dt = torch.zeros_like(t1)
    K.relpos_bias_block_bwd(dbias, bucket, ids1, n1, 0, dt, S, H)
    tt = t1.clone().requires_grad_(True)
    full = tt[bucket].permute(2, 0, 1)[None].expand(B, -1, -1, -1)
    w = full.gather(2, pos[:, None, :, None].expand(-1, H, -1, n_full)).gather(3, pos[:, None, None, :].expand(-1, H, n1, -1))
    (w * dbias[:, :, :n1, :n1]).sum().backward()
    torch.testing.assert_close(dt, tt.grad, atol=1e-4, rtol=1e-4)


def _attn_ref(qkv, bias, key_pad, B, S, H):
    D = H * 64
    q, k, v = (qkv.float().view(B, S, 3, H, 64)[:, :, i].transpose(1, 2) for i in range(3))
    a = q @ k.transpose(-1, -2)
    if bias is not None:
        a = a + (bias if bias.dim() == 4 else bias[None])[..., :S]
    if key_pad is not None:
        a = a.masked_fill(key_pad.bool()[:, None, None, :], float("-inf"))
    return (torch.softmax(a, -1) @ v).transpose(1, 2).reshape(B * S, D)


def test_attention_per_sample_bias_forward_backward(K):
    """bias_batch_stride form of opb_attention_fwd / _bwd: one (H,S,S_pad) table per sample."""
    g = torch.Generator(device="cuda").manual_seed(13)
    B, S, H = 3, 45, 4
    s_pad = 48
    D = H * 64
    qkv = (torch.randn(B * S, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
    bias = torch.zeros(B, H, S, s_pad, device="cuda")
    bias[..., :S] = torch.randn(B, H, S, S, device="cuda", generator=g)
    pad = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
    pad[1, -5:] = 1
    lse = torch.empty(B * H * S, device="cuda")
    out = K.attention(qkv, bias, pad, B, S, H, lse=lse)
    want = _attn_ref(qkv, bias, pad, B, S, H)
    assert relerr(out, want) < 2e-2
    # backward vs torch autograd
    d_out = (torch.randn(B * S, D, device="cuda", generator=g) * 0.1).bfloat16()
    dqkv = torch.empty_like(qkv)
    dbias = torch.zeros_like(bias)
    K.attention_bwd(qkv, out, d_out, bias, pad, lse, dqkv, dbias, B, S, H, 1.0)
    qf = qkv.float().clone().requires_grad_(True)
    bf = bias.clone().requires_grad_(True)
    (_attn_ref(qf, bf, pad, B, S, H) * d_out.float()).sum().backward()
    assert relerr(dqkv, qf.grad) < 3e-2
    assert relerr(dbias[..., :S], bf.grad[..., :S]) < 3e-2


def test_attention_tc_two_segments(K):
    """'vl' form of the LUT-bias attention: concatenated LUTs, block-diagonal bias (zero across modalities)."""
    import numpy as np
    from one_peace_b200 import relpos
    g = torch.Generator(device="cuda").manual_seed(14)
    B, H, S1, w = 2, 4, 21, 6
    S2 = w * w + 1
    S = S1 + S2
    D = H * 64
    # buckets: text-style (difference) and image-style (2-D) with CLS ids
    b1 = (torch.arange(S1)[:, None] - torch.arange(S1)[None, :] + S1).clone()
    b1[0, :] = 2 * S1 + 1; b1[:, 0] = 2 * S1 + 2; b1[0, 0] = 2 * S1 + 3
    from one_peace_b200.adapter.image import make_image_bucket_position
    nrd = (2 * w - 1) ** 2 + 3
    b2 = make_image_bucket_position(w, nrd)
    t1 = torch.randn(2 * S1 + 4, H, device="cuda", generator=g)
    t2 = torch.randn(nrd, H, device="cuda", generator=g)
    rp = K.build_segmented_lut([(t1, relpos.build_lut_index(b1.numpy(), relpos.text_codes(S1)), S1),
                                (t2, relpos.build_lut_index(b2.numpy(), relpos.image_codes(S2, w)), S2)], "cuda")
    qkv = (torch.randn(B * S, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
    pad = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
    pad[1, S1 - 4:S1] = 1
    out = K.attention_tc(qkv, rp, pad, B, S, H)
    dense = torch.zeros(H, S, S, device="cuda")
    dense[:, :S1, :S1] = t1[b1.cuda()].permute(2, 0, 1)
    dense[:, S1:, S1:] = t2[b2.cuda()].permute(2, 0, 1)
    want = _attn_ref(qkv, dense, pad, B, S, H)
    assert relerr(out, want) < 2e-2


def test_dcl_form_of_one_direction_infonce_forward(K):
    """n_valid / coef form: single-direction label-smoothed NLL over a ragged number of classes
    (compute_dcl_loss, image_text_pretrain_loss.py:187-208)."""
    g = torch.Generator(device="cuda").manual_seed(15)
    nm, nt, d = 37, 101, 256
    stu = torch.nn.functional.normalize(torch.randn(nm, d, device="cuda", generator=g), dim=1)
    tea = torch.nn.functional.normalize(torch.randn(nt, d, device="cuda", generator=g), dim=1)
    tea[:nm] = torch.nn.functional.normalize(stu + 0.4 * tea[:nm], dim=1)
    n8 = (nt + 7) // 8 * 8
    tea_p = torch.zeros(n8, d, device="cuda")
    tea_p[:nt] = tea
    scale = torch.tensor([2.5], device="cuda")
    a3, b3 = K.split_bf16x3([stu, tea_p], [0, 1])
    (lse,), out3, loss, am = K.infonce_forward([(a3, b3)], scale, 0, 0.1, n_valid=nt, rows=True)
    sa = stu.clone().requires_grad_(True)
    sim = 2.5 * sa @ tea.t()
    lp = torch.log_softmax(sim, -1)
    tgt = torch.arange(nm, device="cuda")
    nll = -lp.gather(1, tgt[:, None]).squeeze(1)
    eps_i = 0.1 / (nt - 1)
    want_rows = (1 - 0.1 - eps_i) * nll + eps_i * (-lp.sum(-1))
    torch.testing.assert_close(loss, want_rows.detach(), atol=2e-4, rtol=2e-4)
    torch.testing.assert_close(out3[0], want_rows.detach().mean(), atol=2e-4, rtol=2e-4)
    assert torch.equal(am.long(), sim.argmax(1))
    grad, _ = K.infonce_grad(a3, b3, scale, lse, 0, 0.1, d, n_valid=nt, coef=1.0 / nm)
    want_rows.mean().backward()
    assert relerr(grad, sa.grad) < 2e-2


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("a_mn,b_mn", [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize("M,N,Kd", [(512, 768, 1000), (1536, 1536, 12608), (96, 256, 77), (4608, 1536, 333)])
def test_gemm_mn_major_operands(K, cg, a_mn, b_mn, M, N, Kd):
    """opb_gemm_bf16_t: contraction over the ROWS of [K, M] / [K, N] matrices without transposed copies (dW = dY^T X)."""
    g = torch.Generator(device="cuda").manual_seed(M + N + Kd)
    if not (a_mn and b_mn) and Kd % 8:
        Kd = Kd // 8 * 8                      # a K-major operand needs an 8-element row pitch
    A = (torch.randn(M, Kd, device="cuda", generator=g) * 0.5).bfloat16()
    B = (torch.randn(N, Kd, device="cuda", generator=g) * 0.1).bfloat16()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    out = torch.empty(M, N, dtype=torch.float32, device="cuda")
    K.gemm_t(a, b, K.EPI_STORE_F32, out, a_mn=a_mn, b_mn=b_mn, cta_group=cg)
    want = A.float() @ B.float().t()
    assert relerr(out, want) < 2e-5
    # strided views (columns of a wider matrix), bf16 output
    wide_b = torch.zeros(b.shape[0], b.shape[1] + 64, dtype=torch.bfloat16, device="cuda")
    wide_b[:, 32:32 + b.shape[1]] = b
    out16 = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    K.gemm_t(a, wide_b[:, 32:32 + b.shape[1]], K.EPI_STORE_BF16, out16, a_mn=a_mn, b_mn=b_mn, cta_group=cg)
    assert relerr(out16, want) < 6e-3
