"""CPU: the fp64 reference and per-element bounds of tests/kernel_ref.py.  A correct kernel, emulated here in fp32 (bf16
operands, fp32 matmul, the epilogue and the LayerNorm statistics in fp32 as the kernel evaluates them), must pass the
bounds; each of the subtle mistakes a GEMM or InfoNCE kernel can make must fail them."""
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
