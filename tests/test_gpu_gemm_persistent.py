"""GPU: the persistent GEMM schedule, where one CTA runs many output tiles in turn, at sizes with several times more tiles
than SMs and an odd number of 128-row panels.  The fused-LayerNorm epilogues take their row statistics and column vectors
from shared memory staged for each tile, so a wrong tile hand-over shows up as wrong rows or columns here."""
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


def partial_records(x, width=256):
    """[parts, M, 2] (sum, sum of squares) records of 256-column slices of x, and the (mu, rstd) they reduce to."""
    M, d = x.shape
    s = x.view(M, d // width, width)
    part = torch.stack([s.sum(2), (s * s).sum(2)], dim=2).transpose(0, 1).contiguous()
    mu = x.mean(1)
    rstd = (x.var(1, unbiased=False) + 1e-5).rsqrt()
    return part, mu, rstd


def test_geglu_ln_partial_many_tiles(K):
    M, d, F = 3900, 512, 3072          # 31 row panels x 24 column tiles
    g = torch.Generator(device="cuda").manual_seed(31)
    x = torch.randn(M, d, device="cuda", generator=g) * 1.3 + 0.2
    part, mu, rstd = partial_records(x)
    xb = x.bfloat16()
    w01 = (torch.randn(2 * F, d, device="cuda", generator=g) * 0.05).bfloat16()
    colsum = torch.randn(2 * F, device="cuda", generator=g)
    bias = torch.randn(2 * F, device="cuda", generator=g)
    u = torch.empty(M, F, dtype=torch.bfloat16, device="cuda")
    stats = torch.full((2 * (2 * F // 256), M, 2), float("nan"), device="cuda")
    K.gemm_ln(xb, w01, K.EPI_GEGLU_BF16, u, ln_partial=(part, d // 256, d, 1e-5), ln_colsum=colsum, bias=bias,
              stats_out=stats)
    z = rstd[:, None] * (xb.float() @ w01.float().t() - mu[:, None] * colsum) + bias
    z = z.view(M, 2 * F // 256, 2, 128)       # packed weight: every 256 rows are 128 gate rows, then 128 linear rows
    want = (torch.nn.functional.gelu(z[:, :, 0]) * z[:, :, 1]).reshape(M, F)
    assert relerr(u, want) < 6e-3
    wt = want.view(M, F // 128, 128)
    torch.testing.assert_close(stats[0::2, :, 0], wt.sum(2).t(), atol=0.05, rtol=1e-2)
    torch.testing.assert_close(stats[0::2, :, 1], (wt * wt).sum(2).t(), atol=0.05, rtol=1e-2)
    assert torch.all(stats[1::2] == 0)
    u2 = torch.empty_like(u)
    K.gemm_ln(xb, w01, K.EPI_GEGLU_BF16, u2, ln_partial=(part, d // 256, d, 1e-5), ln_colsum=colsum, bias=bias)
    assert torch.equal(u, u2)


def test_resid_in_place_ln_partial_many_tiles(K):
    M, d, N = 12608, 768, 1536         # 99 row panels x 6 column tiles
    g = torch.Generator(device="cuda").manual_seed(32)
    x = torch.randn(M, d, device="cuda", generator=g) * 0.8 - 0.1
    part, mu, rstd = partial_records(x)
    xb = x.bfloat16()
    w = (torch.randn(N, d, device="cuda", generator=g) * 0.05).bfloat16()
    colsum = torch.randn(N, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    y = res.clone()
    yb = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    stats = torch.full((N // 256, M, 2), float("nan"), device="cuda")
    K.gemm_ln(xb, w, K.EPI_RESID_F32, y, ln_partial=(part, d // 256, d, 1e-5), ln_colsum=colsum, bias=bias, gamma=gamma,
              resid=y, stats_out=stats, out_bf16=yb)
    want = res + gamma * (rstd[:, None] * (xb.float() @ w.float().t() - mu[:, None] * colsum) + bias)
    assert relerr(y, want) < 1e-4
    assert torch.equal(yb, y.bfloat16())
    yt = y.view(M, N // 256, 256)
    torch.testing.assert_close(stats[:, :, 0], yt.sum(2).t(), atol=1e-2, rtol=1e-4)
    torch.testing.assert_close(stats[:, :, 1], (yt * yt).sum(2).t(), atol=1e-2, rtol=1e-4)
