"""GPU: the residual GEMM (EPI_RESID_F32) reads a batch of residual values before it stores the outputs of that batch.  So
it accepts a residual that overlaps an output only as the in-place update (resid is the fp32 output, same pitch, no
broadcast period), refuses every other overlap before launching anything, and in place gives the same bits as with a
separate residual buffer."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M, N, KD = 300, 768, 192     # 3 row panels (the last one partial) x 3 column tiles


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


def bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


@pytest.fixture(scope="module")
def case():
    g = torch.Generator(device="cuda").manual_seed(61)
    a = torch.randn(M, KD, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, KD, device="cuda", generator=g) * 0.05).bfloat16()
    vecs = dict(bias=torch.randn(N, device="cuda", generator=g), gamma=torch.randn(N, device="cuda", generator=g))
    res = torch.randn(M, N, device="cuda", generator=g)
    return a, w, vecs, res


def test_in_place_matches_separate_residual(K, case):
    a, w, vecs, res = case
    n_t = (N + 255) // 256
    outs = []
    for in_place in (False, True):
        y = res.clone() if in_place else torch.full((M, N), float("nan"), device="cuda")
        yb = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        st = torch.empty(n_t * M * 2, device="cuda")
        K.gemm_ln(a, w, K.EPI_RESID_F32, y, resid=y if in_place else res, stats_out=st, out_bf16=yb, **vecs)
        outs.append((y, yb, st))
    for sep, inp in zip(*outs):
        assert torch.equal(bits(sep), bits(inp))


def test_overlapping_residual_is_refused(K, case):
    a, w, vecs, res = case
    buf = torch.zeros(M + 1, 2 * N, device="cuda")
    out = buf[:M, :N]
    bad = {
        "shifted by a row": dict(resid=buf[1:M + 1, :N]),
        "shifted by 8 columns": dict(resid=buf[:M, 8:N + 8]),
        "same start, other pitch": dict(resid=buf.view(-1)[:M * N].view(M, N)),
        "broadcast period": dict(resid=out, resid_period=M // 2),
    }
    for what, kw in bad.items():
        with pytest.raises(RuntimeError, match="opb_gemm_bf16"):
            K.gemm(a, w, K.EPI_RESID_F32, out, **vecs, **kw)
        assert torch.count_nonzero(buf) == 0, f"{what}: refused call wrote"
    with pytest.raises(RuntimeError, match="opb_gemm_bf16_ex"):   # the bf16 copy written over the residual
        K.gemm_ln(a, w, K.EPI_RESID_F32, out, resid=res, out_bf16=res.view(torch.bfloat16)[:, :N], **vecs)
    assert torch.count_nonzero(buf) == 0
    # a residual apart from the outputs is accepted, also right behind them in the same allocation
    big = torch.zeros(2 * M, N, device="cuda")
    K.gemm(a, w, K.EPI_RESID_F32, big[:M], resid=big[M:], **vecs)
    want = (a.float() @ w.float().t() + vecs["bias"]) * vecs["gamma"]
    torch.testing.assert_close(big[:M], want, rtol=1e-4, atol=1e-4)
