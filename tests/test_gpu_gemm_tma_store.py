"""GPU: the bf16 GEMM epilogues written through shared memory and TMA bulk stores (gemm_bf16_tma_out_kernel) give the same
bits as the direct-store kernel.

A call takes the TMA-store kernel when its output is 16-byte aligned with a 16-byte multiple row pitch (and it is a single
group without split-K or row remapping); otherwise it keeps the direct-store kernel.  Both evaluate every value in the same
registers in the same order, so the same call on an aligned output and on a misaligned one (4 bytes past a 16-byte boundary,
or a row pitch of N + 2) must agree bit for bit, GeGLU's statistics records included.  Every output sits in a NaN canary
buffer with spare rows and a wider pitch: the TMA stores clip rows >= M and columns >= N through the tensor map and must
not write anything else."""
import zlib

import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


def bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def out_buffer(M, n, layout):
    """(view, canary buffer): `aligned` takes the TMA-store path, `offset` (2 elements = 4 bytes past a 16-byte boundary) and
    `pitch` (row pitch n + 2) the direct-store path"""
    if layout == "aligned":
        return R.canary_out((M, n), ldo_extra=8, rows_before=1, rows_after=3, dtype=BF16)
    if layout == "pitch":
        return R.canary_out((M, n), ldo_extra=2, rows_before=1, rows_after=3, dtype=BF16)
    buf = torch.full((M + 4, n + 8), float("nan"), dtype=BF16, device="cuda")
    return buf[1:1 + M, 2:2 + n], buf


LAYOUTS = ("aligned", "offset", "pitch")


def assert_same_bits(runs, what):
    (out0, _), *rest = runs
    for (out, _), layout in zip(rest, LAYOUTS[1:]):
        assert torch.equal(bits(out), bits(out0)), f"{what}: the {layout} output differs from the TMA-stored one"


def check_layouts(K, a, w, epi, kw):
    """the same gemm_ln call on the three output layouts: canaries intact, outputs (and GeGLU records) bit-identical"""
    M, N = a.shape[0], w.shape[0]
    n_out = N // 2 if epi == K.EPI_GEGLU_BF16 else N
    outs, stats = [], []
    for layout in LAYOUTS:
        out, buf = out_buffer(M, n_out, layout)
        ekw = dict(kw)
        if epi == K.EPI_GEGLU_BF16:
            ekw["stats_out"] = torch.full((N // 128, M, 2), float("nan"), device="cuda")
            stats.append(ekw["stats_out"])
        K.gemm_ln(a, w, epi, out, **ekw)
        R.assert_canary(buf, out, what=f"{layout} output")
        outs.append((out, buf))
    assert_same_bits(outs, "output")
    for st in stats[1:]:
        assert torch.equal(bits(st), bits(stats[0])), "GeGLU statistics records differ between the store paths"


def operands(M, N, Kd, g):
    x = torch.randn(M, Kd, device="cuda", generator=g) * (1 + 0.3 * torch.rand(M, 1, device="cuda", generator=g))
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).bfloat16()
    return x, w


def epilogue_case(K, case, x, w, g):
    N, Kd = w.shape
    bias = torch.randn(N, device="cuda", generator=g)
    cs = torch.rand(N, device="cuda", generator=g) + 0.5
    colsum = w.float().sum(1)
    if case == "store_bf16_ln_bias_cs":
        mu, rstd = x.mean(1), (x.var(1, unbiased=False) + 1e-5).rsqrt()
        return K.EPI_STORE_BF16, dict(ln_mu=mu, ln_rstd=rstd, ln_colsum=colsum, bias=bias, colscale=cs)
    if case == "gelu_bf16":
        return K.EPI_GELU_BF16, dict(bias=bias, colscale=cs)
    parts = 8                                            # geglu_ln: LayerNorm from partial (sum, sum of squares) records
    s = x.view(x.shape[0], parts, -1)
    rec = torch.stack([s.sum(2), (s * s).sum(2)], 2).transpose(0, 1).contiguous()
    return K.EPI_GEGLU_BF16, dict(ln_partial=(rec, parts, Kd, 1e-5), ln_colsum=colsum, bias=bias)


# the schedules of test_gpu_gemm_contract.py: one tile, 420 tiles, M % 128 = 1 / 64 / 127, N % 256 = 248 / 8 / 128
SCHEDULES = {
    "one_tile": (100, 248, 1000),
    "many_tiles": (1727, 7680, 1544),
    "m_tail_1": (257, 504, 1000),
    "m_tail_64": (320, 264, 1544),
    "m_tail_127": (383, 384, 1000),
}
CASES = ["store_bf16_ln_bias_cs", "gelu_bf16", "geglu_ln"]


@pytest.mark.parametrize("sched", list(SCHEDULES))
@pytest.mark.parametrize("case", CASES)
def test_store_paths_agree(K, case, sched):
    M, N, Kd = SCHEDULES[sched]
    if case == "geglu_ln":
        N = (N + 255) // 256 * 256          # GeGLU works on whole gate / linear tile pairs
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"tma/{case}/{sched}".encode()))
    x, w = operands(M, N, Kd, g)
    epi, kw = epilogue_case(K, case, x, w, g)
    check_layouts(K, x.bfloat16(), w, epi, kw)


@pytest.mark.parametrize("case,N", [("store_bf16_ln_bias_cs", 4608), ("gelu_bf16", 4608), ("geglu_ln", 2 * 6144)])
def test_store_paths_agree_encoder_shapes(K, case, N):
    """the QKV and GeGLU launches of the 4B vision encoder: 64 images x 197 tokens, d = 1536"""
    g = torch.Generator(device="cuda").manual_seed(N + len(case))
    x, w = operands(12608, N, 1536, g)
    epi, kw = epilogue_case(K, case, x, w, g)
    check_layouts(K, x.bfloat16(), w, epi, kw)


@pytest.mark.parametrize("M,N,Kd,a_mn,b_mn", [(1536, 1536, 12608, True, True), (200, 264, 1001, True, True),
                                              (264, 200, 1000, True, False), (383, 504, 1000, False, True)])
def test_store_paths_agree_mn_major(K, M, N, Kd, a_mn, b_mn):
    """gemm_t: the bf16 weight gradient dW = dY^T X and the other MN-major operand forms"""
    g = torch.Generator(device="cuda").manual_seed(M * 3 + N + Kd)
    A = (torch.randn(M, Kd, device="cuda", generator=g) * 0.5).bfloat16()
    B = (torch.randn(N, Kd, device="cuda", generator=g) * 0.1).bfloat16()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    bias = torch.randn(N, device="cuda", generator=g)
    outs = []
    for layout in LAYOUTS:
        out, buf = out_buffer(M, N, layout)
        K.gemm_t(a, b, K.EPI_STORE_BF16, out, a_mn=a_mn, b_mn=b_mn, bias=bias)
        R.assert_canary(buf, out, what=f"{layout} output")
        outs.append((out, buf))
    assert_same_bits(outs, "gemm_t output")


def gemm_kernels(launch):
    """names of the GEMM kernels one call launches"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        launch()
        torch.cuda.synchronize()
    return {name for name in (e.key for e in prof.key_averages()) if "gemm_bf16" in name or "gemm_split" in name}


def test_store_path_selection(K):
    """which kernel a call takes: the TMA-store one only for bf16 epilogues on an aligned plain output"""
    g = torch.Generator(device="cuda").manual_seed(7)
    M, N, Kd = 300, 512, 256
    x, w = operands(M, N, Kd, g)
    a = x.bfloat16()

    def takes_tma(launch):
        names = gemm_kernels(launch)
        assert names, "no GEMM kernel seen by the profiler"
        tma = any("gemm_bf16_tma_out_kernel" in n for n in names)
        assert tma != any("gemm_bf16_kernel" in n for n in names), names
        return tma

    for layout, want in zip(LAYOUTS, (True, False, False)):
        out, _ = out_buffer(M, N, layout)
        assert takes_tma(lambda: K.gemm_ln(a, w, K.EPI_STORE_BF16, out)) == want, layout
        out, _ = out_buffer(M, N // 2, layout)
        assert takes_tma(lambda: K.gemm_ln(a, w, K.EPI_GEGLU_BF16, out)) == want, f"geglu {layout}"
    out, _ = out_buffer(M, N, "aligned")
    assert takes_tma(lambda: K.gemm_t(a, w, K.EPI_STORE_BF16, out))
    # fp32 outputs, row remapping and the small-M split-K schedule keep the direct stores
    f32 = torch.empty(M, N, device="cuda")
    assert not takes_tma(lambda: K.gemm_ln(a, w, K.EPI_STORE_F32, f32))
    remap = torch.empty(M + 3, N, dtype=BF16, device="cuda")
    assert not takes_tma(lambda: K.gemm_ln(a, w, K.EPI_STORE_BF16, remap, out_group=100, out_group_stride=101,
                                           out_row_offset=1))
    small = torch.empty(17, 1536, dtype=BF16, device="cuda")
    w2 = (torch.randn(1536, 1536, device="cuda", generator=g) * 0.05).bfloat16()
    a2 = torch.randn(17, 1536, device="cuda", generator=g).bfloat16()
    ws = torch.empty(16 << 20 >> 2, device="cuda")
    names = gemm_kernels(lambda: K.gemm_ln(a2, w2, K.EPI_STORE_BF16, small, workspace=ws))
    assert any("gemm_split_epilogue_kernel" in n for n in names) and not any("tma_out" in n for n in names), names
