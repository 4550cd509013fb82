"""GPU: the residual GEMM epilogue (EPI_RESID_F32) that loads its residual into the stage ring with TMA and stores the fp32
result and the bf16 copy with TMA (gemm_bf16_resid_tma_kernel) gives the same bits as the direct-store kernel.

A call takes the ring kernel when the residual, the fp32 output and the bf16 copy are 16-byte aligned with 16-byte multiple
row pitches (and it is a single group without split-K, row remapping or a residual period); otherwise it keeps
gemm_bf16_kernel.  Both evaluate every value with the same operations in the same order, so the same call with its fp32
output 8 bytes past a 16-byte boundary (the direct kernel, which stores float2 pairs) must agree bit for bit with the
aligned one: the output, the bf16 copy and the per-256-column statistics records.  Every output sits in a NaN canary buffer with spare rows and a wider pitch:
the TMA stores clip rows >= M and columns >= N through the tensor maps and must not write anything else."""
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


def f32_out(M, N, aligned):
    """(view, canary buffer): `aligned` takes the ring kernel, otherwise the view starts 8 bytes past a 16-byte boundary"""
    if aligned:
        return R.canary_out((M, N), ldo_extra=8, rows_before=1, rows_after=3)
    buf = torch.full((M + 4, N + 8), float("nan"), device="cuda")
    return buf[1:1 + M, 2:2 + N], buf


def operands(M, N, Kd, g):
    x = torch.randn(M, Kd, device="cuda", generator=g) * (1 + 0.3 * torch.rand(M, 1, device="cuda", generator=g))
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).bfloat16()
    res = torch.randn(M, N, device="cuda", generator=g) * 2
    return x, w, res


def epilogue_args(case, x, w, g):
    """the epilogue operands of `case`, and whether it writes the bf16 copy"""
    M, Kd = x.shape
    N = w.shape[0]
    kw = {}
    if case in ("full_ln_partial", "ln_mu"):
        kw["ln_colsum"] = w.float().sum(1)
        if case == "ln_mu":
            kw.update(ln_mu=x.mean(1), ln_rstd=(x.var(1, unbiased=False) + 1e-5).rsqrt())
        else:
            parts = 8
            s = x.view(M, parts, -1)
            rec = torch.stack([s.sum(2), (s * s).sum(2)], 2).transpose(0, 1).contiguous()
            kw["ln_partial"] = (rec, parts, Kd, 1e-5)
    if case != "bare":
        kw["bias"] = torch.randn(N, device="cuda", generator=g)
    if case in ("full_ln_partial", "ln_mu", "bias_gamma_no_copy"):
        kw["gamma"] = torch.rand(N, device="cuda", generator=g) * 0.2 + 0.05
    return kw, case not in ("bare", "bias_gamma_no_copy")


def run(K, a, w, res, kw, with_copy, aligned, in_place):
    M, N = a.shape[0], w.shape[0]
    out, buf = f32_out(M, N, aligned)
    if in_place:
        out.copy_(res)
    copy, copy_buf = R.canary_out((M, N), ldo_extra=8, rows_before=2, rows_after=1, dtype=BF16) if with_copy else (None, None)
    stats = torch.full(((N + 255) // 256, M, 2), float("nan"), device="cuda")
    K.gemm_ln(a, w, K.EPI_RESID_F32, out, resid=out if in_place else res, out_bf16=copy, stats_out=stats, **kw)
    R.assert_canary(buf, out, what="fp32 output")
    if with_copy:
        R.assert_canary(copy_buf, copy, what="bf16 copy")
    assert torch.isfinite(stats).all(), "statistics records not written"
    return out, copy, stats


def check_paths_agree(K, a, w, res, kw, with_copy, in_place):
    ring = run(K, a, w, res, kw, with_copy, True, in_place)
    direct = run(K, a, w, res, kw, with_copy, False, in_place)
    for what, x, y in zip(("fp32 output", "bf16 copy", "statistics records"), ring, direct):
        if x is not None:
            assert torch.equal(bits(x), bits(y)), f"{what}: the ring kernel differs from the direct-store kernel"


# the schedules of test_gpu_gemm_contract.py: one tile, 420 tiles, M % 128 = 1 / 64 / 127, N % 256 = 248 / 8 / 128
SCHEDULES = {
    "one_tile": (100, 248, 1000),
    "many_tiles": (1727, 7680, 1544),
    "m_tail_1": (257, 504, 1000),
    "m_tail_64": (320, 264, 1544),
    "m_tail_127": (383, 384, 1000),
}


@pytest.mark.parametrize("in_place", [False, True], ids=["separate", "in_place"])
@pytest.mark.parametrize("sched", list(SCHEDULES))
def test_resid_paths_agree(K, sched, in_place):
    M, N, Kd = SCHEDULES[sched]
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"resid_tma/{sched}/{in_place}".encode()))
    x, w, res = operands(M, N, Kd, g)
    kw, with_copy = epilogue_args("full_ln_partial", x, w, g)
    check_paths_agree(K, x.bfloat16(), w, res, kw, with_copy, in_place)


@pytest.mark.parametrize("case", ["ln_mu", "bare", "bias_gamma_no_copy"])
def test_resid_paths_agree_operand_sets(K, case):
    """with and without the fused LayerNorm (precomputed statistics or none), bias, LayerScale and the bf16 copy"""
    M, N, Kd = SCHEDULES["m_tail_64"]
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"resid_tma/{case}".encode()))
    x, w, res = operands(M, N, Kd, g)
    kw, with_copy = epilogue_args(case, x, w, g)
    for in_place in (False, True):
        check_paths_agree(K, x.bfloat16(), w, res, kw, with_copy, in_place)


@pytest.mark.parametrize("Kd", [1536, 6144], ids=["out_proj", "fc2"])
def test_resid_paths_agree_encoder_shapes(K, Kd):
    """the out_proj and fc2 launches of the 4B vision encoder: 64 images x 197 tokens, d = 1536, updated in place"""
    g = torch.Generator(device="cuda").manual_seed(Kd)
    x, w, res = operands(12608, 1536, Kd, g)
    kw, with_copy = epilogue_args("full_ln_partial", x, w, g)
    check_paths_agree(K, x.bfloat16(), w, res, kw, with_copy, in_place=True)


def gemm_kernels(launch):
    """names of the GEMM kernels one call launches"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        launch()
        torch.cuda.synchronize()
    return {name for name in (e.key for e in prof.key_averages()) if "gemm_bf16" in name or "gemm_split" in name}


def test_resid_path_selection(K):
    """which kernel a residual call takes: the ring kernel only for aligned plain operands without split-K or remapping"""
    g = torch.Generator(device="cuda").manual_seed(11)
    M, N, Kd = 300, 512, 256
    x, w, res = operands(M, N, Kd, g)
    a = x.bfloat16()
    vecs = dict(bias=torch.randn(N, device="cuda", generator=g), gamma=torch.randn(N, device="cuda", generator=g))

    def takes_ring(launch):
        names = gemm_kernels(launch)
        assert names, "no GEMM kernel seen by the profiler"
        ring = any("gemm_bf16_resid_tma_kernel" in n for n in names)
        assert ring != any("gemm_bf16_kernel" in n for n in names), names
        return ring

    out, _ = f32_out(M, N, True)
    copy = torch.empty(M, N, dtype=BF16, device="cuda")
    assert takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, out, resid=res, out_bf16=copy, **vecs))
    assert takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, out, resid=out, **vecs))
    # no residual, a misaligned output, residual or bf16 copy, row remapping and a residual period keep the direct stores
    assert not takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, out, **vecs))
    off, _ = f32_out(M, N, False)
    assert not takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, off, resid=res, **vecs))
    res_off, _ = f32_out(M, N, False)
    res_off.copy_(res)
    assert not takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, out, resid=res_off, **vecs))
    copy_buf = torch.empty(M, N + 8, dtype=BF16, device="cuda")
    assert not takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, out, resid=res, out_bf16=copy_buf[:, 2:2 + N], **vecs))
    remap = torch.empty(M + 3, N, device="cuda")
    res_remap = torch.randn(M + 3, N, device="cuda", generator=g)
    assert not takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, remap, resid=res_remap, out_group=100,
                                            out_group_stride=101, out_row_offset=1, **vecs))
    assert not takes_ring(lambda: K.gemm_ln(a, w, K.EPI_RESID_F32, out, resid=res[:100], resid_period=100, **vecs))
    # the small-M split-K schedule
    small = torch.empty(17, 1536, device="cuda")
    w2 = (torch.randn(1536, 1536, device="cuda", generator=g) * 0.05).bfloat16()
    a2 = torch.randn(17, 1536, device="cuda", generator=g).bfloat16()
    ws = torch.empty(16 << 20 >> 2, device="cuda")
    names = gemm_kernels(lambda: K.gemm_ln(a2, w2, K.EPI_RESID_F32, small, resid=torch.randn_like(small), workspace=ws))
    assert any("gemm_split_epilogue_kernel" in n for n in names) and not any("resid_tma" in n for n in names), names
