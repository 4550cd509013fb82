"""GPU: the contract of the wgmma GEMM (csrc/gemm_wgmma.cu) for every epilogue and schedule, element by element against the
fp64 reference of tests/kernel_ref.py (|err| <= tau * mag + extra + u_out * |ref|, tau = 2^-16).

Every case writes into NaN-canary buffers (spare rows around the output, a row pitch wider than the output), so a store
outside the logical output or a skipped store shows up, and runs twice: the two runs must be bit-identical.  Covered:
the epilogues on a single tile, on a persistent schedule with several tiles per CTA and an odd number of row panels, on
row and column tails and on K tails; the small-M split-K schedule at the shapes of the 4B text stack (QKV, out_proj and
fc2 with their partial-record LayerNorm statistics) and its fallbacks; the row remap; MN-major operands."""
import zlib

import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
TAU = R.TAU
BF16, F32 = torch.bfloat16, torch.float32


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def ratios():
    """largest fraction of the bound used, per epilogue family (printed at the end of the module; run with -s to see it)"""
    seen = {}
    yield seen
    for k in sorted(seen):
        print(f"bound used: {k:<28s} {seen[k]:.3g}")


def note(ratios, family, r):
    ratios[family] = max(ratios.get(family, 0.0), r)


def bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def twice(launch):
    """launch() -> {name: (view, buffer)} on fresh buffers; run it twice, the buffers must match bit for bit"""
    r1, r2 = launch(), launch()
    for name in r1:
        assert torch.equal(bits(r1[name][1]), bits(r2[name][1])), f"{name}: two launches differ"
    return r1


def records(x, parts):
    """[parts, M, 2] (sum, sum of squares) records of equal column slices of the fp32 rows x"""
    s = x.view(x.shape[0], parts, -1)
    return torch.stack([s.sum(2), (s * s).sum(2)], 2).transpose(0, 1).contiguous()


def rows_fp32(M, Kd, g, spread=0.3):
    """fp32 rows whose scale and offset vary from row to row (so every row has its own LayerNorm statistics)"""
    return (torch.randn(M, Kd, device="cuda", generator=g) * (1 + spread * torch.rand(M, 1, device="cuda", generator=g))
            + spread * torch.randn(M, 1, device="cuda", generator=g))


def canary(shape, dtype):
    return R.canary_out(shape, ldo_extra=8, rows_before=1, rows_after=3, dtype=dtype)


def nan_full(shape):
    return torch.full(shape, float("nan"), device="cuda")


# --------------------------------------------------------------------------------------------------------------------
# epilogues x schedules
# --------------------------------------------------------------------------------------------------------------------
SCHEDULES = {
    "one_tile": (100, 248, 1000),          # M, N, K: one 128 x 256 tile, column tail, partial last k-block
    "many_tiles": (1727, 7680, 1544),      # 14 row panels (not a multiple of the band of 8) x 30 column tiles: 420 tiles
    "m_tail_1": (257, 504, 1000),          # M % 128 = 1, N % 256 = 248
    "m_tail_64": (320, 264, 1544),         # M % 128 = 64, N % 256 = 8
    "m_tail_127": (383, 384, 1000),        # M % 128 = 127, N % 256 = 128
}
EPILOGUES = ["store_bf16", "store_bf16_ln_bias_cs", "store_f32", "gelu_bf16", "resid_in_place", "resid_separate", "geglu_ln"]


@pytest.mark.parametrize("sched", list(SCHEDULES))
@pytest.mark.parametrize("case", EPILOGUES)
def test_epilogue_schedule(K, ratios, case, sched):
    M, N, Kd = SCHEDULES[sched]
    if case == "geglu_ln":
        N = (N + 255) // 256 * 256          # GeGLU works on whole gate / linear tile pairs
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"{case}/{sched}".encode()))
    x = rows_fp32(M, Kd, g)
    a = x.bfloat16()
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    cs = torch.rand(N, device="cuda", generator=g) + 0.5
    gamma = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    colsum = w.float().sum(1)
    parts = 8
    ln_part = (records(x, parts), parts, Kd, 1e-5)
    mu, rstd = x.mean(1), (x.var(1, unbiased=False) + 1e-5).rsqrt()
    n_rec = (N + 255) // 256

    if case == "store_bf16":
        epi, dt, kw, rkw = K.EPI_STORE_BF16, BF16, {}, {}
    elif case == "store_bf16_ln_bias_cs":
        kw = dict(ln_mu=mu, ln_rstd=rstd, ln_colsum=colsum, bias=bias, colscale=cs)
        epi, dt, rkw = K.EPI_STORE_BF16, BF16, kw
    elif case == "store_f32":
        epi, dt, kw, rkw = K.EPI_STORE_F32, F32, dict(bias=bias), dict(bias=bias)
    elif case == "gelu_bf16":
        epi, dt, kw = K.EPI_GELU_BF16, BF16, dict(bias=bias, colscale=cs)
        rkw = kw
    elif case == "resid_in_place":
        epi, dt = K.EPI_RESID_F32, F32
        kw = dict(ln_partial=ln_part, ln_colsum=colsum, bias=bias, gamma=gamma)
        rkw = dict(kw, resid=res, stats=True)
    elif case == "resid_separate":
        epi, dt = K.EPI_RESID_F32, F32
        kw = dict(bias=bias, resid=res)
        rkw = dict(kw, stats=True)
    else:
        epi, dt = K.EPI_GEGLU_BF16, BF16
        kw = dict(ln_partial=ln_part, ln_colsum=colsum, bias=bias)
        rkw = dict(kw, stats=True)
        n_rec = N // 128
    n_out = N // 2 if epi == K.EPI_GEGLU_BF16 else N

    def launch():
        out, buf = canary((M, n_out), dt)
        bufs = {"out": (out, buf)}
        ekw = dict(kw)
        if case == "resid_in_place":
            out.copy_(res)
            ekw["resid"] = out
        if epi in (K.EPI_RESID_F32, K.EPI_GEGLU_BF16):
            st = nan_full((n_rec, M, 2))
            ekw["stats_out"] = st
            bufs["stats"] = (st, st)
        if epi == K.EPI_RESID_F32:
            ob, bb = canary((M, N), BF16)
            ekw["out_bf16"] = ob
            bufs["out_bf16"] = (ob, bb)
        K.gemm_ln(a, w, epi, out, **ekw)
        return bufs

    got = twice(launch)
    ref = R.gemm_ref(a, w, epi, **rkw)
    out, buf = got["out"]
    R.assert_canary(buf, out)
    note(ratios, case, R.assert_within(out, ref.y, ref.mag, TAU, dt, extra=ref.extra))
    if "stats" in got:
        note(ratios, case + " stats", R.assert_within(got["stats"][0], ref.stats, ref.stats_mag, TAU, F32,
                                                      extra=ref.stats_extra, what="statistics records"))
    if "out_bf16" in got:
        ob, bb = got["out_bf16"]
        R.assert_canary(bb, ob, what="bf16 copy")
        assert torch.equal(ob, out.bfloat16())


# --------------------------------------------------------------------------------------------------------------------
# small-M split-K at the 4B text-stack shapes
# --------------------------------------------------------------------------------------------------------------------
D, FFN, HEADS = 1536, 6144, 24


def layer_case(layer, M, g):
    """operands of one encoder GEMM as forward_rows_fused issues it for M text rows"""
    if layer == "qkv":          # LayerNorm of the residual stream from the previous fc2's 6 records; q pre-scaled
        x = rows_fp32(M, D, g)
        rec, parts, dim, n = records(x, D // 256), D // 256, D, 3 * D
        epi = 0
    elif layer == "out_proj":   # sub-LayerNorm of the attention output from its 24 per-head records
        x = rows_fp32(M, D, g, spread=0.1) * 0.3
        rec, parts, dim, n = records(x, HEADS), HEADS, D, D
        epi = 2
    else:                       # fc2: sub-LayerNorm of the GeGLU output, 96 records, every second one zero
        x = rows_fp32(M, FFN, g, spread=0.2) * 0.5
        r = records(x, FFN // 128)
        rec = torch.stack([r, torch.zeros_like(r)], 1).reshape(FFN // 64, M, 2).contiguous()
        parts, dim, n = FFN // 64, FFN, D
        epi = 2
    kd = x.shape[1]
    w = (torch.randn(n, kd, device="cuda", generator=g) * 0.03).bfloat16()
    kw = dict(ln_partial=(rec, parts, dim, 1e-5), ln_colsum=w.float().sum(1), bias=0.1 * torch.randn(n, device="cuda", generator=g))
    if layer == "qkv":
        kw["colscale"] = torch.cat([torch.full((D,), 0.125, device="cuda"), torch.ones(2 * D, device="cuda")])
    else:
        kw["gamma"] = 0.1 * torch.randn(n, device="cuda", generator=g)
    return x.bfloat16(), w, epi, kw


def run_layer(K, a, w, epi, kw, res, workspace):
    """one launch on fresh canary buffers: {name: (view, buffer)}"""
    M, n = a.shape[0], w.shape[0]
    dt = BF16 if epi == K.EPI_STORE_BF16 else F32
    out, buf = canary((M, n), dt)
    bufs = {"out": (out, buf)}
    ekw = dict(kw, workspace=workspace)
    if epi == K.EPI_RESID_F32:
        out.copy_(res)
        st = nan_full(((n + 255) // 256, M, 2))
        ob, bb = canary((M, n), BF16)
        ekw.update(resid=out, stats_out=st, out_bf16=ob)
        bufs.update(stats=(st, st), out_bf16=(ob, bb))
    K.gemm_ln(a, w, epi, out, **ekw)
    return bufs


def check_layer(K, ratios, family, a, w, epi, kw, res, workspace, same_as_tiled=False):
    """the split run (with `workspace`) and the tiled run (without) against fp64, and against each other"""
    dt = BF16 if epi == K.EPI_STORE_BF16 else F32
    rkw = dict(kw)
    if epi == K.EPI_RESID_F32:
        rkw.update(resid=res, stats=True)
    ref = R.gemm_ref(a, w, epi, **rkw)
    split = twice(lambda: run_layer(K, a, w, epi, kw, res, workspace))
    tiled = twice(lambda: run_layer(K, a, w, epi, kw, res, None))
    for name, run in (("split", split), ("tiled", tiled)):
        out, buf = run["out"]
        R.assert_canary(buf, out, what=f"{name} output")
        note(ratios, f"{family} {name}", R.assert_within(out, ref.y, ref.mag, TAU, dt, extra=ref.extra, what=f"{name} output"))
        if "stats" in run:
            note(ratios, f"{family} {name} stats", R.assert_within(run["stats"][0], ref.stats, ref.stats_mag, TAU, F32,
                                                                   extra=ref.stats_extra, what=f"{name} statistics records"))
            ob, bb = run["out_bf16"]
            R.assert_canary(bb, ob, what=f"{name} bf16 copy")
            assert torch.equal(ob, out.bfloat16())
    ys, yt = split["out"][0], tiled["out"][0]
    if same_as_tiled:
        for name in split:
            assert torch.equal(bits(split[name][1]), bits(tiled[name][1])), f"{name}: differs from the tiled schedule"
        return
    # the two schedules round differently; each is within the bound of fp64, so they are within twice it of each other
    # (plus both bf16 roundings)
    u = 2.0 ** -8 * ys.double().abs() if dt == BF16 else 0.0
    R.assert_within(ys, yt, 2 * ref.mag, TAU, dt, extra=2 * ref.extra + u, what="split vs tiled")
    if "stats" in split:
        R.assert_within(split["stats"][0], tiled["stats"][0], 2 * ref.stats_mag, TAU, F32, extra=2 * ref.stats_extra,
                        what="split vs tiled statistics")


@pytest.fixture(scope="module")
def workspace():
    return torch.empty(64 << 20 >> 2, device="cuda")       # 64 MB of fp32 slabs


@pytest.mark.parametrize("M", [1, 17, 126, 129, 256])
@pytest.mark.parametrize("layer", ["qkv", "out_proj", "fc2"])
def test_small_m_split_k_layers(K, ratios, workspace, layer, M):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + len(layer))
    a, w, epi, kw = layer_case(layer, M, g)
    res = torch.randn(M, w.shape[0], device="cuda", generator=g)
    check_layer(K, ratios, f"split-K {layer}", a, w, epi, kw, res, workspace)


def _resid_case(M, N, Kd, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = rows_fp32(M, Kd, g)
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).bfloat16()
    kw = dict(ln_partial=(records(x, Kd // 64), Kd // 64, Kd, 1e-5), ln_colsum=w.float().sum(1),
              bias=torch.randn(N, device="cuda", generator=g), gamma=torch.randn(N, device="cuda", generator=g))
    return x.bfloat16(), w, kw, torch.randn(M, N, device="cuda", generator=g)


def test_split_k_piece_limits(K, ratios, workspace):
    """num_k_blocks = 8 (K = 512) still splits; a workspace of two slabs splits in two and writes nothing past them; a
    workspace of one slab, or more tiles than SMs, silently keeps the tiled schedule and leaves the workspace untouched"""
    M, N = 17, 1536
    slab = 128 * N                                          # fp32 elements of one [M rounded up to 128, N] slab
    a, w, kw, res = _resid_case(M, N, 512, 41)
    check_layer(K, ratios, "split-K limits", a, w, K.EPI_RESID_F32, kw, res, workspace)
    a, w, kw, res = _resid_case(M, N, 1536, 42)
    ws3 = torch.full((3 * slab,), float("nan"), device="cuda")
    check_layer(K, ratios, "split-K limits", a, w, K.EPI_RESID_F32, kw, res, ws3[:2 * slab])
    assert torch.equal(bits(ws3[2 * slab:]), bits(torch.full((slab,), float("nan"), device="cuda"))), "wrote past the workspace"
    ws1 = torch.full((slab,), float("nan"), device="cuda")
    check_layer(K, ratios, "split-K limits", a, w, K.EPI_RESID_F32, kw, res, ws1, same_as_tiled=True)
    assert torch.isnan(ws1).all(), "a one-slab workspace must not be used"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_wide = 256 * (sms // 2 + 1)                           # 2 row panels x (sms / 2 + 1) column tiles > sms tiles
    a, w, kw, res = _resid_case(256, n_wide, 512, 43)
    ws = torch.full((4 * 256 * n_wide,), float("nan"), device="cuda")
    check_layer(K, ratios, "split-K limits", a, w, K.EPI_RESID_F32, kw, res, ws, same_as_tiled=True)
    assert torch.isnan(ws).all(), "more tiles than SMs must keep the tiled schedule"


# --------------------------------------------------------------------------------------------------------------------
# row remap, MN-major operands
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("epi_name", ["resid", "store_bf16"])
def test_row_remap(K, ratios, epi_name):
    """out_row = (m / group) * stride + m % group + offset with rows m % group >= valid skipped, and a residual broadcast
    with period `group` (a positional table behind a CLS slot): skipped rows and the CLS slots stay untouched"""
    B, P, valid, N, Kd = 3, 200, 190, 264, 200
    M = B * P
    g = torch.Generator(device="cuda").manual_seed(51)
    a = torch.randn(M, Kd, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    pos = torch.randn(P + 1, N, device="cuda", generator=g)
    remap = dict(out_group=P, out_group_stride=P + 1, out_row_offset=1, out_group_valid=valid)
    if epi_name == "resid":
        epi, dt, kw = K.EPI_RESID_F32, F32, dict(bias=bias, resid=pos, resid_period=P, resid_row_offset=1, **remap)
    else:
        epi, dt, kw = K.EPI_STORE_BF16, BF16, dict(bias=bias, **remap)

    def launch():
        out, buf = R.canary_out((B * (P + 1), N), ldo_extra=8, rows_before=2, rows_after=2, dtype=dt)
        K.gemm_ln(a, w, epi, out, **kw)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    ref = R.gemm_ref(a, w, epi, **kw)
    written = torch.zeros(B * (P + 1), N, dtype=torch.bool, device="cuda")
    written[ref.rows[ref.valid]] = True
    R.assert_canary(buf, out, written=written)
    note(ratios, f"remap {epi_name}", R.assert_within(out[ref.rows[ref.valid]], ref.y[ref.valid], ref.mag[ref.valid], TAU, dt))


@pytest.mark.parametrize("M,N,Kd,a_mn,b_mn,epi_name", [(1536, 1536, 12608, True, True, "store_f32"),
                                                       (200, 264, 1001, True, True, "store_bf16")])
def test_mn_major_operands(K, ratios, M, N, Kd, a_mn, b_mn, epi_name):
    """dW = dY^T X at the vision encoder's shape, and both operands MN-major with a K that is not a multiple of 8"""
    g = torch.Generator(device="cuda").manual_seed(M + Kd)
    A = (torch.randn(M, Kd, device="cuda", generator=g) * 0.5).bfloat16()
    B = (torch.randn(N, Kd, device="cuda", generator=g) * 0.1).bfloat16()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    bias = torch.randn(N, device="cuda", generator=g)
    epi, dt = (K.EPI_STORE_F32, F32) if epi_name == "store_f32" else (K.EPI_STORE_BF16, BF16)

    def launch():
        out, buf = canary((M, N), dt)
        K.gemm_t(a, b, epi, out, a_mn=a_mn, b_mn=b_mn, bias=bias)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    R.assert_canary(buf, out)
    ref = R.gemm_ref(A, B, epi, bias=bias)
    note(ratios, f"mn-major {epi_name}", R.assert_within(out, ref.y, ref.mag, TAU, dt, extra=ref.extra))
