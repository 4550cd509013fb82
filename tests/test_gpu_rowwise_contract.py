"""GPU: the contract of the row kernels (csrc/layernorm.cu, csrc/backward.cu, csrc/pack.cu, csrc/gather.cu) element by
element against the fp64 references of tests/kernel_ref.py (module docstring, "Row kernels").

Inputs with a row pitch wider than the row carry NaN in the gap, which must never reach a result.  Outputs are views into
NaN buffers with spare rows, a wider pitch or a NaN tail, so a store outside the logical output (the padding columns of
the channel-group remap, rows with t >= row_valid, halo rows, past the end of dgamma / colsum) or a skipped store shows
up.  Every kernel without atomics runs twice and must repeat bit for bit, the column reductions included.  Data: N(0, 1)
rows plus stress rows (|mean| / std ~ 10^3, an outlier in column 0, constant rows, var << eps), GELU inputs up to |z| = 8,
dropped rows (row_scale 0) and many duplicate indices for the atomic scatters."""
import zlib

import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
EPS = 1e-5


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def ratios():
    """largest fraction of the bound used, per kernel and output (printed at the end of the module; run with -s)"""
    seen = {}
    yield seen
    print(f"\nbound used on {torch.cuda.get_device_name()}:")
    for k in sorted(seen):
        print(f"bound used: {k:<34s} {seen[k]:.3g}")


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


def seed(*key):
    g = torch.Generator(device="cuda")
    return g.manual_seed(zlib.crc32("/".join(map(str, key)).encode()))


def nan_tail(n, extra=64):
    buf = torch.full((n + extra,), float("nan"), device="cuda")
    return buf[:n], buf


def assert_tail(view, buf, what):
    n = view.numel()
    assert torch.equal(bits(buf[n:]), bits(torch.full_like(buf[n:], float("nan")))), f"{what}: written past the end"
    assert torch.isfinite(view).all(), f"{what}: not every element written"


def gapped(rows, dim, dtype, gap=8):
    """a [rows, dim] view of a [rows, dim + gap] buffer whose gap columns hold NaN"""
    buf = torch.full((rows, dim + gap), float("nan"), dtype=dtype, device="cuda")
    return buf[:, :dim]


def ln_data(rows, dim, g, stress=True):
    """N(0, 1) rows of varied scale; with ``stress`` every 7th row has |mean| / std ~ 10^3, every 11th an outlier of 40
    in column 0, every 13th is constant and every 17th has var << eps"""
    x = torch.randn(rows, dim, device="cuda", generator=g) * (0.5 + torch.rand(rows, 1, device="cuda", generator=g))
    if stress:
        r = torch.arange(rows, device="cuda")
        x[r % 7 == 3] += 1000.0
        x[(r % 11 == 5), 0] += 40.0
        x[r % 13 == 6] = 0.75
        x[r % 17 == 8] = 0.3 + 1e-4 * x[r % 17 == 8]
    return x


def affine(dim, g, wide=False):
    """gamma, beta; ``wide``: |gamma| up to ~8 so that GELU sees inputs up to |z| = 8"""
    s = 3.0 if wide else 0.3
    return 1 + s * torch.randn(dim, device="cuda", generator=g), 0.3 * torch.randn(dim, device="cuda", generator=g)


# --------------------------------------------------------------------------------------------------------------------
# LayerNorm forward
# --------------------------------------------------------------------------------------------------------------------
def ln_fwd_case(K, ratios, family, x, gamma, beta, out_shape, out_dtype, *, gelu=False, accumulate=False, **lay):
    rows, dim = x.shape
    orow, col, wr = (t.cuda() for t in R.ln_layout(rows, dim, **lay))
    ro, co = orow[wr][:, None], col[wr]
    init = torch.randn(out_shape, device="cuda") if accumulate else None

    def launch():
        out, buf = R.canary_out(out_shape, ldo_extra=8, rows_before=1, rows_after=2, dtype=out_dtype)
        if accumulate:
            out.copy_(init)
        K.layernorm(x, gamma, beta, out, rows=rows, dim=dim, eps=EPS, gelu=gelu, accumulate=accumulate, **lay)
        return {"y": (out, buf)}

    out, buf = twice(launch)["y"]
    written = torch.zeros(out_shape, dtype=torch.bool, device="cuda")
    written[ro, co] = True
    if accumulate:
        R.assert_canary(buf, out, what=family)
        assert torch.equal(out[~written], init[~written]), f"{family}: rows outside the map changed"
    else:
        R.assert_canary(buf, out, written, what=family)
    r = R.layernorm_ref(x[wr], gamma, beta, EPS, gelu=gelu, prev=init[ro, co] if accumulate else None)
    note(ratios, family, R.assert_within(out[ro, co], r.y, r.err, 1.0, out_dtype, what=family))


LN_PAIRS = [(F32, BF16), (BF16, BF16), (F32, F32), (BF16, F32)]
# every VPL boundary of the one-warp-per-row forward (8 per lane-vector, 256 columns per VPL step) and its neighbours
LN_DIMS = [8, 248, 256, 264, 504, 512, 520, 1016, 1024, 1032, 1528, 1536, 1544, 2040, 2048, 3064, 3072, 3080, 6136, 6144]
LN_ROWS = [1, 5, 31, 33, 1055, 1056, 1057, 2 * 1056 + 17]


@pytest.mark.parametrize("i", range(len(LN_DIMS)), ids=[f"dim{d}" for d in LN_DIMS])
def test_layernorm_dims(K, ratios, i):
    dim = LN_DIMS[i]
    pairs = [p for p in LN_PAIRS if p[0] == BF16 or dim <= 2048]         # fp32 rows are supported up to 2048
    tin, tout = pairs[i % len(pairs)]
    rows = LN_ROWS[i % len(LN_ROWS)]
    g = seed("ln", dim)
    x = gapped(rows, dim, tin)
    x.copy_(ln_data(rows, dim, g))
    gamma, beta = affine(dim, g, wide=i % 2 == 1)
    ln_fwd_case(K, ratios, f"layernorm {str(tin)[6:]}->{str(tout)[6:]}", x, gamma, beta, (rows, dim), tout, gelu=i % 2 == 1)
    if i % 3 == 0:                                                   # non-affine
        ln_fwd_case(K, ratios, "layernorm plain", x, None, None, (rows, dim), tout)


def test_layernorm_production_rows(K, ratios):
    """the 12608-row d = 1536 stream of the text / image stacks, fp32 in, bf16 out"""
    g = seed("ln12608")
    x = ln_data(12608, 1536, g)
    gamma, beta = affine(1536, g)
    ln_fwd_case(K, ratios, "layernorm f32->bf16", x, gamma, beta, (12608, 1536), BF16)


@pytest.mark.parametrize("g1", [56, 64])
def test_layernorm_merge(K, ratios, g1):
    """hMLP stem: LN -> GELU with the 2 x 2 pixel-merge scatter at both stages (R = 224: 56 / 28, R = 256: 64 / 32),
    c4 = 384 channels, two images"""
    g = seed("merge", g1)
    for w in (g1, g1 // 2):
        rows, dim = 2 * w * w, 384
        x = ln_data(rows, dim, g, stress=False).bfloat16()
        gamma, beta = affine(dim, g, wide=True)
        ln_fwd_case(K, ratios, "layernorm merge gelu", x, gamma, beta, (rows // 4, 4 * dim), BF16, gelu=True,
                    merge_grid_w=w)


@pytest.mark.parametrize("accumulate", [False, True])
def test_layernorm_group_remap(K, ratios, accumulate):
    """audio positional convolution: non-affine LN -> GELU over B x Tp rows, rows t >= T skipped, output shifted by the
    halo and its 16 channel groups of 96 padded to 104 (bf16); or accumulated into the fp32 stream (no padding)"""
    B, T, Tp, halo, d, cg, cpad = 3, 50, 56, 64, 1536, 96, 104
    g = seed("group", accumulate)
    x = ln_data(B * Tp, d, g).bfloat16()
    if accumulate:
        ln_fwd_case(K, ratios, "layernorm remap accumulate", x, None, None, (B * (T + 1), d), F32, gelu=True,
                    accumulate=True, row_period=Tp, row_valid=T, out_period=T + 1, out_row_shift=1)
    else:
        ln_fwd_case(K, ratios, "layernorm remap groups", x, None, None, (B * (Tp + 2 * halo), 16 * cpad), BF16, gelu=True,
                    row_period=Tp, row_valid=T, out_period=Tp + 2 * halo, out_row_shift=halo, group_in=cg, group_out=cpad)


def test_head_layernorm_strided(K, ratios):
    """the head LayerNorm of the CLS rows: B = 8 rows read at a pitch of S * d"""
    B, S, d = 8, 197, 1536
    g = seed("headln")
    full = ln_data(B * S, d, g)
    full.view(B, S * d)[:, d:] = float("nan")                          # only the CLS rows are read
    x = full.view(B, S * d)[:, :d]
    gamma, beta = affine(d, g)
    ln_fwd_case(K, ratios, "layernorm head", x, gamma, beta, (B, d), F32)


@pytest.mark.parametrize("rows,dim", [(5, 8), (1057, 1536), (12608, 1536), (33, 2048)])
def test_row_stats_cast(K, ratios, rows, dim):
    """the ``raw`` mode: bf16(x) bit for bit, and mu / rstd for the fused-LN GEMM"""
    g = seed("raw", rows, dim)
    x = gapped(rows, dim, F32)
    x.copy_(ln_data(rows, dim, g))

    def launch():
        out, buf = R.canary_out((rows, dim), ldo_extra=8, rows_before=1, rows_after=1, dtype=BF16)
        mu, mb = nan_tail(rows)
        rs, rb = nan_tail(rows)
        K.row_stats_cast(x, out, mu, rs, EPS)
        return {"out": (out, buf), "mu": (mu, mb), "rstd": (rs, rb)}

    res = twice(launch)
    out, buf = res["out"]
    R.assert_canary(buf, out, what="raw out")
    assert torch.equal(bits(out), bits(x.bfloat16())), "raw: the copy is not bf16(x)"
    r = R.layernorm_ref(x, None, None, EPS)
    for name, ref, bound in (("mu", r.mu, r.dmu), ("rstd", r.rstd, r.rel * r.rstd)):
        assert_tail(*res[name], f"raw {name}")
        note(ratios, f"row_stats_cast {name}", R.assert_within(res[name][0], ref, bound, 1.0, F32, what=name))


@pytest.mark.parametrize("parts,rows", [(6, 12608), (24, 33), (96, 1057)])
def test_ln_stats_finalize(K, ratios, parts, rows):
    """records of stress rows (|mean| / std ~ 10^3 included), up to 96 parts"""
    dim = parts * 64
    g = seed("fin", parts, rows)
    x = ln_data(rows, dim, g).double()
    s = x.view(rows, parts, 64)
    rec = torch.stack([s.sum(2), (s * s).sum(2)], 2).transpose(0, 1).float().contiguous()
    mu_ref, rstd_ref, dmu, rel = R.ln_stats_ref(rec, parts, rows, dim, EPS)

    def launch():
        mu, mb = nan_tail(rows)
        rs, rb = nan_tail(rows)
        K.ln_stats_finalize(rec, parts, rows, dim, EPS, mu, rs)
        return {"mu": (mu, mb), "rstd": (rs, rb)}

    res = twice(launch)
    for name, ref, bound in (("mu", mu_ref, dmu), ("rstd", rstd_ref, rel * rstd_ref)):
        assert_tail(*res[name], f"finalize {name}")
        note(ratios, f"ln_stats_finalize {name}", R.assert_within(res[name][0], ref, bound, 1.0, F32, what=name))


# --------------------------------------------------------------------------------------------------------------------
# LayerNorm backward
# --------------------------------------------------------------------------------------------------------------------
LNB_TRIPLES = [(x, y, z) for x in (F32, BF16) for y in (F32, BF16) for z in (F32, BF16)]
# float4 groups x threads: 128 x 1 (dim <= 512, with prefetch), 128 x 3 (<= 1536, prefetch), 256 x 3 (<= 3072), 256 x 6
LNB_DIMS = [4, 8, 508, 512, 516, 1532, 1536, 1540, 2048, 3072, 3076, 6140, 6144]
LNB_ROWS = [1, 5, 31, 33, 1055, 1056, 1057, 2 * 1056 + 17, 12608]


def ln_bwd_case(K, ratios, family, x, dy_store, gamma, beta, dxdt, *, gelu=False, accumulate=False, merge_w=0,
                dx_pitch=8, dx_view=None):
    """x [rows, dim] (any pitch); dy_store: dy as the kernel reads it ([rows, dim], or the merged [rows / 4, 4 dim])"""
    rows, dim = x.shape
    old = torch.randn(rows, dim, device="cuda") if accumulate else None

    def launch():
        if dx_view is not None:
            dx, buf = dx_view()
        else:
            dx, buf = R.canary_out((rows, dim), ldo_extra=dx_pitch, rows_before=1, rows_after=1, dtype=dxdt)
        if accumulate:
            dx.copy_(old)
        dg, dgb = nan_tail(dim)
        db, dbb = nan_tail(dim)
        K.layernorm_bwd(x, dy_store, gamma, beta, dx, eps=EPS, gelu=gelu, accumulate=accumulate, dgamma=dg, dbeta=db,
                        rows=rows, dim=dim, dy_merge_w=merge_w)
        return {"dx": (dx, buf), "dgamma": (dg, dgb), "dbeta": (db, dbb)}

    res = twice(launch)
    if merge_w:
        src, c0 = (t.cuda() for t in R.merge_rows(rows, dim, merge_w))
        dy = dy_store[src[:, None], c0[:, None] + torch.arange(dim, device="cuda")[None, :]]
    else:
        dy = dy_store
    r = R.layernorm_bwd_ref(x, dy, gamma, beta, EPS, gelu=gelu, old=old)
    dx, buf = res["dx"]
    if dx_view is None:
        R.assert_canary(buf, dx, what=f"{family} dx")
    note(ratios, f"{family} dx", R.assert_within(dx, r.dx, r.dx_err, 1.0, dxdt, what=f"{family} dx"))
    for name, ref, bound in (("dgamma", r.dgamma, r.dgamma_err), ("dbeta", r.dbeta, r.dbeta_err)):
        assert_tail(*res[name], f"{family} {name}")
        note(ratios, f"layernorm_bwd {name}", R.assert_within(res[name][0], ref, bound, 1.0, F32, what=f"{family} {name}"))
    return res


@pytest.mark.parametrize("i", range(len(LNB_DIMS)), ids=[f"dim{d}" for d in LNB_DIMS])
def test_layernorm_bwd_dims(K, ratios, i):
    """every dtype triple, every config boundary and its neighbours, rows around the 1056-CTA grid cap; the dy and x
    rows carry NaN in a pitch gap"""
    dim = LNB_DIMS[i]
    xdt, dydt, dxdt = LNB_TRIPLES[i % 8]
    rows = LNB_ROWS[i % len(LNB_ROWS)]
    if dim > 1536 and rows > 2200:
        rows = 2 * 1056 + 17
    g = seed("lnb", dim)
    x = gapped(rows, dim, xdt)
    x.copy_(ln_data(rows, dim, g))
    dy = gapped(rows, dim, dydt)
    dy.copy_(torch.randn(rows, dim, device="cuda", generator=g))
    gamma, beta = affine(dim, g)
    gelu = i % 3 == 2
    if gelu:
        gamma, beta = affine(dim, g, wide=True)
    fam = f"layernorm_bwd {'gelu' if gelu else 'plain'}"
    ln_bwd_case(K, ratios, fam, x, dy, gamma, beta, dxdt, gelu=gelu)
    if dxdt == F32:
        ln_bwd_case(K, ratios, fam + " acc", x, dy, gamma, beta, dxdt, gelu=gelu, accumulate=True)
    if i % 4 == 0:
        ln_bwd_case(K, ratios, fam, x, dy, None, None, dxdt, gelu=gelu)


@pytest.mark.parametrize("k", range(8))
def test_layernorm_bwd_triples(K, ratios, k):
    """all 8 (x, dy, dx) dtype triples at d = 1536 and F = 6144 (the encoder layer's LayerNorms)"""
    xdt, dydt, dxdt = LNB_TRIPLES[k]
    for rows, dim in ((1057, 1536), (300, 6144)):
        g = seed("trip", k, dim)
        x = ln_data(rows, dim, g).to(xdt)
        dy = torch.randn(rows, dim, device="cuda", generator=g).to(dydt)
        gamma, beta = affine(dim, g)
        ln_bwd_case(K, ratios, "layernorm_bwd plain", x, dy, gamma, beta, dxdt, gelu=k % 2 == 1)


def test_layernorm_bwd_production_rows(K, ratios):
    g = seed("lnb12608")
    x = ln_data(12608, 1536, g)
    dy = torch.randn(12608, 1536, device="cuda", generator=g).bfloat16()
    gamma, beta = affine(1536, g)
    ln_bwd_case(K, ratios, "layernorm_bwd plain acc", x, dy, gamma, beta, F32, accumulate=True)


@pytest.mark.parametrize("g1", [56, 64])
def test_layernorm_bwd_merge(K, ratios, g1):
    """adjoint of the hMLP stem's LN -> GELU -> 2 x 2 merge: dy read through the merge map"""
    for w in (g1, g1 // 2):
        rows, dim = 2 * w * w, 384
        g = seed("lnbm", w)
        x = ln_data(rows, dim, g, stress=False).bfloat16()
        dy = torch.randn(rows // 4, 4 * dim, device="cuda", generator=g).bfloat16()
        gamma, beta = affine(dim, g, wide=True)
        ln_bwd_case(K, ratios, "layernorm_bwd merge", x, dy, gamma, beta, BF16, gelu=True, merge_w=w)


def test_layernorm_bwd_head_strided(K, ratios):
    """HeadFn.backward: B = 8 CLS rows of x and dx at a pitch of S * d (dx rows in between must stay untouched)"""
    B, S, d = 8, 197, 1536
    g = seed("headbwd")
    full = ln_data(B * S, d, g)
    full.view(B, S * d)[:, d:] = float("nan")
    x = full.view(B, S * d)[:, :d]
    dy = torch.randn(B, d, device="cuda", generator=g)
    gamma, beta = affine(d, g)
    bufs = []

    def dx_view():
        buf = torch.full((B * S + 1, d), float("nan"), device="cuda")
        bufs.append(buf)
        return buf.view(-1)[:B * S * d].view(B, S * d)[:, :d], buf

    res = ln_bwd_case(K, ratios, "layernorm_bwd head", x, dy, gamma, beta, F32, dx_view=dx_view)
    buf = res["dx"][1]
    rest = buf.view(-1)[:B * S * d].view(B, S * d)[:, d:]
    assert torch.isnan(rest).all() and torch.isnan(buf[B * S:]).all(), "head dx: rows between the CLS rows written"


# --------------------------------------------------------------------------------------------------------------------
# GeGLU, LayerScale residual, column sums
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,F", [(1, 8), (33, 6144), (1057, 6144), (517, 2056)])
def test_geglu(K, ratios, rows, F):
    g = seed("geglu", rows, F)
    gl = (torch.randn(rows, 2 * F, device="cuda", generator=g) * 2.7).clamp(-8, 8).bfloat16()
    du = torch.randn(rows, F, device="cuda", generator=g).bfloat16()

    def launch():
        u, ub = R.canary_out((rows, F), rows_before=1, rows_after=1, dtype=BF16)
        dgl, db = R.canary_out((rows, 2 * F), rows_before=1, rows_after=1, dtype=BF16)
        K.geglu_fwd(gl, u)
        K.geglu_bwd(gl, du, dgl)
        return {"u": (u, ub), "dgl": (dgl, db)}

    res = twice(launch)
    for name, (ref, bound) in (("u", R.geglu_ref(gl)), ("dgl", R.geglu_bwd_ref(gl, du))):
        view, buf = res[name]
        R.assert_canary(buf, view, what=f"geglu {name}")
        note(ratios, f"geglu {name}", R.assert_within(view, ref, bound, 1.0, BF16, what=f"geglu {name}"))


def sres_case(K, ratios, family, dx, o, gamma, rs, rows, n, **gat):
    def launch():
        d_o, buf = R.canary_out((rows, n), rows_before=1, rows_after=1, dtype=BF16)
        dg, dgb = nan_tail(n)
        db, dbb = nan_tail(n)
        K.scale_resid_bwd(dx, o, gamma, rs, d_o, dgamma=dg if o is not None else None, dbias=db, **gat)
        return {"d_o": (d_o, buf), "dgamma": (dg, dgb), "dbias": (db, dbb)}

    res = twice(launch)
    idx = R.scale_resid_rows(rows, gat.get("in_period", 0), gat.get("in_valid", 0), gat.get("in_shift", 0)).cuda()
    r = R.scale_resid_bwd_ref(dx[idx], o, gamma, rs)
    d_o, buf = res["d_o"]
    R.assert_canary(buf, d_o, what=f"{family} d_o")
    note(ratios, f"{family} d_o", R.assert_within(d_o, r.d_o, r.d_o_err, 1.0, BF16, what=f"{family} d_o"))
    outs = (("dgamma", r.dgamma, r.dgamma_err), ("dbias", r.dbias, r.dbias_err)) if o is not None else \
        (("dbias", r.dbias, r.dbias_err),)
    for name, ref, bound in outs:
        assert_tail(*res[name], f"{family} {name}")
        note(ratios, f"{family} {name}", R.assert_within(res[name][0], ref, bound, 1.0, F32, what=f"{family} {name}"))
    if o is None:
        assert torch.isnan(res["dgamma"][1]).all(), f"{family}: dgamma written without o"


@pytest.mark.parametrize("rows,n", [(1, 4), (8, 1536), (31, 1540), (1057, 1536), (2129, 6144), (12608, 1536)])
def test_scale_resid(K, ratios, rows, n):
    """LayerScale + drop-path residual, forward and backward; half the rows' row_scale is 0 (dropped)"""
    g = seed("sres", rows, n)
    x = torch.randn(rows, n, device="cuda", generator=g)
    o = torch.randn(rows, n, device="cuda", generator=g).bfloat16()
    gamma = torch.randn(n, device="cuda", generator=g)
    rs = (torch.rand(rows, device="cuda", generator=g) < 0.5).float() / 0.5

    def launch():
        out, buf = R.canary_out((rows, n), rows_before=1, rows_after=1)
        K.scale_resid_fwd(x, o, gamma, rs, out)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    R.assert_canary(buf, out, what="scale_resid_fwd")
    ref, bound = R.scale_resid_ref(x, o, gamma, rs)
    note(ratios, "scale_resid_fwd", R.assert_within(out, ref, bound, 1.0, F32, what="scale_resid_fwd"))
    sres_case(K, ratios, "scale_resid_bwd", x, o, gamma, rs, rows, n)
    sres_case(K, ratios, "scale_resid_bwd", x, o, None, None, rows, n)


@pytest.mark.parametrize("S", [197, 257])
def test_scale_resid_bwd_gather(K, ratios, S):
    """image adapter: the token rows behind the CLS slot of B = 4 samples, bias gradient only (no o, gamma, row_scale)"""
    B, d = 4, 1536
    g = seed("gat", S)
    dx = torch.randn(B * S, d, device="cuda", generator=g)
    sres_case(K, ratios, "scale_resid_bwd gather", dx, None, None, None, B * (S - 1), d, in_period=S, in_valid=S - 1,
              in_shift=1)


@pytest.mark.parametrize("rows,n", [(8, 1536), (33, 4), (1057, 6144), (12608, 1536)])
def test_colsum(K, ratios, rows, n):
    g = seed("colsum", rows, n)
    y = gapped(rows, n, BF16)
    y.copy_(torch.randn(rows, n, device="cuda", generator=g))

    def launch():
        out, buf = nan_tail(n)
        K.colsum(y, out)
        return {"colsum": (out, buf)}

    out, buf = twice(launch)["colsum"]
    assert_tail(out, buf, "colsum")
    ref, bound = R.colsum_ref(y)
    note(ratios, "colsum", R.assert_within(out, ref, bound, 1.0, F32, what="colsum"))


# --------------------------------------------------------------------------------------------------------------------
# ln_fold, l2_normalize_bwd, batch_sum, window_scatter
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("interleave", [0, 1, 2])
@pytest.mark.parametrize("wdt", [F32, BF16])
def test_ln_fold(K, ratios, interleave, wdt):
    """Wg bit for bit, colsum of the rounded Wg, bias' = W beta + b; K = 1000 (not a multiple of 128); the interleave
    writes every other 128-row block of a 2N-row operand and leaves the rest alone"""
    N, Kd = 384, 1000
    g = seed("fold", interleave, wdt)
    W = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).to(wdt)
    lw, lb = 1 + 0.2 * torch.randn(Kd, device="cuda", generator=g), 0.1 * torch.randn(Kd, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    n_out = N if interleave == 0 else 2 * N

    def launch():
        wo, wb = R.canary_out((n_out, Kd), ldo_extra=8, rows_before=1, rows_after=1, dtype=BF16)
        cs, cb = nan_tail(n_out)
        bo, bb = nan_tail(n_out)
        K.ln_fold(W, lw, lb, bias, wo, cs, bo, interleave=interleave)
        return {"w": (wo, wb), "colsum": (cs, cb), "bias": (bo, bb)}

    res = twice(launch)
    f = R.ln_fold_ref(W, lw, lb, bias, interleave)
    written = torch.zeros(n_out, dtype=torch.bool, device="cuda")
    written[f.rows] = True
    wo, wb = res["w"]
    R.assert_canary(wb, wo, written[:, None].expand(n_out, Kd), what="ln_fold w")
    assert torch.equal(bits(wo[f.rows]), bits(f.wg)), "ln_fold: Wg is not bf16(W g)"
    for name, ref, bound in (("colsum", f.colsum, f.colsum_err), ("bias", f.bias, f.bias_err)):
        v, b = res[name]
        assert torch.isnan(b[n_out:]).all() and torch.isnan(v[~written]).all(), f"ln_fold {name}: written outside the map"
        note(ratios, f"ln_fold {name}", R.assert_within(v[f.rows], ref, bound, 1.0, F32, what=f"ln_fold {name}"))


@pytest.mark.parametrize("rows,D", [(1, 32), (64, 768), (257, 1536)])
def test_l2_normalize_bwd(K, ratios, rows, D):
    g = seed("l2", rows, D)
    x = gapped(rows, D, F32)
    x.copy_(torch.randn(rows, D, device="cuda", generator=g) * torch.rand(rows, 1, device="cuda", generator=g) * 10)
    dy = gapped(rows, D, F32)
    dy.copy_(torch.randn(rows, D, device="cuda", generator=g))

    def launch():
        d16, d32 = K.l2_normalize_bwd(x, dy, want_f32=True)
        return {"dx16": (d16, d16), "dx32": (d32, d32)}

    res = twice(launch)
    ref, bound = R.l2_normalize_bwd_ref(x, dy)
    for name, dt in (("dx16", BF16), ("dx32", F32)):
        note(ratios, f"l2_normalize_bwd {name}", R.assert_within(res[name][0], ref, bound, 1.0, dt, what=name))


@pytest.mark.parametrize("accumulate", [False, True])
def test_batch_sum(K, ratios, accumulate):
    """out (+)= sum over B = 37 rows at a pitch wider than n (the gap holds NaN)"""
    B, n = 37, 5000
    g = seed("bsum", accumulate)
    x = gapped(B, n, F32, gap=24)
    x.copy_(torch.randn(B, n, device="cuda", generator=g))
    init = torch.randn(n, device="cuda", generator=g)

    def launch():
        out, buf = nan_tail(n)
        if accumulate:
            out.copy_(init)
        K.batch_sum(x, out, B, n, x.stride(0), accumulate=accumulate)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    assert_tail(out, buf, "batch_sum")
    ref, bound = R.scatter_ref(init[None] if accumulate else torch.zeros(1, n, device="cuda"),
                               torch.zeros(B, dtype=torch.long, device="cuda"), x)
    note(ratios, "batch_sum", R.assert_within(out, ref[0], bound[0], 1.0, F32, what="batch_sum"))


@pytest.mark.parametrize("B,t_in,t_out,stride,kw,pad,groups,C", [(2, 400, 79, 5, 10, 0, 1, 512),
                                                                 (2, 100, 101, 1, 128, 64, 16, 512)])
def test_window_scatter(K, ratios, B, t_in, t_out, stride, kw, pad, groups, C):
    """col2im of the audio feature-extractor convolution (stride 5, 10 taps) and of the grouped positional convolution
    (128 taps, 16 groups)"""
    g = seed("wsc", kw)
    cg = C // groups
    dwin = torch.randn(groups, B * t_out, kw * cg, device="cuda", generator=g).bfloat16()

    def launch():
        dx = K.window_scatter(dwin, B, t_in, t_out, stride, kw, pad)
        return {"dx": (dx, dx)}

    dx = twice(launch)["dx"][0]
    ref, bound = R.window_scatter_ref(dwin, B, t_in, t_out, stride, kw, pad)
    note(ratios, "window_scatter", R.assert_within(dx, ref, bound, 1.0, BF16, what="window_scatter"))


# --------------------------------------------------------------------------------------------------------------------
# scatter-add adjoints (fp32 atomics: no bit-repeatability)
# --------------------------------------------------------------------------------------------------------------------
def test_text_embed_bwd(K, ratios):
    """B = 8 texts of T = 40 tokens from a vocabulary of 50 (many duplicates), pad id 1 at different lengths (one text
    all padding): pad tokens contribute nothing"""
    B, T, D, V = 8, 40, 1536, 50
    g = seed("tembed")
    tok = torch.randint(2, V, (B, T), device="cuda", generator=g)
    for b in range(B):
        tok[b, [40, 33, 1, 0, 17, 39, 25, 8][b]:] = 1
    dx = torch.randn(B, T + 1, D, device="cuda", generator=g)
    t0, p0, c0 = (torch.randn(*s, device="cuda", generator=g) for s in ((V, D), (T + 1, D), (1, D)))
    dt, dp, dc = t0.clone(), p0.clone(), c0.clone()
    K.text_embed_bwd(dx, tok, dt, dp, dc[0], pad_idx=1)
    bi, si = (tok != 1).nonzero(as_tuple=True)
    live = dx[bi, si + 1]
    cases = (("dtable", dt, t0, tok[bi, si], live),
             ("dpos", dp, p0, torch.cat([torch.zeros(B, dtype=torch.long, device="cuda"), si + 1]), torch.cat([dx[:, 0], live])),
             ("dcls", dc, c0, torch.zeros(B, dtype=torch.long, device="cuda"), dx[:, 0]))
    for name, got, init, dest, src in cases:
        ref, bound = R.scatter_ref(init, dest, src)
        note(ratios, f"text_embed_bwd {name}", R.assert_within(got, ref, bound, 1.0, F32, what=name))


def test_relpos_bias_bwd(K, ratios):
    """dtable[bucket[i, j], h] += dbias[h, i, j] with S = 197 and NaN in the table's pad columns"""
    S, H, NB = 197, 4, 60
    s_pad = 200
    g = seed("rpb")
    db = torch.full((H, S, s_pad), float("nan"), device="cuda")
    db[..., :S] = torch.randn(H, S, S, device="cuda", generator=g)
    bucket = torch.randint(0, NB, (S, S), device="cuda", generator=g)
    t0 = torch.randn(NB, H, device="cuda", generator=g)
    got = t0.clone()
    K.relpos_bias_bwd(db, bucket, got, S)
    dest = (bucket[None] * H + torch.arange(H, device="cuda")[:, None, None]).reshape(-1)
    ref, bound = R.scatter_ref(t0.view(-1, 1), dest, db[..., :S].reshape(-1, 1))
    note(ratios, "relpos_bias_bwd", R.assert_within(got.view(-1, 1), ref, bound, 1.0, F32, what="relpos_bias_bwd"))


def test_relpos_bias_block_bwd(K, ratios):
    """one modality's block [lo, lo + n) of Bb = 3 per-sample canvases, preserve ids with -1 (mapped to n - 1)"""
    Bb, H, S, n, lo, NB = 3, 4, 90, 70, 12, 40
    s_pad = 96
    g = seed("rpbb")
    db = torch.full((Bb, H, S, s_pad), float("nan"), device="cuda")         # NaN outside the block
    db[:, :, lo:lo + n, lo:lo + n] = torch.randn(Bb, H, n, n, device="cuda", generator=g)
    bucket = torch.randint(0, NB, (n, n), device="cuda", generator=g)
    ids = torch.stack([torch.randperm(n, device="cuda", generator=g) for _ in range(Bb)])
    ids[0, 50:] = -1
    ids[2, ::3] = -1
    t0 = torch.randn(NB, H, device="cuda", generator=g)
    got = t0.clone()
    K.relpos_bias_block_bwd(db, bucket, ids, n, lo, got, S, H)
    p = torch.where(ids < 0, torch.full_like(ids, n - 1), ids)
    bk = bucket[p[:, :, None], p[:, None, :]]                                        # [Bb, n, n]
    dest = (bk[:, None] * H + torch.arange(H, device="cuda")[None, :, None, None]).reshape(-1)
    src = db[:, :, lo:lo + n, lo:lo + n].reshape(-1, 1)
    ref, bound = R.scatter_ref(t0.view(-1, 1), dest, src)
    note(ratios, "relpos_bias_block_bwd", R.assert_within(got.view(-1, 1), ref, bound, 1.0, F32, what="block_bwd"))


@pytest.mark.parametrize("dt", [F32, BF16])
def test_row_scatter_add(K, ratios, dt):
    """dsrc[idx[r]] += dout[r]: 3000 rows onto 37 (many duplicates), every fifth idx -1 (skipped); dout at a wider pitch
    with NaN in the gap"""
    rows, n, dim = 3000, 37, 1540
    g = seed("rsa", dt)
    dout = gapped(rows, dim, dt)
    dout.copy_(torch.randn(rows, dim, device="cuda", generator=g))
    idx = torch.randint(0, n, (rows,), device="cuda", generator=g)
    idx[::5] = -1
    d0 = torch.randn(n, dim, device="cuda", generator=g)
    got = d0.clone()
    K.row_scatter_add(dout, idx, got)
    ref, bound = R.scatter_ref(d0, idx, dout)
    note(ratios, "row_scatter_add", R.assert_within(got, ref, bound, 1.0, F32, what="row_scatter_add"))
