"""GPU: the contract of the kernels that turn model inputs into the first residual stream, move rows between layouts and
rank retrieval candidates (csrc/adapters.cu, ``relpos_lut_build`` in csrc/attention.cu, csrc/gather.cu, ``transpose_bf16``
in csrc/infonce.cu, csrc/recall.cu), element by element against the exact and fp64 references of tests/kernel_ref.py
(module docstring, "Embedding, gather, transpose and ranking kernels").

Every kernel is called through the C ABI with its outputs inside NaN (or sentinel) buffers with spare rows or a tail, so a
store outside the logical output or a skipped store shows up; inputs with a row pitch wider than the row carry NaN in the
gap, and tables are followed by NaN rows, so a read past either reaches a result.  Every launch runs twice and must repeat
bit for bit.  Shapes sit at the boundaries each kernel's thread mapping creates: D / 4 threads rounded up to a warp and
capped at 256 (``text_embed``), 128-thread strided rows, one warp per gathered row, 64 x 64 transpose tiles on the
vectorised and the scalar path, and one warp per top-10 row with 32 strided lane lists."""
import zlib

import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
OK, INVALID = 0, 1
PAD_IDX = 1


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import _lib
    return _lib.load()


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
    if t.dtype == BF16:
        return t.view(torch.int16)
    return t.view(torch.int32) if t.dtype == F32 else t


def twice(launch):
    """launch() -> {name: (view, buffer)} on fresh buffers; run it twice, the buffers must match bit for bit"""
    r1, r2 = launch(), launch()
    for name in r1:
        assert torch.equal(bits(r1[name][1]), bits(r2[name][1])), f"{name}: two launches differ"
    return r1


def seed(*key):
    g = torch.Generator(device="cuda")
    return g.manual_seed(zlib.crc32("/".join(map(str, key)).encode()))


def stream():
    return torch.cuda.current_stream().cuda_stream


def tail(n, fill, dtype=F32, extra=64):
    """a flat output of n elements at the start of a buffer whose ``extra`` trailing elements hold ``fill``"""
    buf = torch.full((n + extra,), fill, dtype=dtype, device="cuda")
    return buf[:n], buf


def assert_tail(view, buf, fill, what):
    n = view.numel()
    want = torch.full_like(buf[n:], fill)
    assert torch.equal(bits(buf[n:]), bits(want)), f"{what}: written past the end"


def followed_by_nan(t, rows=1):
    """a copy of t [n, ...] at the start of a buffer with ``rows`` NaN rows after it"""
    buf = torch.full((t.shape[0] + rows, *t.shape[1:]), float("nan"), dtype=t.dtype, device="cuda")
    buf[:t.shape[0]] = t
    return buf[:t.shape[0]]


def gapped(rows, dim, dtype, gap=8):
    """a [rows, dim] view of a [rows, dim + gap] buffer whose gap columns hold NaN"""
    buf = torch.full((rows, dim + gap), float("nan"), dtype=dtype, device="cuda")
    return buf[:, :dim]


def nan_payloads(x, g):
    """x fp32 with NaN payloads (quiet, signalling, negative) scattered over it"""
    iv = x.view(torch.int32).view(-1)
    pick = torch.rand(iv.numel(), device="cuda", generator=g)
    for lo, hi, pattern in ((0.0, 0.05, 0x7FC01234), (0.05, 0.1, 0x7FA00001), (0.1, 0.15, 0xFFC0BEEF - 2 ** 32)):
        iv[(pick >= lo) & (pick < hi)] = pattern
    return x


# --------------------------------------------------------------------------------------------------------------------
# text_embed, cls_row_init, zero_padded_rows
# --------------------------------------------------------------------------------------------------------------------
EMB_D = [4, 132, 1020, 1024, 1536]      # 1, 33 -> 64, 255 -> 256, 256 and 256 threads (the last one loops)
EMB_T = [1, 16, 76, 511]
VOCAB = 777


def embed_tokens(B, T, g):
    """ids 0 and vocab - 1, a pad at position 1 (the first token), one mid-row, a padded tail, and a whole padded row"""
    tok = torch.randint(2, VOCAB, (B, T), device="cuda", generator=g)
    tok[0, 0] = VOCAB - 1
    tok[0, -1] = 0 if T > 1 else tok[0, -1]
    tok[1, 0] = PAD_IDX
    tok[1, T // 2] = PAD_IDX
    tok[2, T // 2:] = PAD_IDX
    tok[3] = PAD_IDX
    return tok


@pytest.mark.parametrize("tdt", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("D", EMB_D)
def test_text_embed(lib, D, tdt):
    B = 4
    for T in EMB_T:
        g = seed("embed", D, T, tdt)
        tok = embed_tokens(B, T, g)
        table = followed_by_nan(torch.randn(VOCAB, D, device="cuda", generator=g).to(tdt))
        pos = followed_by_nan(torch.randn(T + 1, D, device="cuda", generator=g))        # exactly T + 1 rows
        cls = followed_by_nan(torch.randn(D, device="cuda", generator=g))
        rows = B * (T + 1)

        def launch():
            x, xb = R.canary_out((rows, D), rows_before=1, rows_after=2)
            pm, pb = tail(rows, 0xA5, torch.uint8)
            assert lib.opb_text_embed(tok.data_ptr(), table.data_ptr(), int(tdt == BF16), pos.data_ptr(), cls.data_ptr(),
                                      x.data_ptr(), pm.data_ptr(), B, T, D, PAD_IDX, stream()) == OK
            return {"x": (x, xb), "pad": (pm, pb)}

        got = twice(launch)
        x, xb = got["x"]
        R.assert_canary(xb, x, what=f"text_embed D={D} T={T}")
        assert_tail(*got["pad"], 0xA5, "text_embed pad mask")
        ref, pad = R.text_embed_ref(tok, table, pos, cls, PAD_IDX)
        assert torch.equal(got["pad"][0], pad.view(-1)), "pad mask"
        live = pad.view(-1) == 0
        assert torch.equal(bits(x[live]), bits(ref.view(rows, D)[live])), f"text_embed D={D} T={T}: live rows"
        assert (x[~live] == 0).all(), f"text_embed D={D} T={T}: pad rows not zero"


@pytest.mark.parametrize("D", [4, 256, 1536])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_cls_row_init(lib, B, D):
    S = 5
    g = seed("cls", B, D)
    init = nan_payloads(torch.randn(B, S, D, device="cuda", generator=g), g)
    cls = followed_by_nan(torch.randn(D, device="cuda", generator=g))
    pos0 = followed_by_nan(torch.randn(D, device="cuda", generator=g))

    def launch():
        x, buf = tail(B * S * D, float("nan"))
        x.copy_(init.view(-1))
        assert lib.opb_cls_row_init(cls.data_ptr(), pos0.data_ptr(), x.data_ptr(), S * D, B, D, stream()) == OK
        return {"x": (x, buf)}

    x, buf = twice(launch)["x"]
    assert_tail(x, buf, float("nan"), "cls_row_init")
    x = x.view(B, S, D)
    assert torch.equal(bits(x[:, 0]), bits((cls + pos0).expand(B, D))), "CLS rows"
    assert torch.equal(bits(x[:, 1:]), bits(init[:, 1:])), "rows other than CLS changed"


@pytest.mark.parametrize("D", [4, 256, 1536])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_zero_padded_rows(lib, B, D):
    S = 7
    rows = B * S
    g = seed("zero_pad", B, D)
    init = nan_payloads(torch.randn(rows, D, device="cuda", generator=g), g)
    pad = torch.tensor([0, 1, 255], dtype=torch.uint8, device="cuda")[torch.randint(0, 3, (rows,), device="cuda", generator=g)]

    def launch():
        x, buf = tail(rows * D, float("nan"))
        x.copy_(init.view(-1))
        assert lib.opb_zero_padded_rows(x.data_ptr(), pad.data_ptr(), rows, D, stream()) == OK
        return {"x": (x, buf)}

    x, buf = twice(launch)["x"]
    assert_tail(x, buf, float("nan"), "zero_padded_rows")
    x = x.view(rows, D)
    z = pad != 0
    assert torch.equal(bits(x[z]), torch.zeros_like(bits(x[z]))), "pad rows are not +0.0"
    assert torch.equal(bits(x[~z]), bits(init[~z])), "live rows changed"


# --------------------------------------------------------------------------------------------------------------------
# relative-position tables: relpos_bias_build, relpos_lut_build, relpos_bias_block
# --------------------------------------------------------------------------------------------------------------------
RP_S = [1, 2, 17, 77, 257, 577, 785, 1025]


def bucket_cases(S):
    """(name, bucket view, table rows, heads): the text buckets (a [:S, :S] view of the 1024 x 1024 buffer) for S <= 1024, and
    for S = w * w + 1 the image buckets of window w (w = 16, 24, 28, 32: the one_piece_g_* ViTs) in a buffer 24 columns wider"""
    import restated
    out = []
    if S <= 1024:
        out.append(("text", restated.make_token_bucket_position(256).cuda(), 514, 5))
    w = int(round((S - 1) ** 0.5))
    if w >= 2 and w * w + 1 == S:
        b = restated.make_image_bucket_position(w).cuda()
        buf = torch.zeros(S, S + 24, dtype=torch.int64, device="cuda")
        buf[:, :S] = b
        out.append((f"image w={w}", buf[:, :S], (2 * w - 1) ** 2 + 3, 24))
    return out


@pytest.mark.parametrize("S", RP_S)
def test_relpos_bias_build(lib, S):
    for name, bucket, nb, H in bucket_cases(S):
        g = seed("relpos", S, name)
        table = followed_by_nan(torch.randn(nb, H, device="cuda", generator=g))
        for s_pad in sorted({S, (S + 7) // 8 * 8, (S + 7) // 8 * 8 + 12}):
            def launch():
                b, buf = tail(H * S * s_pad, float("nan"))
                assert lib.opb_relpos_bias_build(table.data_ptr(), bucket.data_ptr(), b.data_ptr(), S, s_pad, H, bucket.stride(0),
                                                 stream()) == OK
                return {"bias": (b, buf)}

            b, buf = twice(launch)["bias"]
            assert_tail(b, buf, float("nan"), f"relpos_bias_build {name} S={S}")
            want = R.relpos_bias_ref(table, bucket, S, s_pad)
            assert torch.equal(bits(b.view(H, S, s_pad)), bits(want)), f"relpos_bias_build {name} S={S} s_pad={s_pad}"


def lut_build(lib, table, idx):
    L, H = idx.numel(), table.shape[1]

    def launch():
        lut, buf = tail(H * L, float("nan"))
        assert lib.opb_relpos_lut_build(table.data_ptr(), idx.data_ptr(), lut.data_ptr(), L, H, stream()) == OK
        return {"lut": (lut, buf)}

    lut, buf = twice(launch)["lut"]
    assert_tail(lut, buf, float("nan"), "relpos_lut_build")
    return lut.view(H, L)


@pytest.mark.parametrize("L,H", [(1, 1), (255, 2), (257, 24), (1000, 3), (2049, 5)])
def test_relpos_lut_build(lib, L, H):
    g = seed("lut", L, H)
    table = followed_by_nan(torch.randn(300, H, device="cuda", generator=g))
    idx = torch.randint(0, 300, (L,), dtype=torch.int32, device="cuda", generator=g)
    idx[0] = 299
    assert torch.equal(bits(lut_build(lib, table, idx)), bits(R.relpos_lut_ref(table, idx)))


@pytest.mark.parametrize("S,w", [(384, 0), (197, 14), (257, 16)], ids=["text384", "image14", "image16"])
def test_relpos_lut_encodes_dense_table(lib, S, w):
    """lut[:, code_row[i] - code_col[j]] is the dense table of the same bucket, bit for bit"""
    import restated
    from one_peace_b200 import relpos
    H = 4
    g = seed("lut dense", S)
    if w:
        bucket, codes, nb = restated.make_image_bucket_position(w), relpos.image_codes(S, w), (2 * w - 1) ** 2 + 3
    else:
        bucket, codes, nb = restated.make_token_bucket_position(256)[:S, :S], relpos.text_codes(S), 514
    table = followed_by_nan(torch.randn(nb, H, device="cuda", generator=g))
    lut_idx, crow, ccol = (torch.from_numpy(a).cuda() for a in relpos.build_lut_index(bucket.numpy(), codes))
    lut = lut_build(lib, table, lut_idx.int().contiguous())
    dense = lut[:, (crow[:S, None] - ccol[None, :S]).long()]
    assert torch.equal(bits(dense), bits(table[bucket.cuda()].permute(2, 0, 1)))


@pytest.mark.parametrize("ids_kind", ["none", "ids", "ids_pad"])
@pytest.mark.parametrize("n", [1, 17, 130])
def test_relpos_bias_block(lib, n, ids_kind):
    """one modality's diagonal block of the bias canvas; the canvas outside every block stays NaN"""
    import restated
    bucket = restated.make_token_bucket_position(256).cuda()
    for Bb in (1, 5):
        for lo in (0, 21):
            for H in (1, 24):
                g = seed("block", n, ids_kind, Bb, lo, H)
                S = lo + n + 3
                s_pad = (S + 7) // 8 * 8 + 4
                table = followed_by_nan(torch.randn(514, H, device="cuda", generator=g))
                ids = None
                if ids_kind != "none":
                    buf = torch.randint(0, 300, (Bb, n + 3), device="cuda", generator=g)
                    if ids_kind == "ids_pad":
                        buf[:, n - min(n, 3):n] = -1
                        buf[:, torch.randint(0, n, (1,), device="cuda", generator=g)] = -1
                    ids = buf[:, :n]

                def launch():
                    canvas = torch.full((Bb, H, S, s_pad), float("nan"), device="cuda")
                    assert lib.opb_relpos_bias_block(table.data_ptr(), bucket.data_ptr(), bucket.stride(0),
                                                     ids.data_ptr() if ids is not None else None,
                                                     ids.stride(0) if ids is not None else 0, Bb, n, lo, canvas.data_ptr(), S,
                                                     s_pad, H, stream()) == OK
                    return {"canvas": (canvas, canvas)}

                canvas = twice(launch)["canvas"][0]
                want, written = R.relpos_bias_block_ref(table, bucket, ids, n, lo, torch.full_like(canvas, float("nan")))
                what = f"relpos_bias_block Bb={Bb} n={n} lo={lo} H={H} {ids_kind}"
                assert torch.equal(bits(canvas[written]), bits(want[written])), what + ": block"
                assert torch.equal(bits(canvas[~written]), bits(want[~written])), what + ": written outside the block"


# --------------------------------------------------------------------------------------------------------------------
# row_gather
# --------------------------------------------------------------------------------------------------------------------
RG_ROWS = [1, 7, 9, 12613]
ADD_PERIOD = 5                          # divides none of the row counts above 1


def row_gather_call(lib, src, idx, out, fill, add, period=None, dim=None):
    dim = src.shape[1] if dim is None else dim
    return lib.opb_row_gather(src.data_ptr(), int(src.dtype == BF16), src.stride(0), idx.data_ptr(),
                              fill.data_ptr() if fill is not None else None, add.data_ptr() if add is not None else None,
                              (ADD_PERIOD if period is None else period) if add is not None else 0, out.data_ptr(),
                              int(out.dtype == BF16), out.stride(0), idx.numel(), dim, stream())


@pytest.mark.parametrize("sdt,odt", [(F32, F32), (F32, BF16), (BF16, F32), (BF16, BF16)],
                         ids=["f32-f32", "f32-bf16", "bf16-f32", "bf16-bf16"])
@pytest.mark.parametrize("dim", [4, 132, 1536])
def test_row_gather(lib, dim, sdt, odt):
    n = 300
    g = seed("gather", dim, sdt, odt)
    src = gapped(n, dim, sdt, gap=4)
    src.copy_(torch.randn(n, dim, device="cuda", generator=g))
    src = src[:n - 1]                                               # the last buffer row (NaN gap only) is past the source
    fill = followed_by_nan(torch.randn(dim, device="cuda", generator=g) + 7.0)
    add = followed_by_nan(torch.randn(ADD_PERIOD, dim, device="cuda", generator=g))
    for rows in RG_ROWS:
        idx = torch.randint(-1, n - 1, (rows,), device="cuda", generator=g)
        idx[0] = -1 if rows > 1 else idx[0]
        idx[rows // 2:rows // 2 + 3] = n - 2                       # duplicates of the last source row
        for use_fill in (False, True):
            for use_add in (False, True):
                f, a = (fill if use_fill else None), (add if use_add else None)

                def launch():
                    out, buf = R.canary_out((rows, dim), ldo_extra=4, rows_before=2, rows_after=1, dtype=odt)
                    assert row_gather_call(lib, src, idx, out, f, a) == OK
                    return {"out": (out, buf)}

                out, buf = twice(launch)["out"]
                what = f"row_gather rows={rows} dim={dim} fill={use_fill} add={use_add}"
                R.assert_canary(buf, out, what=what)
                assert torch.equal(bits(out), bits(R.row_gather_ref(src, idx, odt, f, a))), what


def test_row_gather_refuses(lib):
    """misaligned pointers, dim or pitches not multiples of 4, a zero addend period and a bad dtype: OPB_ERR_INVALID and no
    store"""
    dim, rows = 64, 8
    src = torch.randn(16, dim + 8, device="cuda")
    src16 = src.bfloat16()
    idx = torch.arange(rows, device="cuda")
    fill = torch.randn(dim + 8, device="cuda")
    add = torch.randn(2 * dim + 8, device="cuda")
    buf = torch.full((rows + 1, dim + 8), float("nan"), device="cuda")
    out = buf[:rows, :dim]
    s = stream()
    p = lambda t, off=0: t.data_ptr() + off * t.element_size()
    bad = [
        (p(src, 1), 0, dim + 8, p(fill), p(add), 1, p(out), 0, dim + 8, dim),          # src 4 bytes off
        (p(src16, 4), 1, dim + 8, p(fill), p(add), 1, p(out), 0, dim + 8, dim),        # bf16 src 8 bytes off
        (p(src), 0, dim + 8, p(fill, 2), p(add), 1, p(out), 0, dim + 8, dim),          # fill 8 bytes off
        (p(src), 0, dim + 8, p(fill), p(add, 1), 1, p(out), 0, dim + 8, dim),          # add 4 bytes off
        (p(src), 0, dim + 8, p(fill), p(add), 1, p(buf, 2), 0, dim + 8, dim),          # out 8 bytes off
        (p(src), 0, dim + 8, None, None, 0, p(out), 0, dim + 8, dim - 2),              # dim % 4 != 0
        (p(src), 0, dim + 6, None, None, 0, p(out), 0, dim + 8, dim),                  # ld_src % 4 != 0
        (p(src), 0, dim + 8, None, None, 0, p(out), 0, dim + 6, dim),                  # ld_out % 4 != 0
        (p(src), 0, dim + 8, None, p(add), 0, p(out), 0, dim + 8, dim),                # addend without a period
        (p(src), 2, dim + 8, None, None, 0, p(out), 0, dim + 8, dim),                  # no such dtype
        (p(src), 0, dim + 8, None, None, 0, p(out), 0, dim + 8, 0),                    # no columns
    ]
    for a in bad:
        assert lib.opb_row_gather(a[0], a[1], a[2], idx.data_ptr(), a[3], a[4], a[5], a[6], a[7], a[8], rows, a[9], s) == INVALID, a
    assert lib.opb_row_gather(p(src), 0, dim + 8, idx.data_ptr(), None, None, 0, p(out), 0, dim + 8, 0, dim, s) == INVALID
    torch.cuda.synchronize()
    assert torch.isnan(buf).all(), "a refused call wrote its output"


# --------------------------------------------------------------------------------------------------------------------
# l2_normalize_rows
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 31, 256, 257, 768, 1536, 4096])
def test_l2_normalize_rows(lib, ratios, D):
    """rows scaled by 10^6 and 10^-6, a zero row, a row below the 1e-12 clamp, a single non-zero entry, N(0, 1) rows"""
    rows = 24
    g = seed("l2", D)
    x0 = torch.randn(rows, D, device="cuda", generator=g) * (0.5 + torch.rand(rows, 1, device="cuda", generator=g))
    x0[1] *= 1e6
    x0[2] *= 1e-6
    x0[3] = 0.0
    x0[4] *= 1e-15                                                 # |x| <= 1e-15 sqrt(D) * 4 < 1e-12
    x0[5] = 0.0
    x0[5, D // 3] = -3.7
    x0[6] = -0.0
    x = gapped(rows, D, F32)
    x.copy_(x0)

    def launch():
        y, yb = R.canary_out((rows, D), rows_before=1, rows_after=2)
        y16, y16b = R.canary_out((rows, D), rows_before=1, rows_after=2, dtype=BF16)
        assert lib.opb_l2_normalize_rows(x.data_ptr(), x.stride(0), y.data_ptr(), y16.data_ptr(), rows, D, stream()) == OK
        return {"y": (y, yb), "y16": (y16, y16b)}

    got = twice(launch)
    y, y16 = got["y"][0], got["y16"][0]
    R.assert_canary(got["y"][1], y, what=f"l2_normalize D={D} y")
    R.assert_canary(got["y16"][1], y16, what=f"l2_normalize D={D} y_bf16")
    ref, bound = R.l2_normalize_ref(x)
    note(ratios, "l2_normalize_rows y", R.assert_within(y, ref, bound, 1.0, F32, extra=None, what=f"l2_normalize D={D}"))
    assert torch.equal(bits(y16), bits(y.bfloat16())), "y_bf16 is not bf16(y)"
    assert (y[3] == 0).all() and (y[6] == 0).all(), "zero row"
    assert (y[5] != 0).sum() == 1 and y[5, D // 3] < 0, "single non-zero entry"
    # no y_bf16: same y
    y2, y2b = R.canary_out((rows, D), rows_before=1, rows_after=2)
    assert lib.opb_l2_normalize_rows(x.data_ptr(), x.stride(0), y2.data_ptr(), None, rows, D, stream()) == OK
    assert torch.equal(bits(y2b), bits(got["y"][1])), "y differs without the bf16 copy"


# --------------------------------------------------------------------------------------------------------------------
# transpose_bf16
# --------------------------------------------------------------------------------------------------------------------
# (rows, cols, ld_in, input offset, output offset) in elements.  Vectorised path: rows, cols and ld multiples of 8 and both
# bases 16-byte aligned; the scalar path: each of those broken in turn.
TR_VEC = [(8, 8, 8, 0, 0), (64, 64, 64, 0, 0), (72, 136, 144, 8, 0), (200, 64, 72, 0, 8), (12608, 1536, 1536, 0, 0)]
TR_SCALAR = [(1, 1, 1, 0, 0), (65, 63, 63, 0, 0), (12, 64, 64, 0, 0), (64, 60, 64, 0, 0), (64, 64, 68, 0, 0),
             (64, 64, 64, 1, 0), (64, 64, 64, 0, 1), (130, 200, 203, 3, 5), (12613, 1536, 1536, 0, 0)]


@pytest.mark.parametrize("case", TR_VEC + TR_SCALAR, ids=[f"{'vec' if c in TR_VEC else 'scalar'}-{c[0]}x{c[1]}-ld{c[2]}-o{c[3]}-{c[4]}"
                                                        for c in TR_VEC + TR_SCALAR])
def test_transpose_bf16(lib, case):
    rows, cols, ld, off_in, off_out = case
    g = seed("transpose", *case)
    src = torch.full((rows * ld + off_in + 16,), float("nan"), dtype=BF16, device="cuda")
    x = src.as_strided((rows, cols), (ld, 1), off_in)
    x.copy_(torch.randn(rows, cols, device="cuda", generator=g))

    def launch():
        buf = torch.full((cols * rows + off_out + 64,), float("nan"), dtype=BF16, device="cuda")
        out = buf[off_out:off_out + cols * rows]
        assert lib.opb_transpose_bf16(x.data_ptr(), ld, out.data_ptr(), rows, cols, stream()) == OK
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    assert torch.equal(bits(out.view(cols, rows)), bits(R.transpose_ref(x))), f"transpose {case}"
    outside = torch.cat([buf[:off_out], buf[off_out + cols * rows:]])
    assert torch.isnan(outside).all() and torch.equal(bits(outside), bits(torch.full_like(outside, float("nan")))), \
        f"transpose {case}: written outside the output"


def test_transpose_refuses(lib):
    x = torch.zeros(8, 8, dtype=BF16, device="cuda")
    out = torch.full((64,), float("nan"), dtype=BF16, device="cuda")
    for rows, cols, ld in ((0, 8, 8), (8, 0, 8), (8, 8, 7)):
        assert lib.opb_transpose_bf16(x.data_ptr(), ld, out.data_ptr(), rows, cols, stream()) == INVALID
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


@pytest.mark.parametrize("M", [13, 16, 12613])
def test_tr_zero_pads_m(M):
    """autograd._tr: [M, n] -> [n, pad8(M)] with zero columns past M (the K-major dW operand)"""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200.autograd import _tr
    n = 264
    x = torch.randn(M, n, device="cuda", generator=seed("tr", M)).bfloat16()
    want = torch.zeros((M + 7) // 8 * 8, n, dtype=BF16, device="cuda")
    want[:M] = x
    assert torch.equal(bits(_tr(x)), bits(want.t().contiguous()))


# --------------------------------------------------------------------------------------------------------------------
# topk10_rows, recall_hits
# --------------------------------------------------------------------------------------------------------------------
TOPK_C = [1, 9, 10, 11, 31, 32, 33, 1003, 25010]
VAL_FILL = 0x7FBADBAD                   # a NaN payload no kernel writes


def topk_rows_data(R_, C, kind, g):
    """'ties': values from a set of six, so that ties fall within a lane (columns c and c + 32) and across lanes;
    'special': the same with -inf, +inf, NaN (of both signs) and signed zeros, and rows that are all -inf, all NaN, all
    equal, or hold fewer than 10 entries above -inf"""
    vals = torch.tensor([-1.5, -0.5, 0.0, 0.5, 1.5, 2.5], device="cuda")
    x = vals[torch.randint(0, 6, (R_, C), device="cuda", generator=g)]
    if kind == "special":
        p = torch.rand(R_, C, device="cuda", generator=g)
        x[p < 0.3] = float("-inf")
        x[(p >= 0.3) & (p < 0.33)] = float("nan")
        x[(p >= 0.33) & (p < 0.35)] = -0.0
        x[(p >= 0.35) & (p < 0.36)] = float("inf")
        x.view(torch.int32)[(p >= 0.36) & (p < 0.37)] = 0xFFC00001 - 2 ** 32
        x[0] = float("-inf")
        if R_ > 4:
            x[1] = float("nan")
            x[2] = 0.5
            x[3] = float("-inf")
            x[3, C // 2] = 1.0
            x[3, C - 1] = float("nan")
            x[4] = float("-inf")
            x[4, torch.randperm(C, device="cuda", generator=g)[:min(C, 7)]] = -0.0
    return x


def topk_launch(lib, sim, R_, C):
    def launch():
        idx, ib = tail(R_ * 10, -7, torch.int32)
        val, vb = tail(R_ * 10, 0.0)
        vb.view(torch.int32).fill_(VAL_FILL)
        assert lib.opb_topk10_rows(sim.data_ptr(), sim.stride(0), idx.data_ptr(), val.data_ptr(), R_, C, stream()) == OK
        return {"idx": (idx, ib), "val": (val, vb)}
    return twice(launch)


@pytest.mark.parametrize("layout", ["contig", "pitch"])
@pytest.mark.parametrize("kind", ["ties", "special"])
@pytest.mark.parametrize("C", TOPK_C)
def test_topk10_rows(lib, C, kind, layout):
    """indices and values bit for bit against the total-order top-10 (NaN by isnan); a row pitch wider than C with NaN in
    the gap, which would rank first if it were read"""
    R_ = 5000 if C <= 1003 else 2000
    g = seed("topk", C, kind, layout)
    x = topk_rows_data(R_, C, kind, g)
    sim = x if layout == "contig" else gapped(R_, C, F32, gap=3)
    if layout == "pitch":
        sim.copy_(x)
    got = topk_launch(lib, sim, R_, C)
    idx, val = got["idx"][0].view(R_, 10), got["val"][0].view(R_, 10)
    assert_tail(*got["idx"], -7, "topk10 idx")
    assert torch.equal(got["val"][1][R_ * 10:].view(torch.int32), torch.full((64,), VAL_FILL, dtype=torch.int32, device="cuda")), \
        "topk10 val: written past the end"
    want_i, want_v = R.topk10_ref(x)
    bad = (idx != want_i).any(1)
    if bad.any():
        r = int(bad.nonzero()[0])
        raise AssertionError(f"topk10 C={C} {kind} {layout}: {int(bad.sum())} of {R_} rows differ; row {r}: got "
                             f"{idx[r].tolist()}, want {want_i[r].tolist()}; row values {x[r, :min(C, 40)].tolist()}")
    nan_g, nan_w = torch.isnan(val), torch.isnan(want_v)
    assert torch.equal(nan_g, nan_w), "topk10 values: NaN placement"
    assert torch.equal(bits(val[~nan_g]), bits(want_v[~nan_w])), "topk10 values"


def test_topk10_retrieval_shape(lib):
    """the COCO evaluation shape, 5000 x 25010, N(0, 1) with a block of planted ties: equals the reference and torch.topk"""
    R_, C = 5000, 25010
    g = seed("topk coco")
    x = torch.randn(R_, C, device="cuda", generator=g)
    x[:100, 3000:3100] = 9.0
    got = topk_launch(lib, x, R_, C)
    want_i, want_v = R.topk10_ref(x)
    assert torch.equal(got["idx"][0].view(R_, 10), want_i) and torch.equal(got["val"][0].view(R_, 10), want_v)
    tv, ti = x[100:].topk(10, dim=1)
    assert torch.equal(want_i[100:].long(), ti) and torch.equal(want_v[100:], tv)


def test_topk10_refuses(lib):
    sim = torch.zeros(4, 16, device="cuda")
    idx = torch.full((64,), -7, dtype=torch.int32, device="cuda")
    for R_, C, ld in ((0, 16, 16), (4, 0, 16), (4, 16, 15)):
        assert lib.opb_topk10_rows(sim.data_ptr(), ld, idx.data_ptr(), None, R_, C, stream()) == INVALID
    torch.cuda.synchronize()
    assert (idx == -7).all()


@pytest.mark.parametrize("R_", [1, 31, 33, 257, 5000])
def test_recall_hits(lib, R_):
    """duplicate candidate ids, planted hits at every rank, -1 ranks (never a hit)"""
    C = 600
    g = seed("hits", R_)
    cand = torch.randint(0, 40, (C,), device="cuda", generator=g)
    own = torch.randint(0, 40, (R_,), device="cuda", generator=g)
    idx = torch.randint(0, C, (R_, 10), device="cuda", generator=g, dtype=torch.int32)
    idx[torch.rand(R_, 10, device="cuda", generator=g) < 0.2] = -1
    idx[0, :] = -1
    plant = torch.rand(R_, device="cuda", generator=g) < 0.5
    where = torch.randint(0, 10, (R_,), device="cuda", generator=g)
    hit_col = (cand[None, :] == own[:, None]).int().argmax(1)                  # a candidate with the row's id (if any)
    rows = plant.nonzero().squeeze(1)
    idx[rows, where[rows]] = hit_col[rows].int()
    idx = idx.contiguous()

    def launch():
        hits, hb = tail(3, -5, torch.int32)
        hits.zero_()
        assert lib.opb_recall_hits(idx.data_ptr(), cand.data_ptr(), own.data_ptr(), R_, hits.data_ptr(), stream()) == OK
        return {"hits": (hits, hb)}

    hits, hb = twice(launch)["hits"]
    assert_tail(hits, hb, -5, "recall_hits")
    assert hits.tolist() == R.recall_hits_ref(idx, cand, own)


# --------------------------------------------------------------------------------------------------------------------
# Recall end to end
# --------------------------------------------------------------------------------------------------------------------
def test_recall_end_to_end(lib):
    """synthetic retrieval set plus planted near-duplicates (texts within 1e-7 of another text, one image twice under two
    ids): each direction's ranking passes ``topk_within`` and Recall@{1,5,10} is within the near-tie rows of the fp64
    counts"""
    import synth
    from one_peace_b200 import kernels as K
    from one_peace_b200.metrics import Recall
    img, txt, img_ids, txt_ids = synth.retrieval_set(300, 5, 256, seed=12, noise=1.6)
    g = torch.Generator().manual_seed(13)
    txt[1:200:7] = txt[0:200:7][:txt[1:200:7].shape[0]] + 1e-7 * torch.randn(txt[1:200:7].shape, generator=g)
    img[5] = img[4]
    rec = Recall()
    rec.initialize(txt_ids.cuda(), txt.cuda())
    for lo in range(0, img.shape[0], 64):
        rec.compute(img_ids[lo:lo + 64].cuda(), img[lo:lo + 64].cuda())
    log = rec.merge_results()
    for a, b, a_ids, b_ids, key in ((img, txt, img_ids, txt_ids, "txt"), (txt, img, txt_ids, img_ids, "img")):
        A, B = a.cuda().double(), b.cuda().double()
        z, dz = A @ B.t(), R.Z_TAU * (A.abs() @ B.abs().t())
        rank = K.topk10_rows(Recall._similarity(a.cuda(), b.cuda()))
        ok = R.topk_within(z, dz, rank)
        assert ok.all(), f"{key}: {int((~ok).sum())} rows ranked outside the logit error"
        hits, near = R.recall_ref(z, dz, b_ids.cuda(), a_ids.cuda())
        for k, h, nr in zip((1, 5, 10), hits, near):
            got = round(log[f"{key}_r{k}"] * a.shape[0] / 100)
            assert abs(got - h) <= nr, (key, k, got, h, nr)
