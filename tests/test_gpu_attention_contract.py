"""GPU: the contract of the attention kernels (csrc/attention.cu, csrc/attention_bwd.cu) for every bias form, forward and
backward, element by element against the fp64 references of tests/kernel_ref.py (module docstring, "Attention").

Forms: the dense fp32 table shared by the batch (``attention`` / ``attention_bwd``), one table per sample, the LUT form
(``attention_tc``, text and image codes), the two-segment LUT of a concatenated sequence, and the transposed half2 tables
of the backward (``attention_bwd_t``, accumulated over two launches, folded and centred as the training stack does).
Dense tables carry NaN in their pad columns [S, s_pad), which must never reach a result or be written.  Outputs are views
into NaN buffers with spare rows or a NaN tail, so a store outside the logical output or a skipped store shows up.  Every
launch runs twice and must repeat bit for bit, except the bias gradient, which is summed with fp32 atomics in no fixed
order.  Forms that read the same fp32 values must agree bit for bit."""
import zlib

import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
Q_SCALE = 0.125


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def ratios():
    """largest fraction of the bound used, per form and output (printed at the end of the module; run with -s)"""
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


def same_bits(a, b, what):
    for name in a:
        assert torch.equal(bits(a[name][1]), bits(b[name][1])), f"{what}: {name} differs"


def seed(*key):
    g = torch.Generator(device="cuda")
    return g.manual_seed(zlib.crc32("/".join(map(str, key)).encode()))


def nan_tail(n, extra=64):
    buf = torch.full((n + extra,), float("nan"), device="cuda")
    return buf[:n], buf


def assert_tail(view, buf, what):
    n = view.numel()
    assert torch.isnan(buf[n:]).all() and torch.equal(bits(buf[n:]), bits(torch.full_like(buf[n:], float("nan")))), \
        f"{what}: written past the end"
    assert torch.isfinite(view).all(), f"{what}: not every element written"


def s_pad_for(S, variant):
    """row pitch of a dense table: S rounded up to 4, to 8, or to 8 plus 12 columns"""
    return [(S + 3) // 4 * 4, (S + 7) // 8 * 8, (S + 7) // 8 * 8 + 12][variant % 3]


def key_pad(B, S, kind):
    """none, or right padding of a different length per sample: the first padded key odd (a live / padded pair), only
    key 0 (CLS) live, and padding that covers whole 64-key blocks"""
    if kind == "none":
        return None
    kp = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
    live = [S - 1 if (S - 1) % 2 else S - 2, 1, ((S - 1) // 64 - 1) * 64]
    for b in range(B):
        kp[b, max(1, live[b % 3]):] = 1
    return kp


def make_bias(shape, S, kind, g):
    """logical fp32 bias: N(0, 1), or the stress case: |b| <= 16, rising along the keys so that a row's maximum lies in
    its last live key block (every new block rescales o and l; early blocks fall to tiny weights)"""
    if kind == "normal":
        return torch.randn(*shape, device="cuda", generator=g)
    ramp = 32.0 * (torch.arange(S, device="cuda") + 0.5) / S - 16.0
    return (ramp + torch.randn(*shape, device="cuda", generator=g)).clamp(-16.0, 16.0)


def dense_table(logical, s_pad):
    """(..., S, s_pad) fp32 table holding `logical` with NaN in the pad columns"""
    t = torch.full((*logical.shape[:-1], s_pad), float("nan"), device="cuda")
    t[..., :logical.shape[-1]] = logical
    return t


def make_qkv(B, S, H, g):
    return (torch.randn(B * S, 3 * H * 64, device="cuda", generator=g) * 0.5).bfloat16()


# --------------------------------------------------------------------------------------------------------------------
# forward
# --------------------------------------------------------------------------------------------------------------------
def fwd_launch(call, B, S, H):
    """call(out, lse, ln_stats) on fresh canary buffers -> {name: (view, buffer)}"""
    out, ob = R.canary_out((B * S, H * 64), rows_before=2, rows_after=2, dtype=BF16)
    lse, lb = nan_tail(B * H * S)
    st, sb = nan_tail(H * B * S * 2)
    call(out, lse, st)
    return {"out": (out, ob), "lse": (lse, lb), "ln_stats": (st, sb)}


def check_fwd(ratios, family, got, ref, B, S, H):
    out, ob = got["out"]
    R.assert_canary(ob, out, what=f"{family} out")
    assert_tail(*got["lse"], f"{family} lse")
    assert_tail(*got["ln_stats"], f"{family} ln_stats")
    note(ratios, f"{family} out", R.assert_within(out, ref.out, ref.out_err, 1.0, BF16, what=f"{family} out"))
    note(ratios, f"{family} lse", R.assert_within(got["lse"][0].view(B, H, S), ref.lse, ref.dlse, 1.0, F32, what=f"{family} lse"))
    note(ratios, f"{family} ln_stats", R.assert_within(got["ln_stats"][0].view(H, B * S, 2), ref.stats, ref.stats_err, 1.0, F32,
                                                       what=f"{family} ln_stats"))


def run_dense(K, qkv, table, kp, B, S, H):
    return twice(lambda: fwd_launch(lambda o, l, s: K.attention(qkv, table, kp, B, S, H, out=o, lse=l, ln_stats=s), B, S, H))


FWD_S = [2, 17, 63, 64, 65, 197, 224, 225, 257, 321, 384, 385, 750]
VIT_S = [577, 785, 1025]            # the 384^2, 448^2 and 512^2 ViTs (w = 24, 28, 32): dense tables only


@pytest.mark.parametrize("bias_kind", ["normal", "stress"])
@pytest.mark.parametrize("pad", ["none", "right"])
@pytest.mark.parametrize("S", FWD_S + VIT_S)
def test_forward_dense(K, ratios, S, pad, bias_kind):
    """shared table; the same table replicated per sample must give the same bits"""
    B, H = 3, 2
    g = seed("dense", S, pad, bias_kind)
    qkv, kp = make_qkv(B, S, H, g), key_pad(B, S, pad)
    bias = make_bias((H, S, S), S, bias_kind, g)
    table = dense_table(bias, s_pad_for(S, (FWD_S + VIT_S).index(S)))
    got = run_dense(K, qkv, table, kp, B, S, H)
    check_fwd(ratios, f"dense {bias_kind}", got, R.attention_ref(qkv, bias, kp, B, S, H), B, S, H)
    rep = table[None].repeat(B, 1, 1, 1).contiguous()
    same_bits(got, run_dense(K, qkv, rep, kp, B, S, H), "shared vs replicated per-sample table")


@pytest.mark.parametrize("pad", ["none", "right"])
@pytest.mark.parametrize("S", FWD_S)
def test_forward_per_sample(K, ratios, S, pad):
    B, H = 3, 2
    g = seed("per_sample", S, pad)
    qkv, kp = make_qkv(B, S, H, g), key_pad(B, S, pad)
    bias = make_bias((B, H, S, S), S, "normal", g)
    table = dense_table(bias, s_pad_for(S, FWD_S.index(S) + 1))
    got = run_dense(K, qkv, table, kp, B, S, H)
    check_fwd(ratios, "per-sample", got, R.attention_ref(qkv, bias, kp, B, S, H), B, S, H)


def lut_form(K, S, H, g):
    """RelPosBias in LUT form for S (image codes when S = w * w + 1, text codes otherwise) and the (H,S,S) bias it encodes"""
    import restated
    from one_peace_b200 import relpos
    w = int(round((S - 1) ** 0.5))
    if S > 2 and w * w + 1 == S:
        bucket, codes, ntab = restated.make_image_bucket_position(w), relpos.image_codes(S, w), (2 * w - 1) ** 2 + 3
    else:
        bucket, codes, ntab = restated.make_token_bucket_position(256)[:S, :S], relpos.text_codes(S), 514
    table = torch.randn(ntab, H, device="cuda", generator=g)
    li = relpos.build_lut_index(bucket.numpy(), codes)
    lut_idx, crow, ccol = (torch.from_numpy(a).cuda() for a in li)
    rp = K.RelPosBias(lut=K.relpos_lut_build(table, lut_idx), code_row=crow, code_col=ccol)
    dense = rp.lut[:, (crow[:S, None] - ccol[None, :S]).long()]
    assert torch.equal(dense, table[bucket.cuda()].permute(2, 0, 1))
    return rp, dense


def run_lut(K, qkv, rp, kp, B, S, H):
    return twice(lambda: fwd_launch(lambda o, l, s: K.attention_tc(qkv, rp, kp, B, S, H, out=o, lse=l, ln_stats=s), B, S, H))


@pytest.mark.parametrize("pad", ["none", "right"])
@pytest.mark.parametrize("S", FWD_S)
def test_forward_lut(K, ratios, S, pad):
    """LUT form; the dense table of the same values must give the same bits"""
    B, H = 3, 2
    g = seed("lut", S, pad)
    qkv, kp = make_qkv(B, S, H, g), key_pad(B, S, pad)
    rp, dense = lut_form(K, S, H, g)
    got = run_lut(K, qkv, rp, kp, B, S, H)
    check_fwd(ratios, "lut", got, R.attention_ref(qkv, dense, kp, B, S, H), B, S, H)
    same_bits(got, run_dense(K, qkv, dense_table(dense, s_pad_for(S, 1)), kp, B, S, H), "LUT vs dense table")


@pytest.mark.parametrize("S1,w", [(21, 6), (17, 14), (28, 14), (187, 14)])     # S = 58, 214, 225, 384
def test_forward_two_segment(K, ratios, S1, w):
    """concatenated text + image sequence: block-diagonal LUT bias, text keys padded just before the image segment;
    its dense block canvas must give the same bits"""
    import restated
    from one_peace_b200 import relpos
    B, H = 3, 2
    S2 = w * w + 1
    S = S1 + S2
    g = seed("two_segment", S1, w)
    b1 = restated.make_token_bucket_position(256)[:S1, :S1]
    b2 = restated.make_image_bucket_position(w)
    t1 = torch.randn(514, H, device="cuda", generator=g)
    t2 = torch.randn((2 * w - 1) ** 2 + 3, H, device="cuda", generator=g)
    rp = K.build_segmented_lut([(t1, relpos.build_lut_index(b1.numpy(), relpos.text_codes(S1)), S1),
                                (t2, relpos.build_lut_index(b2.numpy(), relpos.image_codes(S2, w)), S2)], "cuda")
    canvas = torch.zeros(H, S, S, device="cuda")
    canvas[:, :S1, :S1] = t1[b1.cuda()].permute(2, 0, 1)
    canvas[:, S1:, S1:] = t2[b2.cuda()].permute(2, 0, 1)
    kp = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
    for b, n in enumerate([0, 3, S1 - 1]):          # the last sample keeps only CLS of the text segment
        kp[b, S1 - n:S1] = 1
    qkv = make_qkv(B, S, H, g)
    got = run_lut(K, qkv, rp, kp, B, S, H)
    check_fwd(ratios, "two-segment", got, R.attention_ref(qkv, canvas, kp, B, S, H), B, S, H)
    same_bits(got, run_dense(K, qkv, dense_table(canvas, s_pad_for(S, 2)), kp, B, S, H), "two-segment LUT vs its canvas")


@pytest.mark.parametrize("form", ["dense", "lut"])
def test_forward_production_shape(K, ratios, form):
    """the 4B vision shape, B = 64, S = 197, H = 24"""
    B, S, H = 64, 197, 24
    g = seed("production", form)
    qkv = make_qkv(B, S, H, g)
    rp, dense = lut_form(K, S, H, g)
    if form == "dense":
        got = run_dense(K, qkv, dense_table(dense, s_pad_for(S, 1)), None, B, S, H)
    else:
        got = run_lut(K, qkv, rp, None, B, S, H)
    check_fwd(ratios, f"{form} B=64 H=24", got, R.attention_ref(qkv, dense, None, B, S, H), B, S, H)


def test_forward_vit_512_shape(K, ratios):
    """the 512^2 ViT shape (one_piece_g_512): B = 1, S = 1025, H = 24, the dense table of the w = 32 image buckets"""
    import restated
    B, S, H, w = 1, 1025, 24, 32
    g = seed("vit 512")
    qkv = make_qkv(B, S, H, g)
    table = torch.randn((2 * w - 1) ** 2 + 3, H, device="cuda", generator=g)
    bias = table[restated.make_image_bucket_position(w).cuda()].permute(2, 0, 1).contiguous()
    got = run_dense(K, qkv, dense_table(bias, s_pad_for(S, 1)), None, B, S, H)
    check_fwd(ratios, "dense B=1 H=24 S=1025", got, R.attention_ref(qkv, bias, None, B, S, H), B, S, H)


# --------------------------------------------------------------------------------------------------------------------
# backward
# --------------------------------------------------------------------------------------------------------------------
def forward_for_bwd(K, qkv, table, kp, B, S, H):
    out = torch.empty(B * S, H * 64, dtype=BF16, device="cuda")
    lse = torch.empty(B * H * S, device="cuda")
    K.attention(qkv, table, kp, B, S, H, out=out, lse=lse)
    return out, lse


def dqkv_canary(B, S, H):
    return R.canary_out((B * S, 3 * H * 64), rows_before=2, rows_after=2, dtype=BF16)


def check_dqkv(ratios, family, dqkv, buf, br):
    R.assert_canary(buf, dqkv, what=f"{family} dqkv")
    note(ratios, f"{family} dqkv", R.assert_within(dqkv, br.dqkv, br.dqkv_err, 1.0, BF16, what=f"{family} dqkv"))


def check_dbias(ratios, family, table, ref, err):
    """finite inside S x S and within the bound, pad columns never written"""
    S, s_pad = table.shape[-2], table.shape[-1]
    flat = table.view(-1, s_pad)
    R.assert_canary(flat, flat[:, :S], what=f"{family} dbias")
    note(ratios, f"{family} dbias", R.assert_within(table[..., :S], ref, err, 1.0, F32, what=f"{family} dbias"))


def bwd_dense_case(K, ratios, family, B, S, H, bias, table, kp, g):
    """attention_bwd with a dense table (shared or per sample) -> dqkv view (for the cross-form comparison)"""
    qkv = make_qkv(B, S, H, g)
    out, lse = forward_for_bwd(K, qkv, table, kp, B, S, H)
    d_out = (torch.randn(B * S, H * 64, device="cuda", generator=g) * 0.5).bfloat16()
    init = 0.01 * torch.randn(bias.shape, device="cuda", generator=g)
    dbias = []

    def launch():
        dq, buf = dqkv_canary(B, S, H)
        db = dense_table(init, table.shape[-1])
        K.attention_bwd(qkv, out, d_out, table, kp, lse, dq, db, B, S, H, Q_SCALE)
        dbias.append(db)
        return {"dqkv": (dq, buf)}

    got = twice(launch)            # dqkv bit-repeatable; dbias is summed with fp32 atomics, so only each run is checked
    br = R.attention_bwd_ref(qkv, out, d_out, lse, bias, kp, B, S, H, Q_SCALE)
    check_dqkv(ratios, family, *got["dqkv"], br)
    ref, err = R.dbias_ref(br, init, per_sample=bias.dim() == 4)
    for db in dbias:
        check_dbias(ratios, family, db, ref, err)
    return qkv, out, d_out, lse, got


@pytest.mark.parametrize("bias_kind", ["normal", "stress"])
@pytest.mark.parametrize("S", [17, 65, 197, 225, 385, 750] + VIT_S)
def test_backward_dense(K, ratios, S, bias_kind):
    """shared table; the same table replicated per sample must give the same dqkv bits"""
    B, H = 3, 2
    g = seed("bwd dense", S, bias_kind)
    kp = key_pad(B, S, "right")
    bias = make_bias((H, S, S), S, bias_kind, g)
    table = dense_table(bias, s_pad_for(S, S))
    qkv, out, d_out, lse, got = bwd_dense_case(K, ratios, f"bwd dense {bias_kind}", B, S, H, bias, table, kp, g)
    rep = table[None].repeat(B, 1, 1, 1).contiguous()
    dq, buf = dqkv_canary(B, S, H)
    K.attention_bwd(qkv, out, d_out, rep, kp, lse, dq, torch.zeros_like(rep), B, S, H, Q_SCALE)
    assert torch.equal(bits(buf), bits(got["dqkv"][1])), "shared vs replicated per-sample table: dqkv differs"


@pytest.mark.parametrize("S", [45, 197])
def test_backward_per_sample(K, ratios, S):
    B, H = 3, 2
    g = seed("bwd per-sample", S)
    kp = key_pad(B, S, "right")
    bias = make_bias((B, H, S, S), S, "normal", g)
    bwd_dense_case(K, ratios, "bwd per-sample", B, S, H, bias, dense_table(bias, s_pad_for(S, S)), kp, g)


@pytest.mark.parametrize("bias_kind", ["normal", "stress"])
@pytest.mark.parametrize("S", [2, 17, 64, 65, 197, 224])
def test_backward_transposed(K, ratios, S, bias_kind):
    """attention_bwd_t twice into one dbias_t, then fold and centre (EncoderStackFn.backward).  The logits carry the fp16
    error of the tables (2^-11 |b|), which the stress case (|b| up to 16) makes visible."""
    B, H = 3, 2
    g = seed("bwd transposed", S, bias_kind)
    kp = key_pad(B, S, "right")
    bias = make_bias((H, S, S), S, bias_kind, g)
    table = dense_table(bias, s_pad_for(S, S))
    qkv = make_qkv(B, S, H, g)
    out, lse = forward_for_bwd(K, qkv, table, kp, B, S, H)
    d_out = (torch.randn(B * S, H * 64, device="cuda", generator=g) * 0.5).bfloat16()
    bias_t = K.relpos_bias_transpose(table)
    dbias_t = torch.zeros(H, K.BIAS_T_KEYS, K.BIAS_T_Q, device="cuda")

    def launch():
        dq, buf = dqkv_canary(B, S, H)
        K.attention_bwd_t(qkv, out, d_out, bias_t, kp, lse, dq, dbias_t, B, S, H, Q_SCALE)
        return {"dqkv": (dq, buf)}

    got = twice(launch)
    assert not dbias_t[:, S:].any() and not dbias_t[:, :, S:].any(), "dbias_t written outside its S x S corner"
    init = 0.01 * torch.randn(H, S, S, device="cuda", generator=g)
    dbias = dense_table(init, table.shape[-1])
    K.relpos_dbias_fold(dbias_t, dbias)
    K.relpos_dbias_center(dbias)
    br = R.attention_bwd_ref(qkv, out, d_out, lse, bias, kp, B, S, H, Q_SCALE, eps_b=R.EPS_B_HALF)
    family = f"bwd transposed {bias_kind}"
    check_dqkv(ratios, family, *got["dqkv"], br)
    check_dbias(ratios, family, dbias, *R.center_ref(*R.dbias_ref(br, init, launches=2)))


def test_backward_transposed_rejects_long_sequences(K):
    """S > 224 does not fit the transposed tables: the call raises and launches nothing"""
    B, S, H = 1, 225, 2
    g = seed("bwd reject")
    qkv = make_qkv(B, S, H, g)
    out = torch.zeros(B * S, H * 64, dtype=BF16, device="cuda")
    lse = torch.zeros(B * H * S, device="cuda")
    bias_t = torch.zeros(H, K.BIAS_T_KEYS, K.BIAS_T_Q // 2, dtype=torch.int32, device="cuda")
    dbias_t = torch.zeros(H, K.BIAS_T_KEYS, K.BIAS_T_Q, device="cuda")
    dq, buf = dqkv_canary(B, S, H)
    with pytest.raises(RuntimeError):
        K.attention_bwd_t(qkv, out, out, bias_t, None, lse, dq, dbias_t, B, S, H, Q_SCALE)
    torch.cuda.synchronize()
    assert torch.isnan(buf).all(), "a rejected call wrote dqkv"
