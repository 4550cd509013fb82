"""GPU: the convolution forms of the wgmma GEMM (csrc/gemm_wgmma.cu) against the fp64 reference of tests/kernel_ref.py,
element by element (|err| <= tau * mag + extra + u_out * |ref|, tau = 2^-16), as the adapters lower them:

* the grouped sliding window (``grouped_conv1d``, the audio positional encoder): the 3-D A tensor map with taps > 1, the
  k-block / tap wrap, the per-group A column and B row offsets, the group-major tile order and the epilogue that keeps
  n_per_group < 256 columns of each tile, at the production geometry (c_pad = 128, two k-blocks per tap) and its edges;
* the same convolution lowered the training way (``window_gather`` and one plain GEMM per group into column slices);
* overlapping strided rows (the feature-extractor convolutions read A at a row pitch below K);
* narrow K (K < 64, one zero-filled k-block): the audio frame conv and the image stem, with the im2col kernels that feed
  them checked bit for bit.

Every GEMM writes into a NaN-canary output (spare rows around it, a wider row pitch) and runs twice; the two runs must be
bit-identical.  Operands are views into NaN-filled buffers where the kernel must not read past them."""
import zlib

import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
TAU = R.TAU
BF16, F32 = torch.bfloat16, torch.float32
EPIS = {"store_bf16": (R.EPI_STORE_BF16, BF16), "store_f32": (R.EPI_STORE_F32, F32), "gelu_bf16": (R.EPI_GELU_BF16, BF16),
        "resid_f32": (R.EPI_RESID_F32, F32)}


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def ratios():
    """largest fraction of the bound used, per family (printed at the end of the module; run with -s to see it)"""
    seen = {}
    yield seen
    for k in sorted(seen):
        print(f"bound used: {k:<34s} {seen[k]:.3g}")


def note(ratios, family, r):
    ratios[family] = max(ratios.get(family, 0.0), r)


def gen(key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(key.encode()))


def bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def twice(launch):
    """launch() -> {name: (view, buffer)} on fresh buffers; run it twice, the buffers must match bit for bit"""
    r1, r2 = launch(), launch()
    for name in r1:
        assert torch.equal(bits(r1[name][1]), bits(r2[name][1])), f"{name}: two launches differ"
    return r1


def canary(shape, dtype):
    return R.canary_out(shape, ldo_extra=8, rows_before=1, rows_after=3, dtype=dtype)


def nan_full(shape, dtype=BF16):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def same_bits(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    bad = int((bits(got) != bits(want)).sum().item())
    assert bad == 0, f"{what}: {bad} of {got.numel()} elements differ from the definition"


# --------------------------------------------------------------------------------------------------------------------
# grouped sliding window
# --------------------------------------------------------------------------------------------------------------------
def pack_halo(K, x, B, T, G, cg, cpad, taps, rows_alloc):
    """the conv operand as audio.py builds it: fp32 rows [B*(T+1), G*cg] (a CLS row before each clip) packed by
    pack_group_halo into [rows_alloc, G, cpad].  Packing into a NaN-filled buffer first checks the kernel bit for bit:
    rows halo..halo+T-1 of each clip hold bf16(x) and zero padding channels, every other row is untouched.  Returns the
    packing into a zeroed buffer (zero halo), the operand the conv reads."""
    halo, S, Tp = taps // 2, T + 1, T + 2 * (taps // 2)
    want = nan_full((rows_alloc, G, cpad))
    body = want[:B * Tp].view(B, Tp, G, cpad)[:, halo:halo + T]
    body[..., :cg] = x.view(B, S, G, cg)[:, 1:].bfloat16()
    body[..., cg:] = 0
    got = nan_full((rows_alloc, G, cpad))
    K.pack_group_halo(x, got, B, T, S, 1, Tp, halo, G * cg, cg, cpad)
    same_bits(got, want, "pack_group_halo")
    X = torch.zeros(rows_alloc, G, cpad, dtype=BF16, device="cuda")
    K.pack_group_halo(x, X, B, T, S, 1, Tp, halo, G * cg, cg, cpad)
    return X


def conv_weights(G, n, cg, cpad, taps, g, scale=0.03):
    """bf16 [G*n, taps*cpad] with zero padding columns (as the adapter packs Conv1d weights)"""
    w = torch.zeros(G * n, taps, cpad, device="cuda")
    w[:, :, :cg] = torch.randn(G * n, taps, cg, device="cuda", generator=g) * scale
    return w.view(G * n, taps * cpad).bfloat16()


def check_grouped(K, ratios, X, W, bias, rows, G, cpad, taps, n, epi_name, family):
    epi, dt = EPIS[epi_name]

    def launch():
        out, buf = canary((rows, G * n), dt)
        K.grouped_conv1d(X, W, bias, out, rows, G, cpad, taps, n, epi=epi)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    R.assert_canary(buf, out)
    ref = R.grouped_window_ref(X, W, rows, G, cpad, taps, n, epi, bias=bias)
    note(ratios, family, R.assert_within(out, ref.y, ref.mag, TAU, dt, extra=ref.extra))
    return out, ref


PROD = dict(B=2, T=749, G=16, cg=96, cpad=128, taps=19)     # two 15 s clips through Conv1d(1536, 1536, k=19, pad=9, groups=16)


@pytest.fixture(scope="module")
def prod(K):
    """the positional conv's operands at the production geometry: rows = 2 * 767 = 1534 (12 row panels x 16 groups = 192
    work units), K = 19 * 128 = 2432 (38 k-blocks, two per tap)"""
    p = PROD
    g = gen("prod")
    x = torch.randn(p["B"] * (p["T"] + 1), p["G"] * p["cg"], device="cuda", generator=g)
    Tp = p["T"] + 2 * (p["taps"] // 2)
    rows = p["B"] * Tp
    X = pack_halo(K, x, p["B"], p["T"], p["G"], p["cg"], p["cpad"], p["taps"], rows + p["taps"])
    W = conv_weights(p["G"], p["cg"], p["cg"], p["cpad"], p["taps"], g)
    bias = 0.1 * torch.randn(p["G"] * p["cg"], device="cuda", generator=g)
    return dict(p, x=x, X=X, W=W, bias=bias, rows=rows, Tp=Tp)


@pytest.mark.parametrize("use_bias", [True, False])
@pytest.mark.parametrize("epi_name", ["store_bf16", "store_f32", "gelu_bf16"])
def test_grouped_window_production(K, ratios, prod, epi_name, use_bias):
    p = prod
    check_grouped(K, ratios, p["X"], p["W"], p["bias"] if use_bias else None, p["rows"], p["G"], p["cpad"], p["taps"], p["cg"],
                  epi_name, f"grouped window {epi_name}")


# name: (B, T, G, cg, cpad, taps, n_per_group, epilogue)
EDGES = {
    "tiny_model": (2, 45, 16, 16, 64, 19, 16, "store_f32"),         # d = 256: one k-block per tap
    "kb_inner_3": (2, 60, 4, 136, 192, 19, 136, "store_f32"),       # three k-blocks per tap
    "n_256": (2, 60, 3, 96, 128, 19, 256, "store_f32"),             # a whole tile per group: no dropped columns
    "n_8": (2, 60, 5, 96, 128, 19, 8, "store_bf16"),                # 248 of 256 tile columns dropped
    "groups_1": (2, 60, 1, 96, 128, 19, 200, "store_f32"),
    "taps_1": (3, 90, 4, 64, 64, 1, 64, "store_f32"),               # no halo, no tap wrap
    "rows_mod_128_1": (1, 111, 4, 96, 128, 19, 96, "store_f32"),    # rows = 129
    "rows_mod_128_127": (1, 237, 4, 96, 128, 19, 96, "store_bf16"),  # rows = 255
    "resid_f32": (2, 60, 4, 96, 128, 19, 96, "resid_f32"),          # the ABI passes only bias: acc + bias in fp32
}


def run_geometry(K, ratios, case, B, T, G, cg, cpad, taps, n, epi_name):
    """one grouped window case on packed random operands -> (x, W, bias, out, ref)"""
    g = gen(case)
    Tp = T + 2 * (taps // 2)
    rows = B * Tp
    x = torch.randn(B * (T + 1), G * cg, device="cuda", generator=g)
    X = pack_halo(K, x, B, T, G, cg, cpad, taps, rows + taps)
    W = conv_weights(G, n, cg, cpad, taps, g)
    bias = torch.randn(G * n, device="cuda", generator=g)
    out, ref = check_grouped(K, ratios, X, W, bias, rows, G, cpad, taps, n, epi_name, f"grouped window {epi_name}")
    return x, W, bias, out, ref


@pytest.mark.parametrize("case", list(EDGES))
def test_grouped_window_geometry(K, ratios, case):
    run_geometry(K, ratios, case, *EDGES[case])


def grouped_conv1d_torch(x, W, bias, B, T, G, cg, cpad, taps):
    """Conv1d(G*cg, G*cg, taps, padding=taps//2, groups=G) in fp64 on the bf16 operands the kernel reads: [B, T, G*cg]"""
    xs = x.view(B, T + 1, G * cg)[:, 1:].bfloat16().double().transpose(1, 2)
    w = W.view(G * cg, taps, cpad)[:, :, :cg].double().permute(0, 2, 1)
    return torch.nn.functional.conv1d(xs, w, bias.double(), padding=taps // 2, groups=G).transpose(1, 2)


def check_conv1d(K, ratios, B, T, G):
    """the kernel within the bound of the fp64 window reference, and that reference equal to torch's Conv1d in fp64 on
    the valid rows t < T of every clip (c_pad = 64, 24 live channels per group)"""
    cg, cpad, taps = 24, 64, 19
    x, W, bias, out, ref = run_geometry(K, ratios, f"conv1d/{B}/{T}/{G}", B, T, G, cg, cpad, taps, cg, "store_f32")
    want = grouped_conv1d_torch(x, W, bias, B, T, G, cg, cpad, taps)
    Tp = T + 2 * (taps // 2)
    torch.testing.assert_close(ref.y.view(B, Tp, G * cg)[:, :T], want, rtol=1e-12, atol=1e-12)


def test_grouped_conv1d_matches_torch(K, ratios):
    """Conv1d(C, C, k=19, padding=9, groups=G) on channel-last data is the grouped sliding-window GEMM on the halo'd,
    group-padded buffer (models/adapter/audio.py:57-80)"""
    check_conv1d(K, ratios, 2, 45, 4)


def test_grouped_conv1d_more_tiles_than_sms(K, ratios):
    """10 row panels x 16 groups = 160 work units, more than the SMs: CTAs run several units of different groups"""
    check_conv1d(K, ratios, 4, 300, 16)


def test_grouped_window_padding_channels_count(K, ratios):
    """the ABI sums over every c < c_pad: finite values in the padding channels of X and W enter the result"""
    B, T, G, cg, cpad, taps = 2, 60, 4, 96, 128, 19
    g = gen("pad_values")
    rows = B * (T + 2 * (taps // 2))
    x = torch.randn(B * (T + 1), G * cg, device="cuda", generator=g)
    X = pack_halo(K, x, B, T, G, cg, cpad, taps, rows + taps)
    X[:, :, cg:] = torch.randn(rows + taps, G, cpad - cg, device="cuda", generator=g).bfloat16()
    W = (torch.randn(G * cg, taps * cpad, device="cuda", generator=g) * 0.03).bfloat16()
    bias = torch.randn(G * cg, device="cuda", generator=g)
    check_grouped(K, ratios, X, W, bias, rows, G, cpad, taps, cg, "store_f32", "grouped window store_f32")
    ref_live = R.grouped_window_ref(X[:, :, :cg].contiguous(), W.view(G * cg, taps, cpad)[:, :, :cg].reshape(G * cg, -1),
                                    rows, G, cg, taps, cg, R.EPI_STORE_F32, bias=bias)
    full = R.grouped_window_ref(X, W, rows, G, cpad, taps, cg, R.EPI_STORE_F32, bias=bias)
    assert ((full.y - ref_live.y).abs() > TAU * full.mag).any(), "the padding channels do not change the reference"


def test_grouped_window_reads_nothing_past_its_operands(K, ratios):
    """X holds rows + taps - 1 rows and W groups * n_per_group rows, both followed by NaN: the row panels past `rows` and
    the last group's 256-row weight box must zero-fill, not read those rows"""
    B, T, G, cg, cpad, taps = 2, 100, 4, 96, 128, 19
    g = gen("nan_outside")
    rows = B * (T + 2 * (taps // 2))
    x = torch.randn(B * (T + 1), G * cg, device="cuda", generator=g)
    Xz = pack_halo(K, x, B, T, G, cg, cpad, taps, rows + taps - 1)
    Xbuf = nan_full((rows + taps - 1 + 130, G, cpad))
    Xbuf[:rows + taps - 1] = Xz
    Wbuf = nan_full((G * cg + 256, taps * cpad))
    Wbuf[:G * cg] = conv_weights(G, cg, cg, cpad, taps, g)
    bias = torch.randn(G * cg, device="cuda", generator=g)
    for epi_name in ("store_f32", "store_bf16"):
        check_grouped(K, ratios, Xbuf[:rows + taps - 1], Wbuf[:G * cg], bias, rows, G, cpad, taps, cg, epi_name,
                      f"grouped window {epi_name}")


def test_training_lowering_of_the_positional_conv(K, ratios, prod):
    """autograd.AudioPosFn runs the same convolution as window_gather ([G, B*T, 19*96], checked bit for bit against its
    definition) and one plain GEMM per group (K = 1824, a partial last k-block; N = 96 written into a column slice of the
    1536-wide output).  Both lowerings are within the bound of the one fp64 reference; their k-blocks straddle taps
    differently, so they need not agree bit for bit."""
    p = prod
    B, T, G, cg, cpad, taps, Tp = p["B"], p["T"], p["G"], p["cg"], p["cpad"], p["taps"], p["Tp"]
    d = G * cg
    p_in = p["x"].view(B, T + 1, d)[:, 1:].reshape(B * T, d).bfloat16()
    Xw = K.window_gather(p_in, B, T, T, 1, taps, taps // 2, G)
    for g in range(G):
        want = R.window_matrix(p["X"], p["rows"], G, cpad, taps, g).view(B, Tp, taps, cpad)[:, :T, :, :cg]
        same_bits(Xw[g], want.reshape(B * T, taps * cg).bfloat16(), f"window_gather group {g}")
    Wt = p["W"].view(d, taps, cpad)[:, :, :cg].reshape(d, taps * cg).contiguous()
    bias = p["bias"]

    def launch():
        out, buf = canary((B * T, d), BF16)
        for g in range(G):
            sl = slice(g * cg, (g + 1) * cg)
            K.gemm(Xw[g], Wt[sl], K.EPI_STORE_BF16, out[:, sl], bias=bias[sl])
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    R.assert_canary(buf, out)
    ref = R.grouped_window_ref(p["X"], p["W"], p["rows"], G, cpad, taps, cg, R.EPI_STORE_BF16, bias=bias)
    valid = lambda t: t.view(B, Tp, d)[:, :T].reshape(B * T, d)
    note(ratios, "window_gather + gemm store_bf16",
         R.assert_within(out, valid(ref.y), valid(ref.mag), TAU, BF16, extra=valid(ref.extra)))


# --------------------------------------------------------------------------------------------------------------------
# overlapping strided rows
# --------------------------------------------------------------------------------------------------------------------
# name: (C_in, C_out, kw, M, epilogue): a stride-2 Conv1d read as an [M, kw*C] view at a row pitch of 2 C
OVERLAP = {
    "layer1_k3": (512, 512, 3, 24000, "store_bf16"),    # 4B feature extractor layer 1, one 15 s clip (P = 750, pitch 32 P)
    "layer5_k2": (512, 512, 2, 1500, "store_bf16"),     # layer 5: adjacent rows (K = lda), pitch 2 P
}


@pytest.mark.parametrize("case", list(OVERLAP))
def test_overlapping_strided_rows(K, ratios, case):
    run_overlap(K, ratios, case, *OVERLAP[case])


def test_gemm_overlapping_strided_rows_is_conv1d(K, ratios):
    """k=3, s=2 Conv1d over 41 channel-last frames is the GEMM on an overlapping strided view (audio.py:270-284); the fp64
    reference of that view is torch's Conv1d in fp64"""
    C, N, kw, M = 64, 128, 3, 20
    flat, w, ref = run_overlap(K, ratios, "conv1d_k3", C, N, kw, M, "store_f32")
    x = flat[:(2 * M + 1) * C].double().view(2 * M + 1, C)
    want = torch.nn.functional.conv1d(x.t()[None], w.double().view(N, kw, C).permute(0, 2, 1), stride=2)[0].t()
    torch.testing.assert_close(ref.y, want, rtol=1e-12, atol=1e-12)


def run_overlap(K, ratios, case, C, N, kw, M, epi_name):
    """a stride-2 Conv1d as a GEMM whose A is read as rows m*lda ... m*lda + K - 1 of a buffer holding exactly
    (M - 1) * lda + K finite elements, then NaN -> (buffer, weights, reference)"""
    epi, dt = EPIS[epi_name]
    Kd, lda = kw * C, 2 * C
    g = gen(case)
    used = (M - 1) * lda + Kd
    flat = nan_full((used + 4 * C,))
    flat[:used] = torch.randn(used, device="cuda", generator=g).bfloat16()
    a = flat.view(-1, C)
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.04).bfloat16()

    def launch():
        out, buf = canary((M, N), dt)
        K.gemm(a, w, epi, out, M=M, K=Kd, lda=lda)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    R.assert_canary(buf, out)
    ref = R.gemm_ref(flat.as_strided((M, Kd), (lda, 1)), w, epi)
    note(ratios, f"overlapping rows {epi_name}", R.assert_within(out, ref.y, ref.mag, TAU, dt, extra=ref.extra))
    return flat, w, ref


# --------------------------------------------------------------------------------------------------------------------
# narrow K
# --------------------------------------------------------------------------------------------------------------------
def frame10_def(wav, pitch):
    """audio_frame10 by its definition: row (b, t), t < pitch, column j holds wav[b, 5t + j] for j < 10 and 5t + j < n,
    zero elsewhere"""
    B, n = wav.shape
    t = torch.arange(pitch, device=wav.device)[:, None]
    j = torch.arange(16, device=wav.device)[None, :]
    idx = 5 * t + j
    live = (j < 10) & (idx < n)
    v = wav.float()[:, idx.clamp(max=n - 1)]
    return torch.where(live, v, torch.zeros_like(v)).bfloat16().reshape(B * pitch, 16)


@pytest.mark.parametrize("wav_dt", [F32, BF16])
@pytest.mark.parametrize("n_samples,pitch", [(16000, 3210), (16003, 3206)])
def test_audio_frame_conv(K, ratios, wav_dt, n_samples, pitch):
    """a0 = audio_frame10(wav) (n % 5 in {0, 3}, pitch past the last frame) bit for bit, nothing written past B * pitch
    rows; then the K = 16 frame conv gemm(a0, w[512, 16]) against fp64"""
    B = 2
    frames = (n_samples - 10) // 5 + 1
    assert pitch > frames
    g = gen(f"frame/{n_samples}/{wav_dt}")
    wav = torch.randn(B, n_samples, device="cuda", generator=g).to(wav_dt)
    buf = nan_full((B * pitch + 5, 16))
    K.audio_frame10(wav, pitch, buf)
    same_bits(buf[:B * pitch], frame10_def(wav, pitch), "audio_frame10")
    same_bits(buf[B * pitch:], nan_full((5, 16)), "audio_frame10 past B * pitch rows")
    a0 = buf[:B * pitch]
    w = (torch.randn(512, 16, device="cuda", generator=g) * 0.3).bfloat16()

    def launch():
        out, obuf = canary((B * pitch, 512), BF16)
        K.gemm(a0, w, K.EPI_STORE_BF16, out)
        return {"out": (out, obuf)}

    out, obuf = twice(launch)["out"]
    R.assert_canary(obuf, out)
    ref = R.gemm_ref(a0, w, R.EPI_STORE_BF16)
    note(ratios, "narrow K audio frames store_bf16", R.assert_within(out, ref.y, ref.mag, TAU, BF16, extra=ref.extra))


@pytest.mark.parametrize("img_dt", [F32, BF16])
def test_image_stem(K, ratios, img_dt):
    """image_patchify4 at R = 224 bit for bit against the torch permute, then the K = 48 stem GEMM against fp64"""
    B, R_, N = 2, 224, 384
    g = gen(f"stem/{img_dt}")
    img = torch.randn(B, 3, R_, R_, device="cuda", generator=g).to(img_dt)
    a1 = K.image_patchify4(img)
    G_ = R_ // 4
    same_bits(a1, img.float().view(B, 3, G_, 4, G_, 4).permute(0, 2, 4, 1, 3, 5).reshape(B * G_ * G_, 48).bfloat16(),
              "image_patchify4")
    w = (torch.randn(N, 48, device="cuda", generator=g) * 0.2).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)

    def launch():
        out, buf = canary((a1.shape[0], N), BF16)
        K.gemm(a1, w, K.EPI_STORE_BF16, out, bias=bias)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    R.assert_canary(buf, out)
    ref = R.gemm_ref(a1, w, R.EPI_STORE_BF16, bias=bias)
    note(ratios, "narrow K image stem store_bf16", R.assert_within(out, ref.y, ref.mag, TAU, BF16, extra=ref.extra))


def test_narrow_k_zero_fills_past_k(K, ratios):
    """K = 16 read from a 24-wide buffer with NaN in columns 16..23: the k-block is zero-filled past K, not read from the
    neighbouring columns"""
    M, N, Kd = 1000, 512, 16
    g = gen("narrow_slice")
    buf24 = nan_full((M, 24))
    buf24[:, :Kd] = torch.randn(M, Kd, device="cuda", generator=g).bfloat16()
    a = buf24[:, :Kd]
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.3).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)

    def launch():
        out, buf = canary((M, N), F32)
        K.gemm(a, w, K.EPI_STORE_F32, out, bias=bias)
        return {"out": (out, buf)}

    out, buf = twice(launch)["out"]
    R.assert_canary(buf, out)
    ref = R.gemm_ref(a, w, R.EPI_STORE_F32, bias=bias)
    note(ratios, "narrow K column slice store_f32", R.assert_within(out, ref.y, ref.mag, TAU, F32, extra=ref.extra))
