"""GPU: the classification-evaluation kernels (csrc/metrics.cu) and the Accuracy / MAP metrics.

* opb_argmax_hits equals torch.argmax exactly: fp32 and bf16, contiguous rows, rows padded to a pitch of 8, a column stride
  of 8, planted ties, NaNs, -inf and signed zeros, C = 1 to 4096, n = 1 to 100,000; hard and soft row scores exactly.
* opb_sigmoid_pack equals torch.sigmoid bit for bit over a dense sweep of fp32 bit patterns, the saturated ranges, +-inf and
  every bf16 value; labels and the flag word exactly.
* opb_average_precision within the bounds of tests/metrics_ref.py for N = 1 to 131,072 and C = 2, 200, 527 with sparse,
  dense, no-positive, all-tied and bf16-tied classes; positive counts exact.
* all four kernels write nothing outside their outputs, repeat bit for bit and refuse bad arguments.
* Accuracy and MAP against the reference's (tests/golden/metrics.pt): counts and hypotheses exactly, soft sums and map
  within bound, predict_results probabilities bit for bit equal to torch.sigmoid on the device.
* the tiny one_peace_classify model's logits (strided bf16 views) through Accuracy against a torch argmax count."""
import os
import warnings

import numpy as np
import pytest
import torch

import metrics_ref as M
import synth_metrics as sm

pytestmark = pytest.mark.gpu


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "metrics.pt"), weights_only=False)


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous().view(torch.int64)


def _logits(n, C, seed, dtype):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, C, generator=g, device="cuda") * 3.0
    tie = torch.rand(n, generator=g, device="cuda") < 0.4
    x[tie] = torch.round(x[tie])                                       # many equal maxima
    nan = torch.rand(n, C, generator=g, device="cuda") < (2.0 / max(C, 2))
    x[nan & (torch.rand(n, 1, generator=g, device="cuda") < 0.2)] = float("nan")
    if n > 3:
        x[1] = float("-inf")
        x[2] = 0.0
        x[2, C // 2] = -0.0
        x[3] = float("nan")
    return x.to(dtype)


def _layout(x, layout):
    """'contig'; 'pitch8': rows padded to a multiple of 8 columns, the [:, :C] view; 'col8': column stride 8."""
    n, C = x.shape
    if layout == "contig":
        return x
    if layout == "pitch8":
        buf = torch.full((n, (C + 7) // 8 * 8), 777.0, dtype=x.dtype, device=x.device)
        buf[:, :C] = x
        return buf[:, :C]
    buf = torch.full((n, 8 * C), 777.0, dtype=x.dtype, device=x.device)
    buf[:, ::8] = x
    return buf[:, ::8]


@pytest.mark.parametrize("layout", ["contig", "pitch8", "col8"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C", [1, 2, 4, 7, 8, 9, 33, 309, 3129, 4096])
def test_argmax_hits_equals_torch_argmax(C, dtype, layout):
    need_gpu()
    from one_peace_b200 import kernels as K
    for n in (1, 1000):
        x = _layout(_logits(n, C, 11 * C + n, dtype), layout)
        t = torch.randint(0, C, (n,), device="cuda")
        hyp, score = K.argmax_hits(x, t)
        want = x.argmax(1)
        assert torch.equal(hyp, want), (n, C, dtype, layout)
        assert torch.equal(score, (want == t).float())


@pytest.mark.parametrize("C", [2, 4, 309, 4096])
def test_argmax_hits_100k_rows(C):
    need_gpu()
    from one_peace_b200 import kernels as K
    n = 100_000
    x = _logits(n, C, C, torch.bfloat16 if C == 4096 else torch.float32)
    hyp, _ = K.argmax_hits(x, torch.zeros(n, dtype=torch.int64, device="cuda"))
    assert torch.equal(hyp, x.argmax(1))


def test_argmax_hits_target_modes():
    """int64 labels, fp32 labels (torch.eq's promotion) and soft scores [n, ldt > C] read at the argmax."""
    need_gpu()
    from one_peace_b200 import kernels as K
    n, C = 777, 3129
    x = _logits(n, C, 5, torch.float32)
    want = x.argmax(1)
    g = torch.Generator(device="cuda").manual_seed(6)
    lab = torch.where(torch.rand(n, generator=g, device="cuda") < 0.5, want, torch.randint(0, C, (n,), device="cuda", generator=g))
    _, s_int = K.argmax_hits(x, lab)
    _, s_f32 = K.argmax_hits(x, lab.float())
    assert torch.equal(s_int, (want == lab).float()) and torch.equal(s_f32, want.eq(lab.float()).float())
    soft = torch.zeros(n, C + 5, device="cuda")
    soft[:, :C] = torch.rand(n, C, generator=g, device="cuda").round(decimals=1)
    hyp, s_soft = K.argmax_hits(x, soft[:, :C])
    assert torch.equal(s_soft, soft[:, :C].gather(1, want.unsqueeze(1)).squeeze(1))


def test_sigmoid_pack_is_torch_sigmoid_bitwise():
    need_gpu()
    from one_peace_b200 import kernels as K
    bits = torch.arange(0, 2 ** 32, 61, dtype=torch.int64, device="cuda").to(torch.int32).view(torch.float32)
    sat = torch.cat([torch.linspace(-120.0, -15.0, 2_000_001), torch.linspace(15.0, 120.0, 2_000_001)]).cuda()
    x = torch.cat([bits, sat, torch.tensor([float("inf"), float("-inf"), 0.0, -0.0], device="cuda")])
    C = 1024
    x = x[:x.numel() // C * C].view(-1, C)
    n = x.shape[0]
    t = torch.zeros(n, C, device="cuda")
    probs = torch.empty(n, C, device="cuda")
    labels = torch.empty(n, C, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(2, dtype=torch.int32, device="cuda")
    K.sigmoid_pack(x, t, probs, labels, 0, flags)
    want = torch.sigmoid(x)
    same = (_bits(probs) == _bits(want)) | (torch.isnan(probs) & torch.isnan(want))
    assert bool(same.all()), int((~same).sum())
    assert int(flags[0]) == 0 and int(flags[1]) == int(torch.isnan(x).sum())
    assert (probs[torch.isfinite(x) & (x > 16.7)] == 1.0).all()
    # every bf16 value, up-cast first
    xb = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(torch.bfloat16).view(-1, 256)
    pb = torch.empty(xb.shape, device="cuda")
    lb = torch.empty(xb.shape, dtype=torch.uint8, device="cuda")
    K.sigmoid_pack(xb, torch.ones(xb.shape, device="cuda"), pb, lb, 0, flags.zero_())
    wb = torch.sigmoid(xb.float())
    assert bool(((_bits(pb) == _bits(wb)) | (torch.isnan(pb) & torch.isnan(wb))).all())
    assert (lb == 1).all()


def test_sigmoid_pack_strided_offset_labels_and_flags():
    need_gpu()
    from one_peace_b200 import kernels as K
    n, C, off = 37, 200, 5
    x = _layout(torch.randn(n, C, device="cuda") * 5, "col8")
    t = torch.randint(0, 2, (n, C), device="cuda").float()
    t[0, :6] = torch.tensor([0.5, float("nan"), 2.0, -0.0, -1.0, 1.0])
    probs = torch.full((off + n + 3, C), -7.0, device="cuda")
    labels = torch.full((off + n + 3, C), 9, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(2, dtype=torch.int32, device="cuda")
    K.sigmoid_pack(x, t, probs, labels, off, flags)
    assert torch.equal(_bits(probs[off:off + n]), _bits(torch.sigmoid(x)))
    assert torch.equal(labels[off:off + n], (t == 1).to(torch.uint8))
    assert (probs[:off] == -7).all() and (probs[off + n:] == -7).all() and (labels[:off] == 9).all() and (labels[off + n:] == 9).all()
    assert flags.tolist() == [4, 0]


def _ap_case(N, C, seed):
    """probs fp32 [N, C] and labels uint8 with column kinds cycling through sparse, dense, no-positive, all-tied, bf16-tied and
    continuous."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(N, C, generator=g)
    y = torch.rand(N, C, generator=g)
    labels = torch.zeros(N, C, dtype=torch.uint8)
    for c in range(C):
        kind = c % 6
        if kind == 0:                                                # sparse
            labels[torch.randint(0, N, (min(3, N),), generator=g), c] = 1
        elif kind == 1:                                              # dense
            labels[:, c] = (y[:, c] < 0.9).to(torch.uint8)
        elif kind == 2:                                              # no positive
            pass
        elif kind == 3:                                              # all tied
            z[:, c] = 0.5
            labels[:, c] = (y[:, c] < 0.3).to(torch.uint8)
        elif kind == 4:                                              # bf16 ties, labels correlated with the score
            z[:, c] = z[:, c].to(torch.bfloat16).float()
            labels[:, c] = (y[:, c] < torch.sigmoid(2 * z[:, c])).to(torch.uint8)
        else:
            labels[:, c] = (y[:, c] < torch.sigmoid(z[:, c])).to(torch.uint8)
    return torch.sigmoid(z), labels


AP_SHAPES = [(N, C) for N in (1, 7, 2000, 10231, 65536, 131072) for C in (2, 200)] + [(7, 527), (2000, 527), (10231, 527),
                                                                                     (131072, 527)]


@pytest.mark.parametrize("N,C", AP_SHAPES)
def test_average_precision_within_bounds(N, C):
    need_gpu()
    from one_peace_b200 import kernels as K
    probs, labels = _ap_case(N, C, N + C)
    ap, mean, npos = K.average_precision(probs.cuda(), labels.cuda())
    want, G, P = M.average_precision_ref(probs.numpy(), labels.numpy())
    assert np.array_equal(npos.cpu().numpy(), P)
    err = np.abs(ap.cpu().numpy() - want)
    assert (err <= M.ap_bound(G)).all(), float(np.max(err / M.ap_bound(G)))
    assert abs(float(mean) - M.map_ref(want, P)) <= M.map_bound(G)
    assert (ap.cpu().numpy()[P == 0] == 0).all()


def test_kernels_write_only_their_outputs_and_repeat_bitwise():
    need_gpu()
    from one_peace_b200 import _lib
    lib = _lib.load()
    s = torch.cuda.current_stream().cuda_stream
    n, C, guard = 300, 200, 64
    x = torch.randn(n, C, device="cuda")
    x[::7, 3] = float("nan")
    lab = torch.randint(0, C, (n,), device="cuda")
    t = torch.randint(0, 2, (n, C), device="cuda").float()
    x0, lab0, t0 = x.clone(), lab.clone(), t.clone()
    probs, labels = _ap_case(2000, C, 3)
    probs, labels = probs.cuda(), labels.cuda()
    runs = []
    for _ in range(3):
        hyp = torch.full((n + guard,), -5, dtype=torch.int64, device="cuda")
        score = torch.full((n + guard,), -5.0, device="cuda")
        ssum = torch.full((1 + guard,), -5.0, dtype=torch.float64, device="cuda")
        pk = torch.full(((n + 2) * C + guard,), -5.0, device="cuda")
        lk = torch.full(((n + 2) * C + guard,), 7, dtype=torch.uint8, device="cuda")
        flags = torch.zeros(2 + guard, dtype=torch.int32, device="cuda")
        ws_bytes = lib.opb_average_precision_ws_bytes(2000, C)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        ap = torch.full((C + guard,), -5.0, dtype=torch.float64, device="cuda")
        mean = torch.full((1 + guard,), -5.0, dtype=torch.float64, device="cuda")
        npos = torch.full((C + guard,), -5, dtype=torch.int64, device="cuda")
        assert lib.opb_argmax_hits(x.data_ptr(), 0, C, 1, n, C, lab.data_ptr(), 0, 0, hyp.data_ptr(), score.data_ptr(), s) == 0
        assert lib.opb_sum_f64(score.data_ptr(), n, ssum.data_ptr(), s) == 0
        assert lib.opb_sigmoid_pack(x.data_ptr(), 0, C, 1, t.data_ptr(), C, n, C, pk.data_ptr(), lk.data_ptr(), 2, flags.data_ptr(),
                                    s) == 0
        assert lib.opb_average_precision(probs.data_ptr(), labels.data_ptr(), 2000, C, ws.data_ptr(), ws_bytes, ap.data_ptr(),
                                         mean.data_ptr(), npos.data_ptr(), s) == 0
        torch.cuda.synchronize()
        assert (hyp[n:] == -5).all() and (score[n:] == -5).all() and (ssum[1:] == -5).all()
        assert (pk[:2 * C] == -5).all() and (pk[(n + 2) * C:] == -5).all() and (lk[:2 * C] == 7).all() and (lk[(n + 2) * C:] == 7).all()
        assert (flags[2:] == 0).all() and (ap[C:] == -5).all() and (mean[1:] == -5).all() and (npos[C:] == -5).all()
        runs.append([hyp[:n].clone(), score[:n].clone(), ssum[:1].clone(), pk.clone(), lk.clone(), flags[:2].clone(),
                     ap[:C].clone(), mean[:1].clone(), npos[:C].clone()])
    assert torch.equal(x.view(torch.int32), x0.view(torch.int32)) and torch.equal(lab, lab0) and torch.equal(t, t0)
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def test_kernels_refuse_bad_arguments():
    need_gpu()
    from one_peace_b200 import _lib
    lib = _lib.load()
    s = torch.cuda.current_stream().cuda_stream
    x = torch.zeros(64, 64, device="cuda")
    h = torch.full((64,), -3, dtype=torch.int64, device="cuda")
    f = torch.full((64,), -3.0, device="cuda")
    d = torch.full((64,), -3.0, dtype=torch.float64, device="cuda")
    u = torch.full((4096,), 9, dtype=torch.uint8, device="cuda")
    fl = torch.zeros(2, dtype=torch.int32, device="cuda")
    p, hp, fp, dp, up, flp = x.data_ptr(), h.data_ptr(), f.data_ptr(), d.data_ptr(), u.data_ptr(), fl.data_ptr()
    bad_argmax = [(p, 0, 8, 1, 0, 8, hp, 0, 0), (p, 0, 8, 1, 4, 0, hp, 0, 0), (p, 0, 8, 1, 4, 4097, hp, 0, 0),
                  (p, 0, 0, 1, 4, 8, hp, 0, 0), (p, 0, 8, 0, 4, 8, hp, 0, 0), (p, 2, 8, 1, 4, 8, hp, 0, 0),
                  (p, 0, 8, 1, 4, 8, hp, 3, 0), (p, 0, 8, 1, 4, 8, p, 2, 4), (None, 0, 8, 1, 4, 8, hp, 0, 0),
                  (p, 0, 8, 1, 4, 8, None, 0, 0)]
    for a in bad_argmax:
        assert lib.opb_argmax_hits(*a, hp, fp, s) == 1, a
    assert lib.opb_argmax_hits(p, 0, 8, 1, 4, 8, hp, 0, 0, None, fp, s) == 1
    assert lib.opb_sum_f64(fp, 0, dp, s) == 1 and lib.opb_sum_f64(None, 4, dp, s) == 1 and lib.opb_sum_f64(fp, 4, None, s) == 1
    bad_pack = [(p, 0, 8, 1, p, 8, 0, 8, 0), (p, 0, 8, 1, p, 8, 4, 4097, 0), (p, 0, 8, 1, p, 4, 4, 8, 0),
                (p, 0, 8, 1, p, 8, 4, 8, -1), (p, 5, 8, 1, p, 8, 4, 8, 0), (p, 0, 0, 1, p, 8, 4, 8, 0)]
    for a in bad_pack:
        assert lib.opb_sigmoid_pack(*a[:8], fp, up, a[8], flp, s) == 1, a
    assert lib.opb_sigmoid_pack(p, 0, 8, 1, p, 8, 4, 8, fp, up, 0, None, s) == 1
    assert lib.opb_average_precision_ws_bytes(0, 2) == -1 and lib.opb_average_precision_ws_bytes(1 << 24, 2) == -1
    assert lib.opb_average_precision_ws_bytes(4, 4097) == -1 and lib.opb_average_precision_ws_bytes(1 << 20, 4096) == -1
    need = lib.opb_average_precision_ws_bytes(16, 4)
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    assert lib.opb_average_precision(p, up, 16, 4, ws.data_ptr(), need - 1, dp, dp, hp, s) == 1
    assert lib.opb_average_precision(p, up, 0, 4, ws.data_ptr(), need, dp, dp, hp, s) == 1
    assert lib.opb_average_precision(p, up, 16, 4, None, need, dp, dp, hp, s) == 1
    assert lib.opb_average_precision(p, None, 16, 4, ws.data_ptr(), need, dp, dp, hp, s) == 1
    torch.cuda.synchronize()
    assert (h == -3).all() and (f == -3).all() and (d == -3).all() and (u == 9).all() and (fl == 0).all()


# ------------------------------------------------------------------------------------------------------------------
# the metrics against the reference's
# ------------------------------------------------------------------------------------------------------------------
def _to_cuda_view(t):
    """A CPU view moved to the device with the same strides (the AQA [4B, 1] -> [B, 4] view stays a strided view)."""
    if t.is_contiguous():
        return t.cuda()
    base = t._base.cuda()
    return torch.as_strided(base, t.size(), t.stride(), t.storage_offset())


@pytest.mark.parametrize("name", list(sm.ACC_CASES))
def test_accuracy_metric_matches_reference(name, golden_dir):
    need_gpu()
    from one_peace_b200.metrics import Accuracy
    rec = _gold(golden_dir)["accuracy"][name]
    ids, logits, targets, cuts = sm.accuracy_case(name)
    lc = _to_cuda_view(logits)
    assert lc.stride() == logits.stride()
    m = Accuracy()
    m.initialize()
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        m.compute(ids[lo:hi].cuda(), lc[lo:hi], targets[lo:hi].cuda())
    got = m.merge_results(output_predict=True)
    want = rec["merged"]
    assert got["score_cnt"] == want["score_cnt"] and isinstance(got["score_cnt"], int)
    assert isinstance(got["score_sum"], float)
    assert list(got["predict_results"]) == list(want["predict_results"])
    assert got["predict_results"] == want["predict_results"]
    assert all(isinstance(k, int) and isinstance(v, int) for k, v in got["predict_results"].items())
    if targets.dim() == 2:
        hyp = rec["hyps"].numpy()
        scores = targets.numpy()[np.arange(len(hyp)), hyp]
        exact = M.soft_sum_exact(scores)
        assert abs(got["score_sum"] - exact) <= M.soft_sum_bound(scores)
        assert abs(got["score_sum"] - want["score_sum"]) <= M.soft_sum_bound_fp32(scores, rec["batches"])
        assert m.merge_results()["score_sum"] == got["score_sum"]                 # the same bits again
    else:
        assert got["score_sum"] == want["score_sum"] and got["accuracy"] == want["accuracy"]
    assert got["accuracy"] == got["score_sum"] / got["score_cnt"]


@pytest.mark.parametrize("name", list(sm.MAP_CASES))
def test_map_metric_matches_reference(name, golden_dir):
    need_gpu()
    from one_peace_b200 import kernels as K
    from one_peace_b200.metrics import MAP
    rec = _gold(golden_dir)["map"][name]
    ids, logits, targets, cuts = sm.map_case(name)
    m = MAP()
    m.initialize()
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        m.compute(ids[lo:hi].cuda(), logits[lo:hi].cuda(), targets[lo:hi].cuda())
    with pytest.warns(UserWarning, match="No positive class"):
        got = m.merge_results(output_predict=True)
    assert got["map_cnt"] == rec["merged"]["map_cnt"] and isinstance(got["map_cnt"], int)
    assert list(got["predict_results"]) == rec["predict_ids"].tolist()
    probs = torch.tensor(list(got["predict_results"].values()), dtype=torch.float32)
    # map.py:34 on the reference's device: torch.sigmoid of the fp32 concatenation
    assert torch.equal(_bits(probs), _bits(torch.sigmoid(logits.cuda().float()).cpu()))
    # the fixture's stand-in sigmoid (kept for every 8th row, restated in full by metrics_ref.sigmoid_f32): a few ulp at
    # most, the same tie groups
    ulp = (_bits(probs[rec["predict_rows"]]).long() - _bits(rec["predict_probs"]).long()).abs()
    assert int(ulp.max()) <= 4
    _, G, P = M.average_precision_ref(probs.numpy(), targets.numpy())
    _, G_fix, _ = M.average_precision_ref(M.sigmoid_f32(logits.float().numpy()), targets.numpy())
    assert np.array_equal(G, G_fix)
    ap, _, npos = K.average_precision(probs.cuda(), (targets == 1).to(torch.uint8).cuda())
    assert np.array_equal(npos.cpu().numpy(), P)
    assert (np.abs(ap.cpu().numpy() - rec["ap"].numpy()) <= 2 * M.ap_bound(G)).all()
    assert abs(got["map"] - rec["merged"]["map"]) <= 2 * M.map_bound(G)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert m.merge_results()["map"] == got["map"]                              # the same bits again


def test_map_raises_where_sklearn_raises():
    need_gpu()
    from one_peace_b200.metrics import MAP
    x = torch.randn(16, 4, device="cuda")
    t = torch.randint(0, 2, (16, 4), device="cuda").float()
    t[:, 0] = 1.0
    m = MAP()
    m.compute(torch.arange(16, device="cuda"), x, torch.where(t == 1, 0.7, t))
    with pytest.raises(ValueError, match="not 0 or 1"):
        m.merge_results()
    m = MAP()
    x[3, 2] = float("nan")
    m.compute(torch.arange(16, device="cuda"), x, t)
    with pytest.raises(ValueError, match="NaN"):
        m.merge_results()


def test_classify_model_logits_through_accuracy():
    """one_peace_classify's logits are a [:, :n_cls] view of rows padded to 8 columns (bf16 model): the metric reads them in
    place; AQA's hinge layout reshapes [4B, 1] into [B, 4] with a column stride of 8."""
    need_gpu()
    import synth_classify as sc
    from test_gpu_classify import build, _cuda
    from one_peace_b200.metrics import Accuracy
    case, sd, sample = sc.classify_case("audio_hard")
    _, m = build(case, sd, dtype="bfloat16")
    s = _cuda(sample)
    with torch.no_grad():
        logits = m(**s["net_input"])
    assert logits.dtype == torch.bfloat16
    n = logits.shape[0]
    labels = torch.arange(n, device="cuda") % logits.shape[1]
    labels[0] = logits.float().argmax(1)[0]
    acc = Accuracy()
    acc.compute(torch.arange(n, device="cuda"), logits, labels)
    got = acc.merge_results(output_predict=True)
    assert got["score_sum"] == float((logits.argmax(1) == labels).sum()) and got["score_cnt"] == n
    assert list(got["predict_results"].values()) == logits.argmax(1).tolist()
    case, sd, sample = sc.classify_case("al_hinge")
    _, m = build(case, sd, dtype="bfloat16")
    ni = _cuda(sample)["net_input"]
    ni = dict(src_tokens=ni["src_tokens"], src_audios=ni["src_audios"].repeat_interleave(4, 0),
              audio_padding_masks=ni["audio_padding_masks"].repeat_interleave(4, 0))
    with torch.no_grad():
        lg = m(**ni)
    view = lg.view(-1, 4)
    assert lg.shape[1] == 1
    acc = Accuracy()
    t = torch.zeros(view.shape[0], dtype=torch.int64, device="cuda")
    acc.compute(torch.arange(view.shape[0], device="cuda"), view, t)
    got = acc.merge_results(output_predict=True)
    assert list(got["predict_results"].values()) == view.argmax(1).tolist()
    assert got["score_sum"] == float((view.argmax(1) == 0).sum())
