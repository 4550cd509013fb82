"""CPU: the fp64 restatement of the classification metrics (tests/metrics_ref.py) against the reference's own Accuracy and MAP
(tests/golden/metrics.pt, made by oracle/make_golden_metrics.py) and against scikit-learn when it is importable; seven planted
mistakes, each of which must exceed a bound at least 100-fold or change an exact count; the distributed exchange of
merge_results over gloo with uneven shards; and the metric names."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import metrics_ref as M
import synth_metrics as sm


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "metrics.pt"), weights_only=False)


@pytest.mark.parametrize("name", list(sm.ACC_CASES))
def test_accuracy_restatement_matches_reference(name, golden_dir):
    rec = _gold(golden_dir)["accuracy"][name]
    ids, logits, targets, cuts = sm.accuracy_case(name)
    hyp = M.argmax_ref(logits.float().numpy())
    assert np.array_equal(hyp, rec["hyps"].numpy())
    merged = rec["merged"]
    assert merged["score_cnt"] == logits.shape[0]
    assert merged["predict_results"] == dict(zip(ids.tolist(), hyp.tolist()))
    if targets.dim() == 2:
        scores = targets.numpy()[np.arange(len(hyp)), hyp].astype(np.float64)
        exact = M.soft_sum_exact(scores)
        assert abs(merged["score_sum"] - exact) <= M.soft_sum_bound_fp32(scores, rec["batches"])
        assert exact != merged["score_sum"]                       # the reference's fp32 accumulator did round
    else:
        assert M.hard_hits(hyp, targets.numpy()).sum() == merged["score_sum"]


@pytest.mark.parametrize("name", list(sm.MAP_CASES))
def test_ap_restatement_matches_reference(name, golden_dir):
    rec = _gold(golden_dir)["map"][name]
    ids, logits, targets, cuts = sm.map_case(name)
    assert torch.equal(rec["predict_ids"], ids)
    probs = M.sigmoid_f32(logits.float().numpy())
    # the fixture keeps the reference's probabilities of every 8th row: the restated route gives them to a few ulp
    kept = probs[rec["predict_rows"].numpy()].view(np.int32).astype(np.int64)
    assert np.abs(kept - rec["predict_probs"].numpy().view(np.int32).astype(np.int64)).max() <= 4
    ap, G, P = M.average_precision_ref(probs, targets.numpy())
    want = rec["ap"].numpy()
    assert (np.abs(ap - want) <= 2 * M.ap_bound(G)).all(), np.max(np.abs(ap - want) / M.ap_bound(G))
    assert abs(M.map_ref(ap, P) - rec["merged"]["map"]) <= 2 * M.map_bound(G)
    assert rec["merged"]["map_cnt"] == logits.shape[0]
    assert (P == 0).sum() == 1 and any("No positive class" in w for w in rec["warnings"])
    # the kinds of column the case was built to hold
    C = logits.shape[1]
    first = C - len(sm.MAP_SPECIAL)
    kinds = ["general"] * first + list(sm.MAP_SPECIAL)
    eq = kinds.index("all_equal")
    assert G[eq] == 1 and ap[eq] == P[eq] / logits.shape[0]
    sat = [c for c, k in enumerate(kinds) if k == "saturated"]
    assert all((probs[:, c] == 1.0).sum() > 100 for c in sat)
    if logits.dtype == torch.bfloat16:
        assert all(G[c] < logits.shape[0] for c in range(first))  # ties in every general column


def _sk():
    return pytest.importorskip("sklearn.metrics")


@pytest.mark.parametrize("N,C,tied", [(7, 2, False), (500, 13, True), (2000, 40, True), (3000, 5, False)])
def test_ap_restatement_matches_sklearn(N, C, tied):
    skm = _sk()
    g = torch.Generator().manual_seed(N + C)
    z = torch.randn(N, C, generator=g)
    if tied:
        z = z.to(torch.bfloat16).float()
    p = torch.sigmoid(z).numpy()
    y = (torch.rand(N, C, generator=g) < 0.3).numpy().astype(np.int64)
    y[0, :] = 1
    ap, G, P = M.average_precision_ref(p, y)
    want = skm.average_precision_score(y, p, average=None)
    assert (np.abs(ap - want) <= 2 * M.ap_bound(G)).all()
    assert abs(M.map_ref(ap, P) - float(np.mean(want))) <= 2 * M.map_bound(G)


def test_ap_no_positive_class_is_zero_as_sklearn():
    skm = _sk()
    p = np.array([[0.2, 0.3], [0.5, 0.5], [0.9, 0.1]], dtype=np.float32)
    y = np.array([[1, 0], [0, 0], [1, 0]])
    ap, G, P = M.average_precision_ref(p, y)
    with pytest.warns(UserWarning, match="No positive class"):
        want = skm.average_precision_score(y, p, average=None)
    assert ap[1] == want[1] == 0.0 and P[1] == 0
    assert abs(ap[0] - want[0]) <= 2 * M.ap_bound(G)[0]


def test_sum_bounds_hold_for_fp32_and_any_order():
    g = torch.Generator().manual_seed(3)
    s = torch.where(torch.rand(50000, generator=g) < 0.1, torch.rand(50000, generator=g), torch.zeros(50000)).numpy()
    exact = M.soft_sum_exact(s)
    assert abs(float(np.sum(s.astype(np.float64)[::-1])) - exact) <= M.soft_sum_bound(s)
    acc = np.float32(0)
    for chunk in np.array_split(s, 37):                          # the reference: per-batch fp32 sums into an fp32 counter
        acc = np.float32(acc + np.float32(chunk.sum(dtype=np.float32)))
    assert abs(float(acc) - exact) <= M.soft_sum_bound_fp32(s, 37)


# ------------------------------------------------------------------------------------------------------------------
# planted mistakes
# ------------------------------------------------------------------------------------------------------------------
def _fsd():
    _, logits, targets, _ = sm.map_case("fsd50k_bf16")
    return logits, targets.numpy(), M.sigmoid_f32(logits.float().numpy())


@pytest.mark.parametrize("mistake", ["position", "precision_first", "recall_over_N"])
def test_planted_ap_mistakes_exceed_the_bound(mistake):
    _, y, p = _fsd()
    ap, G, P = M.average_precision_ref(p, y)
    bad, _, _ = M.average_precision_ref(p, y, mistake)
    assert np.max(np.abs(bad - ap) / M.ap_bound(G)) > 100.0


def test_planted_mistake_drop_no_positive_from_mean():
    _, y, p = _fsd()
    ap, G, P = M.average_precision_ref(p, y)
    assert abs(M.map_ref(ap, P, "drop_no_positive") - M.map_ref(ap, P)) > 100.0 * M.map_bound(G)


def test_planted_mistake_fp64_sigmoid_splits_the_saturated_group():
    logits, y, p32 = _fsd()
    x = logits.float().numpy()
    ap, G, P = M.average_precision_ref(p32, y)
    bad, G64, _ = M.average_precision_ref(M.sigmoid_f64(x), y)
    assert (G64 > G).any()
    assert np.max(np.abs(bad - ap) / M.ap_bound(G)) > 100.0


@pytest.mark.parametrize("mistake", ["last_index", "nan_ignored"])
def test_planted_argmax_mistakes_flip_counts(mistake, golden_dir):
    gold = _gold(golden_dir)["accuracy"]
    flipped_hyp = flipped_count = 0
    for name in sm.ACC_CASES:
        ids, logits, targets, cuts = sm.accuracy_case(name)
        bad = M.argmax_ref(logits.float().numpy(), mistake)
        flipped_hyp += int((bad != gold[name]["hyps"].numpy()).sum())
        if targets.dim() == 1:
            flipped_count += M.hard_hits(bad, targets.numpy()).sum() != gold[name]["merged"]["score_sum"]
    assert flipped_hyp > 0 and flipped_count > 0


# ------------------------------------------------------------------------------------------------------------------
# the exchange of merge_results over gloo
# ------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


SHARDS = (5, 3)


def _shard(rank):
    lo = sum(SHARDS[:rank])
    n = SHARDS[rank]
    ids = torch.arange(lo, lo + n, dtype=torch.int64) + 100
    probs = torch.arange(lo * 4, (lo + n) * 4, dtype=torch.float32).reshape(n, 4) / 64
    labels = (torch.arange(lo * 4, (lo + n) * 4).reshape(n, 4) % 3 == 0).to(torch.uint8)
    return ids, probs, labels


def _exchange_worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from one_peace_b200.metrics.accuracy import exchange
    ids, probs, labels = _shard(rank)
    counters = torch.tensor([SHARDS[rank], 10 * rank + 1], dtype=torch.int64)
    out = exchange(counters, ids, probs, labels)
    torch.save([t.clone() for t in out], os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_exchange_gathers_uneven_shards_rank_major_gloo(tmp_path):
    world = len(SHARDS)
    mp.spawn(_exchange_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    parts = [_shard(r) for r in range(world)]
    want = [torch.cat([p[i] for p in parts]) for i in range(3)]
    for r in range(world):
        counters, ids, probs, labels = torch.load(tmp_path / f"r{r}.pt", weights_only=False)
        assert counters.tolist() == [sum(SHARDS), 12]
        assert torch.equal(ids, want[0]) and torch.equal(probs, want[1]) and torch.equal(labels, want[2])


def test_exchange_without_process_group_returns_inputs():
    from one_peace_b200.metrics.accuracy import exchange
    c, a = torch.tensor([1]), torch.arange(3)
    out = exchange(c, a)
    assert out[0] is c and out[1] is a


def test_metric_names_and_protocol():
    from one_peace_b200.metrics import MAP, Accuracy
    for cls in (Accuracy, MAP):
        for name in ("initialize", "compute", "merge_results"):
            assert callable(getattr(cls, name))
