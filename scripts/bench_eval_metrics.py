"""Times the classification evaluation metrics over a whole evaluation stream: every ``compute`` call, then ``merge_results``,
for three recipe shapes, against an eager restatement of the reference (torch.cat onto growing tensors, argmax / gather,
torch.sigmoid and scikit-learn's average_precision_score on the host when scikit-learn is importable).

* FSD50K ``MAP``: 10,231 clips x 200 classes in batches of 8, fp32 logits.
* VGGSound ``Accuracy``: 15,446 clips x 309 classes in batches of 32, hard labels.
* VQA ``Accuracy``: 40,000 questions x 3,129 answers in batches of 64, soft scores; bf16 logits as the classification model
  returns them (the [:, :3129] view of rows padded to 3,136 columns).

Every stream lives on the device before timing starts; each figure is the median of --repeat runs after one warm-up run.
Prints one JSON line and writes it to --out if given.

    python scripts/bench_eval_metrics.py [--repeat 3] [--out result.json]
"""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_classify_step import card  # noqa: E402


class EagerAccuracy:
    """metrics/accuracy.py restated in eager torch (the baseline)."""

    def initialize(self):
        dev = torch.device("cuda")
        self.score_sum = torch.zeros(1, device=dev)
        self.score_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ids = torch.zeros(0, dtype=torch.int64, device=dev)
        self.hyps = torch.zeros(0, dtype=torch.int64, device=dev)

    def compute(self, ids, logits, targets):
        predict_labels = logits.argmax(1)
        if targets.dim() == 2:
            n_correct = targets.gather(1, predict_labels.unsqueeze(1)).sum()
        else:
            n_correct = predict_labels.eq(targets).sum()
        self.score_sum += n_correct
        self.score_cnt += logits.size(0)
        self.ids = torch.cat([self.ids, ids], dim=0)
        self.hyps = torch.cat([self.hyps, predict_labels], dim=0)

    def merge_results(self):
        return self.score_sum.item() / self.score_cnt.item()


class EagerMAP:
    """metrics/map.py restated: torch.cat growth on the device, sigmoid, then scikit-learn on the host."""

    def initialize(self):
        dev = torch.device("cuda")
        self.logits = torch.zeros(0, device=dev)
        self.targets = torch.zeros(0, device=dev)
        self.ids = torch.zeros(0, dtype=torch.int64, device=dev)

    def compute(self, ids, logits, targets):
        self.ids = torch.cat([self.ids, ids], dim=0)
        self.logits = torch.cat([self.logits, logits], dim=0)
        self.targets = torch.cat([self.targets, targets], dim=0)

    def merge_results(self):
        import numpy as np
        from sklearn.metrics import average_precision_score
        preds = torch.sigmoid(self.logits).cpu().numpy()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return float(np.mean(average_precision_score(self.targets.cpu().numpy(), preds, average=None)))


def stream(kind):
    g = torch.Generator(device="cuda").manual_seed(0)
    if kind == "fsd50k_map":
        N, C, bs = 10231, 200, 8
        logits = torch.randn(N, C, device="cuda", generator=g) * 2 - 3
        targets = (torch.rand(N, C, device="cuda", generator=g) < torch.sigmoid(logits + 1)).float()
    elif kind == "vggsound_accuracy":
        N, C, bs = 15446, 309, 32
        logits = torch.randn(N, C, device="cuda", generator=g)
        targets = torch.randint(0, C, (N,), device="cuda", generator=g)
    else:
        N, C, bs = 40000, 3129, 64
        padded = torch.randn(N, 3136, device="cuda", generator=g).to(torch.bfloat16)
        logits = padded[:, :C]
        targets = torch.zeros(N, C, device="cuda")
        cols = torch.randint(0, C, (N, 3), device="cuda", generator=g)
        targets.scatter_(1, cols, torch.rand(N, 3, device="cuda", generator=g).round(decimals=1))
    ids = torch.arange(N, device="cuda")
    batches = [(ids[lo:lo + bs], logits[lo:lo + bs], targets[lo:lo + bs]) for lo in range(0, N, bs)]
    return dict(N=N, C=C, batch=bs, batches=batches)


def run(metric, batches):
    """-> (compute ms over the stream, merge ms, result)."""
    metric.initialize()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in batches:
        metric.compute(*b)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = metric.merge_results()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    if isinstance(out, dict):
        out = out.get("map", out.get("accuracy"))
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3, out


def median_run(metric, batches, repeat):
    run(metric, batches)
    rs = [run(metric, batches) for _ in range(repeat)]
    return round(statistics.median(r[0] for r in rs), 2), round(statistics.median(r[1] for r in rs), 2), rs[-1][2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from one_peace_b200.metrics import MAP, Accuracy
    try:
        import sklearn  # noqa: F401
        have_sklearn = True
    except ImportError:
        have_sklearn = False
    res = dict(metric="eval_metrics", card=card(), sklearn=have_sklearn)
    for kind in ("fsd50k_map", "vggsound_accuracy", "vqa_accuracy"):
        s = stream(kind)
        ours_cls, eager_cls = (MAP, EagerMAP) if kind.endswith("map") else (Accuracy, EagerAccuracy)
        c, m, v = median_run(ours_cls(), s["batches"], args.repeat)
        rec = dict(N=s["N"], C=s["C"], batch=s["batch"], compute_ms=c, merge_ms=m, value=v)
        if kind.endswith("map") and not have_sklearn:
            rec.update(eager_compute_ms=None, eager_merge_ms=None, eager_value=None)
        else:
            ec, em, ev = median_run(eager_cls(), s["batches"], args.repeat)
            rec.update(eager_compute_ms=ec, eager_merge_ms=em, eager_value=ev)
        res[kind] = rec
        del s
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
