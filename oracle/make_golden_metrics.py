"""TEST INFRASTRUCTURE.  Generates tests/golden/metrics.pt by executing the reference's OWN metrics/accuracy.py and metrics/map.py
(via oracle/ref_stub.py) on the seeded evaluation streams of oracle/synth_metrics.py.  It needs the reference source tree and
scikit-learn (map.py ranks with sklearn.metrics.average_precision_score):

    python oracle/make_golden_metrics.py

Two stand-ins are installed, and recorded in the fixture:
  * one_peace.utils.data_utils (imported for its distributed all_gather, which a single process never calls) becomes an empty
    module, and both metrics run on the CPU with initialize()'s tensors created there;
  * map.py's torch.sigmoid becomes the same fp32 formula evaluated elementwise (SIGMOID_STANDIN).  The reference runs it on
    the GPU; torch's CPU sigmoid is not even a function of its input (its vectorised body and its scalar tail differ by up to
    4 ulp, so equal logits can land in different tie groups).  The stand-in differs from torch's CUDA result by a few ulp
    at most, and synth_metrics.map_case keeps every logit out of the band where that could change a tie group, so the
    per-class AP and the map are the ones the reference computes on its device.
Besides each merged result the fixture keeps scikit-learn's per-class AP of the reference's own probabilities and targets,
the warnings map.py raised and the scikit-learn version.  Of MAP's predict_results it keeps every id, in order, and the
probabilities of every PREDICT_STRIDE-th row.  The inputs are not stored: the tests regenerate them from synth_metrics.py.
The fixture is committed; the tests read only the fixture.
"""
import os
import sys
import types
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402
import synth_metrics as sm  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
# predict_results keeps every id in order but the probabilities of every PREDICT_STRIDE-th row only, which keeps the fixture
# small; the per-class AP and the map cover every row, and the tests recompute the full probabilities
PREDICT_STRIDE = 8
SIGMOID_STANDIN = "fp32(1 / (1 + fp32(exp(-x)))) with exp in fp64 and the add and the division in fp32, for torch.sigmoid"


def _sigmoid_standin(x):
    import numpy as np
    x = x.detach().to(torch.float32).numpy()
    with np.errstate(over="ignore"):
        e = np.exp(-x.astype(np.float64)).astype(np.float32)
        return torch.from_numpy((np.float32(1.0) / (np.float32(1.0) + e)).astype(np.float32))


class _TorchWithSigmoidStandin(types.ModuleType):
    """torch as map.py sees it: every name is torch's except sigmoid."""

    sigmoid = staticmethod(_sigmoid_standin)

    def __getattr__(self, name):
        return getattr(torch, name)


def _install():
    ref_stub.install()
    if "one_peace.utils" not in sys.modules:
        u = types.ModuleType("one_peace.utils")
        u.__path__ = []
        sys.modules["one_peace.utils"] = u
        sys.modules["one_peace.utils.data_utils"] = types.ModuleType("one_peace.utils.data_utils")
        sys.modules["one_peace.utils.data_utils"].all_gather = None
    if "one_peace.metrics" not in sys.modules:
        m = types.ModuleType("one_peace.metrics")
        m.__path__ = [os.path.join(ref_stub.REF_PKG, "metrics")]
        sys.modules["one_peace.metrics"] = m


def accuracy_cases():
    mod = ref_stub.ref_module("one_peace.metrics.accuracy")
    out = {}
    for name in sm.ACC_CASES:
        ids, logits, targets, cuts = sm.accuracy_case(name)
        a = mod.Accuracy()
        a.score_sum, a.score_cnt = torch.FloatTensor([0]), torch.IntTensor([0])
        a.ids, a.hyps = torch.LongTensor([]), torch.LongTensor([])
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            a.compute(ids[lo:hi], logits[lo:hi], targets[lo:hi])
        merged = a.merge_results(output_predict=True)
        out[name] = {"merged": merged, "hyps": a.hyps.clone(), "batches": len(cuts) - 1}
        print(name, merged["score_sum"], merged["score_cnt"], merged["accuracy"])
    return out


def map_cases():
    mod = ref_stub.ref_module("one_peace.metrics.map")
    mod.torch = _TorchWithSigmoidStandin("torch")
    from sklearn.metrics import average_precision_score
    out = {}
    for name in sm.MAP_CASES:
        ids, logits, targets, cuts = sm.map_case(name)
        a = mod.MAP()
        a.logits, a.targets, a.ids = torch.FloatTensor([]), torch.FloatTensor([]), torch.LongTensor([])
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            a.compute(ids[lo:hi], logits[lo:hi], targets[lo:hi])
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            merged = a.merge_results(output_predict=True)
            ap = average_precision_score(a.targets.numpy(), _sigmoid_standin(a.logits).numpy(), average=None)
        pr = merged.pop("predict_results")
        keys = list(pr)
        out[name] = {"merged": merged, "ap": torch.from_numpy(ap).clone(),
                     "predict_ids": torch.tensor(keys, dtype=torch.int64),
                     "predict_rows": torch.arange(0, len(keys), PREDICT_STRIDE),
                     "predict_probs": torch.tensor([pr[k] for k in keys[::PREDICT_STRIDE]], dtype=torch.float32),
                     "warnings": sorted({f"{w.category.__name__}: {w.message}" for w in caught})}
        print(name, merged["map"], merged["map_cnt"], out[name]["warnings"])
    return out


def metrics():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    _install()
    import sklearn
    out = {"sklearn_version": sklearn.__version__, "sigmoid_standin": SIGMOID_STANDIN, "accuracy": accuracy_cases(),
           "map": map_cases()}
    path = os.path.join(OUT, "metrics.pt")
    torch.save(out, path)
    print("metrics.pt", os.path.getsize(path))


if __name__ == "__main__":
    metrics()
