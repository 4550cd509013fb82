"""Drop-in for ``one_peace.metrics.map.MAP`` (metrics/map.py), the evaluation of FSD50K: the mean over classes of
scikit-learn's average precision of the sigmoid probabilities against multi-hot targets.  Same protocol (``initialize()``,
``compute(ids, logits, targets)`` per batch, ``merge_results(output_predict)``) and the same return keys and types: ``map``
(float), ``map_cnt`` (int), ``predict_results`` ({int id: [probability, ...]}).

``compute`` runs opb_sigmoid_pack (csrc/metrics.cu), which writes torch.sigmoid's fp32 probabilities bit for bit and uint8
labels into a buffer that grows by doubling, and counts non-binary targets and NaN probabilities on the device; nothing
synchronises.  ``merge_results`` ranks on the device with opb_average_precision: scikit-learn's definition (ties grouped on
equal probabilities), exact counts, fp64 terms summed in a fixed order.  Where scikit-learn raises (a target outside {0, 1}, a
NaN probability) this raises ``ValueError``; a class without positives gets AP 0 with a ``UserWarning``, as scikit-learn 1.9
does.  scikit-learn is not needed."""
import warnings

import torch

from .. import kernels as K
from .accuracy import _ids, exchange


class MAP:
    def __init__(self):
        self.initialize()

    def initialize(self):
        self.ids_list = []
        self.probs = self.labels = self.flags = None          # [capacity, C]; rows [0, self.rows) are written
        self.rows = 0
        self.device = None

    def _reserve(self, n, C, device):
        if self.probs is None:
            cap = max(n, 256)
            self.probs = torch.empty(cap, C, dtype=torch.float32, device=device)
            self.labels = torch.empty(cap, C, dtype=torch.uint8, device=device)
            self.flags = torch.zeros(2, dtype=torch.int32, device=device)
            return
        if self.probs.shape[1] != C:
            raise ValueError(f"MAP.compute: {C} classes after {self.probs.shape[1]} in earlier batches")
        if self.rows + n > self.probs.shape[0]:
            cap = max(2 * self.probs.shape[0], self.rows + n)
            probs = torch.empty(cap, C, dtype=torch.float32, device=device)
            labels = torch.empty(cap, C, dtype=torch.uint8, device=device)
            probs[:self.rows].copy_(self.probs[:self.rows])
            labels[:self.rows].copy_(self.labels[:self.rows])
            self.probs, self.labels = probs, labels

    def compute(self, ids, logits, targets):
        """map.py:20-23, with the sigmoid of :34 taken here."""
        n, C = logits.shape
        self.device = logits.device
        self._reserve(n, C, logits.device)
        K.sigmoid_pack(logits, targets.to(logits.device), self.probs, self.labels, self.rows, self.flags)
        self.rows += n
        self.ids_list.append(_ids(ids, logits.device))

    def merge_results(self, output_predict=False):
        """map.py:25-48."""
        if self.probs is None:
            raise ValueError("MAP.merge_results: no samples were computed")
        dev = self.device
        probs, labels = self.probs[:self.rows], self.labels[:self.rows]
        ids = torch.cat(self.ids_list)
        counters = self.flags.to(torch.int64)
        counters, ids, probs, labels = exchange(counters, ids, probs, labels)
        bad_targets, nan_probs = counters.tolist()
        if bad_targets:
            raise ValueError(f"MAP: {bad_targets} targets are not 0 or 1; average precision needs multi-hot targets")
        if nan_probs:
            raise ValueError(f"MAP: {nan_probs} probabilities are NaN (NaN logits)")
        ap, mean, npos = K.average_precision(probs.contiguous(), labels.contiguous())
        missing = (npos == 0).nonzero().flatten().tolist()
        if missing:
            warnings.warn(f"No positive class found in y_true for classes {missing}: their average precision is 0.",
                          UserWarning)
        predict_results = {}
        if output_predict:
            for i, pred in zip(ids.cpu().tolist(), probs.cpu().tolist()):
                predict_results[i] = pred
        return {"map": float(mean.item()), "map_cnt": int(probs.shape[0]), "predict_results": predict_results}
