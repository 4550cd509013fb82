"""Drop-in for ``one_peace.metrics.accuracy.Accuracy`` (metrics/accuracy.py), the evaluation of VQA, NLVR2, VGGSound, AQA and
``image_classify``: the share of rows whose argmax hits the target.  Same protocol (``initialize()``, ``compute(ids, logits,
targets)`` per batch, ``merge_results(output_predict)``) and the same return keys and types: ``accuracy``, ``score_sum``
(float), ``score_cnt`` (int), ``predict_results`` ({int id: int hyp}).

Targets are hard labels [n] (``argmax == target`` counts 1) or soft scores [n, C] (the row scores ``targets[r, argmax]``, VQA).
The argmax and the row score come from opb_argmax_hits (csrc/metrics.cu) with torch.argmax's rules (first maximal index,
NaN is the maximum), reading fp32 or bf16 logits in place, padded rows and column-strided views included.  ``compute`` only
enqueues kernels and keeps the per-batch tensors; ``merge_results`` concatenates them once and sums the row scores in fp64 in a
fixed order (opb_sum_f64), so a hard-label ``score_sum`` is the exact count and a soft one the same bits on every run."""
import torch
import torch.distributed as dist

from .. import kernels as K
from .recall import _all_gather_cat


def exchange(counters, *tensors):
    """The distributed step of ``merge_results``: ``counters`` (int64 [k]) summed over the ranks, each tensor gathered in rank
    order with the uneven-shard gather (utils/data_utils.py:50-85), so that every rank evaluates the same whole set.  Without
    an initialised process group the inputs come back as they are."""
    if not dist.is_initialized():
        return (counters,) + tensors
    dist.all_reduce(counters, op=dist.ReduceOp.SUM)
    return (counters,) + tuple(_all_gather_cat(t) for t in tensors)


def _ids(ids, device):
    """ids as the reference keeps them: concatenated onto an int64 tensor (so float ids promote as torch.cat would)."""
    return ids.to(device=device, dtype=torch.promote_types(torch.int64, ids.dtype))


class Accuracy:
    def __init__(self):
        self.initialize()

    def initialize(self):
        self.ids_list, self.hyps_list, self.scores_list = [], [], []
        self.score_cnt = 0
        self.device = None

    def compute(self, ids, logits, targets):
        """accuracy.py:20-30."""
        self.device = logits.device
        hyp, score = K.argmax_hits(logits, targets.to(logits.device))
        self.score_cnt += logits.size(0)
        self.ids_list.append(_ids(ids, logits.device))
        self.hyps_list.append(hyp)
        self.scores_list.append(score)

    def merge_results(self, output_predict=False):
        """accuracy.py:32-55."""
        dev = self.device if self.device is not None else torch.device("cuda")
        ids = torch.cat(self.ids_list) if self.ids_list else torch.empty(0, dtype=torch.int64, device=dev)
        hyps = torch.cat(self.hyps_list) if self.hyps_list else torch.empty(0, dtype=torch.int64, device=dev)
        scores = torch.cat(self.scores_list) if self.scores_list else torch.empty(0, dtype=torch.float32, device=dev)
        counters = torch.tensor([self.score_cnt], dtype=torch.int64, device=dev)
        counters, ids, hyps, scores = exchange(counters, ids, hyps, scores)
        score_cnt = int(counters.item())
        score_sum = float(K.sum_f64(scores).item()) if scores.numel() else 0.0
        predict_results = {}
        if output_predict:
            for i, hyp in zip(ids.cpu().tolist(), hyps.cpu().tolist()):
                predict_results[i] = hyp
        return {"accuracy": score_sum / score_cnt, "score_sum": score_sum, "score_cnt": score_cnt,
                "predict_results": predict_results}
