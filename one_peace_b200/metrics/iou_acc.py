"""Drop-in for ``one_peace.metrics.iou_acc.IouAcc`` (metrics/iou_acc.py), the visual-grounding accuracy: the share of predicted
boxes whose IoU with the reference box is at least 0.5.  Same protocol (``initialize()``, ``compute(ids, hyps, refs)`` per
batch, ``merge_results(output_predict)``) and the same return keys and types: ``iou_acc``, ``score_sum`` (float),
``score_cnt`` (int), ``predict_results`` ({float id: box}; ids are float32 as in the reference, which concatenates them onto
an empty float tensor).

The hit test runs in opb_iou_acc (csrc/grounding.cu) in the reference's fp32 operation order, so the count is the reference's
exactly, and accumulates on the device: ``compute`` never synchronises, only ``merge_results`` does."""
import torch
import torch.distributed as dist

from .. import kernels as K
from .recall import _all_gather_cat


class IouAcc:
    def __init__(self):
        self.initialize()

    def initialize(self):
        self.ids_list, self.hyps_list = [], []
        self.hits = None
        self.score_cnt = 0

    def compute(self, ids, hyps, refs):
        """iou_acc.py:20-35: count the hits of this batch and keep its ids and boxes."""
        if self.hits is None:
            self.hits = torch.zeros(1, dtype=torch.int32, device=hyps.device)
        h = hyps.to(torch.float32)
        K.iou_acc(h if h.stride(-1) == 1 else h.contiguous(), refs.to(device=hyps.device, dtype=torch.float32).contiguous(),
                  self.hits)
        self.score_cnt += hyps.size(0)
        self.ids_list.append(ids.to(device=hyps.device, dtype=torch.float32))
        self.hyps_list.append(h)

    def merge_results(self, output_predict=False):
        """iou_acc.py:37-60."""
        dev = self.hits.device if self.hits is not None else torch.device("cuda")
        hits = self.hits if self.hits is not None else torch.zeros(1, dtype=torch.int32, device=dev)
        ids = torch.cat(self.ids_list, 0) if self.ids_list else torch.empty(0, dtype=torch.float32, device=dev)
        hyps = torch.cat(self.hyps_list, 0) if self.hyps_list else torch.empty(0, 4, dtype=torch.float32, device=dev)
        counters = torch.cat([hits.to(torch.int64), torch.tensor([self.score_cnt], dtype=torch.int64, device=dev)])
        if dist.is_initialized():
            dist.all_reduce(counters, op=dist.ReduceOp.SUM)
            ids, hyps = _all_gather_cat(ids), _all_gather_cat(hyps)
        score_sum, score_cnt = counters.tolist()
        score_sum = float(score_sum)
        predict_results = {}
        if output_predict:
            for i, hyp in zip(ids.cpu().tolist(), hyps.cpu().tolist()):
                predict_results[i] = hyp
        return {"iou_acc": score_sum / score_cnt, "score_sum": score_sum, "score_cnt": score_cnt,
                "predict_results": predict_results}
