"""Drop-in for ``refcoco_criterion`` (criterions/refcoco_loss.py), the visual-grounding criterion: same (empty) config,
``forward(model, sample, reduce)`` return triple, logging keys, ``reduce_metrics`` and ``logging_outputs_can_be_summed``.

The loss is refcoco_loss.py:36-46: with p = sigmoid(logits) the predicted box (x0, y0, x1, y1),

    loss = sum |p - target| / nsentences + mean over the valid rows of (1 - GIoU(p, target)),

a row being valid when p0 < p2 and p1 < p3.  The value and its gradient come from one launch of opb_refcoco_loss
(csrc/grounding.cu) with a fixed-order reduction.  As in the reference, a batch without a valid row (a fresh or diverging head
can produce one) has a NaN loss, the mean of an empty tensor, while its gradient is finite: the L1 part only.  fairseq's
trainer checks the gradient norm, not the loss, so such a step is taken and the NaN only shows in the logged loss.
sample_size is 1: the L1 part is already divided by nsentences and the GIoU part is a mean."""
from dataclasses import dataclass

from ..autograd_classify import RefcocoLossFn
from ..fairseq_compat import FairseqCriterion, FairseqDataclass, metrics, register_criterion


@dataclass
class RefCOCOCriterionConfig(FairseqDataclass):
    pass


@register_criterion("refcoco_criterion", dataclass=RefCOCOCriterionConfig)
class RefCOCOCriterion(FairseqCriterion):
    def __init__(self, task):
        super().__init__(task)

    def forward(self, model, sample, reduce=True):
        """refcoco_loss.py:27-55."""
        logits = model(**sample["net_input"])
        loss, _, _ = RefcocoLossFn.apply(logits, sample["target"], sample["nsentences"])
        sample_size = 1
        logging_output = {"loss": loss.data, "nsentences": sample["nsentences"], "sample_size": sample_size}
        return loss, sample_size, logging_output

    @staticmethod
    def reduce_metrics(logging_outputs) -> None:
        """refcoco_loss.py:56-72."""
        loss_sum = sum(log.get("loss", 0) for log in logging_outputs)
        nsentences = sum(log.get("nsentences", 0) for log in logging_outputs)
        sample_size = sum(log.get("sample_size", 0) for log in logging_outputs)
        metrics.log_scalar("loss", loss_sum / sample_size, sample_size, round=3)
        metrics.log_scalar("nsentences", nsentences, 1, round=3)
        metrics.log_scalar("sample_size", sample_size, 1, round=3)

    @staticmethod
    def logging_outputs_can_be_summed() -> bool:
        return True
