"""Drop-in for ``classify_criterion`` (criterions/classify_loss.py) and ``hinge_loss`` (criterions/hinge_loss.py): same config
fields, ``forward(model, sample, reduce)`` return triple, logging keys and ``reduce_metrics``.  The loss, its gradient and
n_correct of every form (hard labels with label smoothing, soft targets, multi-label BCE, hinge over answer choices) come from
one launch of opb_classify_loss (csrc/classify.cu) with a fixed-order reduction; sample_size = nsentences."""
from dataclasses import dataclass

import torch

from .. import kernels as K
from ..autograd_classify import ClassifyLossFn
from ..fairseq_compat import FairseqCriterion, FairseqDataclass, metrics, register_criterion


@dataclass
class ClassifyCriterionConfig(FairseqDataclass):
    use_multi_label: bool = False
    label_smoothing: float = 0.0


def _reduce_metrics(logging_outputs):
    """classify_loss.py:76-103 (hinge_loss.py:65-92 is identical)."""
    loss_sum = sum(log.get("loss", 0) for log in logging_outputs)
    nsentences = sum(log.get("nsentences", 0) for log in logging_outputs)
    sample_size = sum(log.get("sample_size", 0) for log in logging_outputs)
    metrics.log_scalar("loss", loss_sum / sample_size, sample_size, round=3)
    metrics.log_scalar("nsentences", nsentences, 1, round=3)
    metrics.log_scalar("sample_size", sample_size, 1, round=3)
    total = float(sample_size)
    if total > 0:
        metrics.log_scalar("total", total)
        n_correct = float(sum(log.get("n_correct", 0) for log in logging_outputs))
        metrics.log_scalar("n_correct", n_correct)
        metrics.log_derived("accuracy", lambda meters: round(meters["n_correct"].sum * 100.0 / meters["total"].sum, 3)
                            if meters["total"].sum > 0 else float("nan"))


@register_criterion("classify_criterion", dataclass=ClassifyCriterionConfig)
class ClassifyCriterion(FairseqCriterion):
    def __init__(self, task, use_multi_label=False, label_smoothing=0.0):
        super().__init__(task)
        self.use_multi_label = use_multi_label
        self.label_smoothing = label_smoothing

    def forward(self, model, sample, reduce=True):
        """classify_loss.py:40-74."""
        logits = model(**sample["net_input"])
        targets = sample["target"]
        if self.use_multi_label:
            mode, labels, soft = K.LOSS_MULTI_LABEL, None, targets.to(torch.float32)
        elif targets.dim() == 2:
            mode, labels, soft = K.LOSS_SOFT, None, targets.to(torch.float32)
        else:
            mode, labels, soft = K.LOSS_HARD, targets.to(torch.int64).contiguous(), None
        loss, n_correct, _ = ClassifyLossFn.apply(logits, mode, labels, soft, float(self.label_smoothing), 1)
        sample_size = sample["nsentences"]
        logging_output = {"loss": loss.data, "nsentences": sample["nsentences"], "sample_size": sample_size,
                          "n_correct": n_correct}
        return loss, sample_size, logging_output

    @staticmethod
    def reduce_metrics(logging_outputs) -> None:
        _reduce_metrics(logging_outputs)

    @staticmethod
    def logging_outputs_can_be_summed() -> bool:
        return True
