"""Drop-in for ``hinge_loss`` (criterions/hinge_loss.py, the AQA recipe): every audio clip is repeated num_choices times next
to its candidate answers, the logits [B * num_choices, 1] are read as [B, num_choices], and
loss = sum max(0, 1 + logits - positive) — the positive's own term contributes its constant 1.  The reference hard-codes that
1: the configured `margin` is kept as a field and not used, exactly as there."""
from dataclasses import dataclass

from .. import kernels as K
from ..autograd_classify import ClassifyLossFn
from ..fairseq_compat import FairseqCriterion, FairseqDataclass, register_criterion
from .classify_loss import _reduce_metrics


@dataclass
class HingeLossConfig(FairseqDataclass):
    margin: float = 1.0
    num_choices: int = 4


@register_criterion("hinge_loss", dataclass=HingeLossConfig)
class HingeLoss(FairseqCriterion):
    def __init__(self, task, margin=1.0, num_choices=4):
        super().__init__(task)
        self.margin = margin
        self.num_choices = num_choices

    def forward(self, model, sample, reduce=True):
        """hinge_loss.py:33-63."""
        ni = sample["net_input"]
        src_audios = ni["src_audios"].repeat_interleave(self.num_choices, 0)
        audio_padding_masks = ni["audio_padding_masks"].repeat_interleave(self.num_choices, 0)
        logits = model(src_tokens=ni["src_tokens"], src_audios=src_audios, audio_padding_masks=audio_padding_masks)
        loss, n_correct, _ = ClassifyLossFn.apply(logits, K.LOSS_HINGE, sample["target"].long().contiguous(), None, 0.0,
                                                  self.num_choices)
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
