"""Drop-ins for the timm criteria that ``main_ft.py:349-353`` picks: ``SoftTargetCrossEntropy`` (with mixup / cutmix) and
``LabelSmoothingCrossEntropy(smoothing)``.  Both are the batch mean of a per-row cross-entropy, computed with its gradient by
``opb_classify_loss`` through autograd_classify.ClassifyLossFn and scaled by 1 / B.

timm's label-smoothed loss, (1 - s) * nll + s * mean_c(-log p_c), is torch's cross_entropy with label_smoothing = s, which is
the kernel's hard-label mode with eps = s."""
import torch.nn as nn

from .. import kernels as K
from ..autograd_classify import ClassifyLossFn


class SoftTargetCrossEntropy(nn.Module):
    """mean over rows of sum_c -target_c * log_softmax(x)_c; x fp32 [B, C] (any row pitch), target fp32 [B, C]."""

    def forward(self, x, target):
        t = target.float().contiguous()
        if t.shape != x.shape:
            raise ValueError(f"SoftTargetCrossEntropy: target {tuple(t.shape)} does not match the logits {tuple(x.shape)}")
        loss, _, _ = ClassifyLossFn.apply(x, K.LOSS_SOFT, None, t, 0.0, 1)
        return loss * (1.0 / x.shape[0])


class LabelSmoothingCrossEntropy(nn.Module):
    """mean over rows of (1 - smoothing) * nll + smoothing * mean_c(-log_softmax(x)_c); target int64 [B]."""

    def __init__(self, smoothing=0.1):
        super().__init__()
        if not 0.0 <= smoothing < 1.0:
            raise ValueError(f"LabelSmoothingCrossEntropy: smoothing must be in [0, 1), got {smoothing}")
        self.smoothing = smoothing
        self.confidence = 1.0 - smoothing

    def forward(self, x, target):
        labels = target.long().contiguous()
        if labels.shape != (x.shape[0],):
            raise ValueError(f"LabelSmoothingCrossEntropy: target {tuple(labels.shape)} must be [B] class ids")
        loss, _, _ = ClassifyLossFn.apply(x, K.LOSS_HARD, labels, None, self.smoothing, 1)
        return loss * (1.0 / x.shape[0])
