"""Drop-in for ``image_text_retrieval_criterion`` (criterions/image_text_retrieval_loss.py:49-152).

Same constructor (task, label_smoothing), same ``forward(model, sample, reduce)`` return triple and logging
keys, same ``compute_itc_loss`` signature.  The arithmetic of compute_itc_loss (two (b x Wb x d) similarity
GEMMs, fp32 log-softmax, label-smoothed NLL, arg-max accuracy, and the local-rows-only gradient) runs in the
wgmma GEMM epilogues + merge kernels of csrc/infonce.cu; the b x Wb logits are never written to HBM in fp32.
The cross-rank exchange is one NCCL all_gather_into_tensor per modality into a rank-major (W*b, d) bf16 buffer
(= the reference's all_gather + cat order, :30-38), forward only, no autograd.
"""
import torch
import torch.distributed as dist

from .. import kernels as K
from ..fairseq_compat import FairseqCriterion, metrics, register_criterion


def gather_without_grad(tensor):
    """criterions/image_text_retrieval_loss.py:29-38: rank-major concatenation of every rank's rows, detached."""
    with torch.no_grad():
        t = tensor.detach().contiguous()
        out = torch.empty(dist.get_world_size() * t.shape[0], *t.shape[1:], dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, t)
    return out


class _InfoNCE(torch.autograd.Function):
    """loss, a2b_ncorrect, b2a_ncorrect = f(a_local, b_local, a_all, b_all, scale).  a = image/audio, b = text.
    Gradients: to a_local via sim(a_local, b_all), to b_local via sim(b_local, a_all), to scale via both;
    *_all are constants (SURVEY.md A.9).  Forward and the gradient factors are computed together (fused
    forward+backward, like a fused cross-entropy) when any input requires grad."""

    @staticmethod
    def forward(ctx, a_local, b_local, a_all, b_all, scale, rank, eps):
        f32 = lambda t: t.detach().to(torch.float32).contiguous()
        d = a_local.shape[1]
        # bf16x3 operand split: logits accurate to ~2^-16 on the bf16 tensor cores (csrc/infonce.cu); the four splits are one launch
        n_cls = a_all.shape[0]
        fa, fb = f32(a_all), f32(b_all)
        if n_cls % 8:                 # the GEMM wants N % 8 == 0: zero rows, ignored through n_valid (tiny global batches)
            padr = torch.zeros((-n_cls) % 8, d, dtype=torch.float32, device=fa.device)
            fa, fb = torch.cat([fa, padr]), torch.cat([fb, padr])
        a3, b3, a_all3, b_all3 = K.split_bf16x3([f32(a_local), f32(b_local), fa, fb], [0, 0, 1, 1])
        s = scale.detach().to(torch.float32).reshape(1).contiguous()
        bsz, n = a3.shape[0], a_all3.shape[0]
        nv = n_cls if n_cls != n else 0
        off = bsz * rank
        # two LSE GEMMs + ONE merge / reduce kernel for both directions (the last block to finish does the fixed-order reduction)
        (lse_a, lse_b), out = K.infonce_forward([(a3, b_all3), (b3, a_all3)], s, off, eps, n_valid=nv)
        if a_local.requires_grad or b_local.requires_grad or scale.requires_grad:
            ga, ws_a = K.infonce_grad(a3, b_all3, s, lse_a, off, eps, d, n_valid=nv)      # G . B_all reads B_all MN-major
            gb, ws_b = K.infonce_grad(b3, a_all3, s, lse_b, off, eps, d, n_valid=nv)
            dlogit = K.infonce_dscale(ws_a, ws_b, bsz, n)        # d loss / d log(scale)
            ctx.save_for_backward(ga, gb, dlogit, s)
        ctx.dtypes = (a_local.dtype, b_local.dtype, scale.dtype)
        ctx.mark_non_differentiable(out[1], out[2])
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_loss, _g1, _g2):
        ga, gb, dlogit, s = ctx.saved_tensors
        da, db, ds = ctx.dtypes
        g = g_loss.to(torch.float32)
        return (ga * g).to(da), (gb * g).to(db), None, None, (dlogit / s * g).reshape(()).to(ds), None, None


def itc_loss(a_local, b_local, a_all, b_all, logit_scale_exp, rank=0, label_smoothing=0.0):
    return _InfoNCE.apply(a_local, b_local, a_all, b_all, logit_scale_exp, rank, float(label_smoothing))


@register_criterion("image_text_retrieval_criterion")
class ImageTextRetrievalCriterion(FairseqCriterion):
    src_key, logits_key = "src_images", "image"
    a2b, b2a = "i2t_ncorrect", "t2i_ncorrect"

    def __init__(self, task, label_smoothing=0.0):
        super().__init__(task)
        self.label_smoothing = label_smoothing

    def forward(self, model, sample, reduce=True):
        """(loss, sample_size=1, logging_output) — image_text_retrieval_loss.py:55-89."""
        ni = sample["net_input"]
        text_logits = model(src_tokens=ni["src_tokens"], encoder_type="text")
        other_logits = self.encode_other(model, ni)
        text_all = gather_without_grad(text_logits) if dist.is_initialized() else text_logits.data
        other_all = gather_without_grad(other_logits) if dist.is_initialized() else other_logits.data
        logit_scale_exp = model(return_logit_scale=True)
        loss, a_ok, b_ok = self.compute_itc_loss(other_logits, text_logits, other_all, text_all, logit_scale_exp)
        logging_output = {"loss": loss.data, "nsentences": sample["nsentences"], "sample_size": 1,
                          self.a2b: a_ok, self.b2a: b_ok, "logit_scale_exp": logit_scale_exp.data}
        return loss, 1, logging_output

    def encode_other(self, model, ni):
        return model(src_images=ni["src_images"], encoder_type="image")

    def compute_itc_loss(self, image_logits, text_logits, image_logits_all, text_logits_all, logit_scale_exp):
        rank = dist.get_rank() if dist.is_initialized() else 0
        return itc_loss(image_logits, text_logits, image_logits_all, text_logits_all, logit_scale_exp, rank,
                        self.label_smoothing)

    @classmethod
    def reduce_metrics(cls, logging_outputs) -> None:
        """image_text_retrieval_loss.py:114-143."""
        loss_sum = sum(log.get("loss", 0) for log in logging_outputs)
        scale_sum = sum(log.get("logit_scale_exp", 0) for log in logging_outputs)
        nsentences = sum(log.get("nsentences", 1) for log in logging_outputs)
        sample_size = sum(log.get("sample_size", 1) for log in logging_outputs)
        metrics.log_scalar("loss", loss_sum / sample_size, sample_size, round=3)
        metrics.log_scalar("logit_scale_exp", scale_sum / sample_size, sample_size, round=3)
        metrics.log_scalar("nsentences", nsentences, 1, round=3)
        metrics.log_scalar("sample_size", sample_size, 1, round=3)
        for key, name in ((cls.a2b, cls.a2b.replace("ncorrect", "accuracy")), (cls.b2a, cls.b2a.replace("ncorrect", "accuracy"))):
            if len(logging_outputs) > 0 and key in logging_outputs[0]:
                ncorrect = sum(log.get(key, 0) for log in logging_outputs)
                metrics.log_scalar(name, 100.0 * ncorrect / nsentences, nsentences, round=1)

    @staticmethod
    def logging_outputs_can_be_summed() -> bool:
        return True
