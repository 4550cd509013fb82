"""Drop-in for ``one_peace.metrics.recall.Recall`` (metrics/recall.py:8-78): image<->text Recall@{1,5,10} of the
retrieval evaluation.  Same protocol (``initialize(text_ids, text_logits)``, ``compute(image_ids, image_logits)`` per
batch, ``merge_results()`` -> the same ``eval_log`` keys).

The (N_img x N_txt) similarity matrix is one wgmma GEMM per direction on bf16x3-split operands (K = 3d: logits to
~2^-16 relative, the same device the InfoNCE head uses, so the ranking equals the fp32 ranking except at exact ties);
top-10 per row and the hit counters are sm_90a kernels (csrc/recall.cu).  Nothing is ranked on the CPU.
"""
import torch
import torch.distributed as dist

from .. import kernels as K


def _all_gather_cat(t):
    """utils/data_utils.py:50-85: rank-major concatenation of shards that may differ in length (the last evaluation batch
    is uneven when the set is not divisible by the world size): exchange the sizes, pad to the longest, gather, trim."""
    world = dist.get_world_size()
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    sizes = torch.empty(world, dtype=torch.int64, device=t.device)
    dist.all_gather_into_tensor(sizes, n)
    sizes = sizes.tolist()
    longest = max(sizes)
    if t.shape[0] != longest:
        padded = torch.zeros(longest, *t.shape[1:], dtype=t.dtype, device=t.device)
        padded[:t.shape[0]].copy_(t)
        t = padded
    out = torch.empty(world * longest, *t.shape[1:], dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous())
    if all(sz == longest for sz in sizes):
        return out
    return torch.cat([out[r * longest:r * longest + sz] for r, sz in enumerate(sizes)], dim=0)


class Recall:
    def __init__(self):
        self.text_ids = self.text_logits = None
        self.image_ids_list, self.image_logits_list = [], []

    def initialize(self, text_ids, text_logits):
        self.text_ids = text_ids
        self.text_logits = text_logits
        self.image_ids_list = []
        self.image_logits_list = []

    def compute(self, image_ids, image_logits):
        self.image_ids_list.append(image_ids)
        self.image_logits_list.append(image_logits)

    def merge_results(self, output_predict=False):
        image_ids = torch.cat(self.image_ids_list, dim=0)
        image_logits = torch.cat(self.image_logits_list, dim=0)
        if dist.is_initialized():
            image_ids, image_logits = _all_gather_cat(image_ids), _all_gather_cat(image_logits)
        self.image_ids, self.image_logits = image_ids, image_logits
        return self.retrieval_eval(output_predict)

    @staticmethod
    def _similarity(a, b):
        """fp32 [Na, Nb] = a b^T through the wgmma GEMM on bf16x3-split operands."""
        a3, b3 = K.split_bf16x3([a.detach().float().contiguous(), b.detach().float().contiguous()], [0, 1])
        nb = b.shape[0]
        nb8 = (nb + 7) // 8 * 8                       # the GEMM wants N % 8 == 0: zero rows, never ranked (C = nb below)
        if nb8 != nb:
            pad = torch.zeros(nb8, b3.shape[1], dtype=b3.dtype, device=b3.device)
            pad[:nb].copy_(b3)
            b3 = pad
        out = torch.empty(a.shape[0], nb8, dtype=torch.float32, device=a.device)
        return K.gemm(a3, b3, K.EPI_STORE_F32, out)[:, :nb]

    def retrieval_eval(self, output_predict=False):
        img_ids, txt_ids = self.image_ids.to(torch.int64).contiguous(), self.text_ids.to(torch.int64).contiguous()
        n_img, n_txt = self.image_logits.shape[0], self.text_logits.shape[0]
        if min(n_img, n_txt) < 10:                     # the reference's topk(k=10) raises here too (recall.py:39,50)
            raise RuntimeError(f"Recall@10 needs at least 10 candidates in each direction; got {n_txt} texts and "
                               f"{n_img} images")
        rank_txt = K.topk10_rows(self._similarity(self.image_logits, self.text_logits))      # image -> text
        rank_img = K.topk10_rows(self._similarity(self.text_logits, self.image_logits))      # text -> image
        i2t = K.recall_hits(rank_txt, txt_ids, img_ids).tolist()
        t2i = K.recall_hits(rank_img, img_ids, txt_ids).tolist()
        tr = [100.0 * c / n_img for c in i2t]
        ir = [100.0 * c / n_txt for c in t2i]
        tr_mean, ir_mean = sum(tr) / 3, sum(ir) / 3
        predict_txt, predict_img = {}, {}
        if output_predict:
            pt = txt_ids[rank_txt.long()].cpu().tolist()
            pi = img_ids[rank_img.long()].cpu().tolist()
            predict_txt = dict(zip(img_ids.cpu().tolist(), pt))
            predict_img = dict(zip(txt_ids.cpu().tolist(), pi))
        return {"txt_r1": tr[0], "txt_r5": tr[1], "txt_r10": tr[2], "txt_r_mean": tr_mean, "img_count": n_img,
                "img_r1": ir[0], "img_r5": ir[1], "img_r10": ir[2], "img_r_mean": ir_mean, "r_mean": (tr_mean + ir_mean) / 2,
                "txt_count": n_txt, "predict_txt": predict_txt, "predict_img": predict_img}
