"""Drop-in for ``TextAdapter`` (models/adapter/text.py:32-185): token embedding + learned absolute positions
+ CLS, and the log-bucket relative-position bias.  Same parameter / buffer names (cls_embedding,
embed_tokens, embed_positions, rel_pos_table_list.N, rp_bucket)."""
import math

import torch

from .. import kernels as K
from .. import relpos
from ..components import Embedding, PackCache, f32, trunc_normal_


def make_token_bucket_position(bucket_size, max_position):
    """Log-spaced relative-position buckets — same index math as models/adapter/text.py:18-29 (int64)."""
    context_pos = torch.arange(max_position, dtype=torch.long)[:, None]
    memory_pos = torch.arange(max_position, dtype=torch.long)[None, :]
    rel = context_pos - memory_pos
    sign = torch.sign(rel)
    mid = bucket_size // 2
    abs_pos = torch.where((rel < mid) & (rel > -mid), mid - 1, torch.abs(rel))
    log_pos = mid + torch.ceil(torch.log(abs_pos / mid) / math.log((max_position - 1) / mid) * (mid - 1)).long()
    bucket_pos = torch.where(abs_pos.le(mid), rel, log_pos * sign).long()
    return bucket_pos + bucket_size - 1


def flat_ids(preserve_ids, seq_len):
    """(B,K) position ids (-1 = padded slot) -> int64 [B*K] flat row indices b * seq_len + id, -1 kept."""
    B = preserve_ids.shape[0]
    base = torch.arange(B, device=preserve_ids.device)[:, None] * seq_len
    return torch.where(preserve_ids >= 0, preserve_ids + base, preserve_ids).reshape(-1).contiguous()


def canvas_index(preserve_ids, seq_len):
    """Inverse of the preserve map for the decoder canvas (adapter/text.py:135-142): int64 [B*seq_len], entry (b, s) = row
    b*K + k of preserve_embed if preserve_ids[b, k] == s, else -1 (mask token)."""
    B, Kk = preserve_ids.shape
    dev = preserve_ids.device
    out = torch.full((B * seq_len,), -1, dtype=torch.int64, device=dev)
    src = torch.arange(B * Kk, device=dev).view(B, Kk)
    dst = preserve_ids + torch.arange(B, device=dev)[:, None] * seq_len
    valid = preserve_ids >= 0
    out[dst[valid]] = src[valid]
    return out


class TextAdapter(torch.nn.Module):
    def __init__(self, cfg, embed_dim, attention_heads, src_dict=None, num_layers=None):
        super().__init__()
        if cfg.layernorm_embedding or cfg.add_type_embedding or cfg.shrink_alpha != 1.0:
            raise NotImplementedError("layernorm_embedding / add_type_embedding / shrink_alpha are off in the 4B config")
        self.attention_heads = attention_heads
        if src_dict is not None:
            self.padding_idx = src_dict.pad()
            self.embed_tokens = Embedding(len(src_dict), embed_dim, self.padding_idx)
        else:
            self.embed_tokens = None
            self.padding_idx = 1
        self.cls_embedding = torch.nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.embed_positions = Embedding(512 + 2, embed_dim)
        if cfg.use_attn_bias:
            num_rel_dis = 2 * cfg.bucket_size - 1
            rp_bucket = make_token_bucket_position(cfg.bucket_size, max_position=1024)
            rp_bucket[0, :] = num_rel_dis
            rp_bucket[:, 0] = num_rel_dis + 1
            rp_bucket[0, 0] = num_rel_dis + 2
            self.register_buffer("rp_bucket", rp_bucket)
            self.rel_pos_table_list = torch.nn.ModuleList(
                [Embedding(num_rel_dis + 3, attention_heads, zero_init=True) for _ in range(num_layers or 1)])
        else:
            self.rel_pos_table_list = None
        trunc_normal_(self.cls_embedding)
        trunc_normal_(self.embed_positions.weight)
        if self.embed_tokens is not None:
            trunc_normal_(self.embed_tokens.weight)
            torch.nn.init.constant_(self.embed_tokens.weight[self.padding_idx], 0)
        self._cache = PackCache()

    def _pack(self):
        ps = [self.cls_embedding, self.embed_positions.weight] + \
             ([t.weight for t in self.rel_pos_table_list] if self.rel_pos_table_list is not None else [])

        def build():
            return dict(cls=f32(self.cls_embedding).view(-1), pos=f32(self.embed_positions.weight),
                        tables=[f32(t.weight) for t in self.rel_pos_table_list] if self.rel_pos_table_list is not None else None)
        return self._cache.get(ps, build)

    def get_rel_pos_bias(self, seq_len):
        """One RelPosBias per table: LUT form for the attention kernel when S <= 384 (kernels.ATTN_TC_MAX_S), dense (H,S,S_pad) otherwise."""
        p = self._pack()
        if not hasattr(self, "_lut_cache"):
            self._lut_cache = relpos.LutCache()
        lut = self._lut_cache.get(seq_len, self.rp_bucket.device, self.rp_bucket, lambda S: relpos.text_codes(S)) if seq_len <= K.ATTN_TC_MAX_S else None
        out = []
        for t in p["tables"]:
            if lut is not None:
                out.append(K.RelPosBias(lut=K.relpos_lut_build(t, lut[0]), code_row=lut[1], code_col=lut[2]))
            else:
                out.append(K.RelPosBias(dense=K.relpos_bias_build(t, self.rp_bucket, seq_len, self.attention_heads)))
        return out

    def bias_source(self, n, ids=None):
        """What the encoder needs to place this modality's relative-position bias block (autograd_general.BlockBiasFn)."""
        if self.rel_pos_table_list is None:
            return None
        return dict(tables=[t.weight for t in self.rel_pos_table_list], bucket=self.rp_bucket, n=n, ids=ids)

    def embed_general(self, src_tokens, preserve_ids=None, preserve_embed=None, mask_token=None):
        """General (pretraining) form of forward (models/adapter/text.py:111-164) -> (x fp32 (B,S,d), pad uint8 (B,S), bias
        source).  preserve_ids (B,K) int64, -1 padded: encoder student pass = rows of (embedding + position) gathered by id
        (:92-95,146-151); with preserve_embed (B,K,d): decoder canvas = mask token everywhere, the preserved rows scattered
        to their positions, plus the positional table (:135-142,157)."""
        from ..autograd import TextEmbedFn
        from ..autograd_general import RowGatherFn
        B, T = src_tokens.shape
        S = T + 1
        d = self.embed_positions.weight.shape[1]
        dev = src_tokens.device
        if preserve_embed is not None:
            src_idx = canvas_index(preserve_ids, S)
            x = RowGatherFn.apply(preserve_embed.reshape(-1, d), src_idx, mask_token, self.embed_positions.weight[:S]).view(B, S, d)
            pad = torch.zeros(B, S, dtype=torch.uint8, device=dev)
            pad[:, 1:] = src_tokens.eq(self.padding_idx)
            return x, pad, self.bias_source(S)
        train = torch.is_grad_enabled() and any(q.requires_grad for q in self.parameters())
        if train:
            x, pad = TextEmbedFn.apply(src_tokens, self.embed_tokens.weight, self.embed_positions.weight, self.cls_embedding,
                                       self.padding_idx)
        else:
            p = self._pack()
            table = self.embed_tokens.weight.detach()
            if table.dtype not in (torch.float32, torch.bfloat16):
                table = table.float()
            x, pad = K.text_embed(src_tokens.contiguous(), table, p["pos"], p["cls"], self.padding_idx)
        if preserve_ids is None:
            return x, pad, self.bias_source(S)
        Kk = preserve_ids.shape[1]
        xg = RowGatherFn.apply(x.reshape(B * S, d), flat_ids(preserve_ids, S), None, None).view(B, Kk, d)
        return xg, preserve_ids.eq(-1).to(torch.uint8).contiguous(), self.bias_source(Kk, preserve_ids.contiguous())

    def forward(self, src_tokens, preserve_ids=None, preserve_embed=None, mask_token=None):
        """-> (x fp32 (B,T+1,d) with padded rows zeroed, padding_mask uint8 (B,T+1), [bias (H,S,S_pad)])"""
        if preserve_ids is not None or preserve_embed is not None:
            return self.embed_general(src_tokens, preserve_ids, preserve_embed, mask_token)
        if torch.is_grad_enabled() and any(q.requires_grad for q in self.parameters()):
            return self.forward_train(src_tokens)
        p = self._pack()
        table = self.embed_tokens.weight.detach()
        if table.dtype not in (torch.float32, torch.bfloat16):
            table = table.float()
        x, pad = K.text_embed(src_tokens.contiguous(), table, p["pos"], p["cls"], self.padding_idx)
        bias = self.get_rel_pos_bias(src_tokens.size(1) + 1) if self.rel_pos_table_list is not None else None
        return x, pad, bias

    def forward_train(self, src_tokens):
        """Same outputs, recorded for autograd: the bias list holds dense (H,S,S_pad) tensors (autograd.RelPosBiasFn)."""
        from ..autograd import RelPosBiasFn, TextEmbedFn, TrainBias
        x, pad = TextEmbedFn.apply(src_tokens, self.embed_tokens.weight, self.embed_positions.weight, self.cls_embedding,
                                   self.padding_idx)
        bias = None
        if self.rel_pos_table_list is not None:
            S = src_tokens.size(1) + 1
            fast = self.get_rel_pos_bias(S)            # LUT form for the attention kernel (S <= 384), same values
            bias = [TrainBias(RelPosBiasFn.apply(t.weight, self.rp_bucket, S, self.attention_heads),
                              f if f.lut is not None else None) for t, f in zip(self.rel_pos_table_list, fast)]
        return x, pad, bias
