"""Drop-in for the reference ``MultiheadAttention`` (models/transformer/multihead_attention.py:29-126).

Same constructor arguments and parameter names (q_proj / k_proj (no bias) / v_proj / out_proj / ln /
c_attn).  The module holds the parameters and launches the fused bias+softmax+PV attention kernel
(:108-115, `run_attention`).  The QKV and out_proj GEMMs (:103-107, :124), with the LayerNorms folded into
them, are issued by the enclosing layer (TransformerEncoderLayer.forward_rows_fused) and by the training
forward (autograd.layer_forward).
"""
import torch
import torch.nn as nn

from .. import kernels as K
from ..components import LayerNorm, Linear


class MultiheadAttention(nn.Module):
    def __init__(self, embed_dim, num_heads, dropout=0.0, scale_heads=False, magneto_scale_attn=False):
        super().__init__()
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.dropout_p = dropout
        self.head_dim = embed_dim // num_heads
        assert self.head_dim * num_heads == self.embed_dim, "embed_dim must be divisible by num_heads"
        if self.head_dim != 64:
            raise NotImplementedError("the sm_90a attention kernel is built for head_dim 64 (all ONE-PEACE configs)")
        self.scaling = self.head_dim ** -0.5
        self.c_attn = nn.Parameter(torch.ones((self.num_heads,)), requires_grad=True) if scale_heads else None
        self.ln = LayerNorm(self.embed_dim) if magneto_scale_attn else None
        self.k_proj = Linear(embed_dim, embed_dim, bias=False)
        self.v_proj = Linear(embed_dim, embed_dim, bias=True)
        self.q_proj = Linear(embed_dim, embed_dim, bias=True)
        self.out_proj = Linear(embed_dim, embed_dim, bias=True)

    def run_attention(self, qkv, bias, key_pad, B, S, out=None, ln_stats=None, lse=None):
        """bias: kernels.RelPosBias (or None), in LUT form (the adapters build it for S <= kernels.ATTN_TC_MAX_S) or as a
        dense table; mma.sync either way."""
        if bias is not None and bias.lut is not None:
            return K.attention_tc(qkv, bias, key_pad, B, S, self.num_heads, out=out, ln_stats=ln_stats, lse=lse)
        dense = bias.dense if bias is not None else None
        return K.attention(qkv, dense, key_pad, B, S, self.num_heads, out=out, ln_stats=ln_stats, lse=lse)
