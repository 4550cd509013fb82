"""TEST INFRASTRUCTURE — not product code.  Stubs for the imports of one_peace_vision/det/models/onepeace.py, on top of
oracle/ref_stub.py's timm shell; only oracle/make_golden_det.py uses it, where the reference tree exists.

  detectron2.modeling.Backbone                   -> nn.Module shell
  detectron2.modeling.backbone.utils.window_partition / window_unpartition / add_decomposed_rel_pos
                                                 restated from detectron2's documented semantics (padding to a multiple of
                                                 the window; linear resize of a rel_pos table of the wrong length)
  detectron2.utils.comm.get_rank                 -> 0
  fairscale.nn.checkpoint.checkpoint_wrapper     -> identity
  timm.models.layers.DropPath                    per-sample stochastic depth (identity in eval)
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

import ref_stub


def window_partition(x, window_size):
    B, H, W, C = x.shape
    pad_h = (window_size - H % window_size) % window_size
    pad_w = (window_size - W % window_size) % window_size
    if pad_h > 0 or pad_w > 0:
        x = F.pad(x, (0, 0, 0, pad_w, 0, pad_h))
    Hp, Wp = H + pad_h, W + pad_w
    x = x.view(B, Hp // window_size, window_size, Wp // window_size, window_size, C)
    windows = x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, window_size, window_size, C)
    return windows, (Hp, Wp)


def window_unpartition(windows, window_size, pad_hw, hw):
    Hp, Wp = pad_hw
    H, W = hw
    B = windows.shape[0] // (Hp * Wp // window_size // window_size)
    x = windows.view(B, Hp // window_size, Wp // window_size, window_size, window_size, -1)
    x = x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, Hp, Wp, -1)
    if Hp > H or Wp > W:
        x = x[:, :H, :W, :].contiguous()
    return x


def get_rel_pos(q_size, k_size, rel_pos):
    max_rel_dist = int(2 * max(q_size, k_size) - 1)
    if rel_pos.shape[0] != max_rel_dist:
        r = F.interpolate(rel_pos.reshape(1, rel_pos.shape[0], -1).permute(0, 2, 1), size=max_rel_dist, mode="linear")
        rel_pos = r.reshape(-1, max_rel_dist).permute(1, 0)
    q_coords = torch.arange(q_size)[:, None] * max(k_size / q_size, 1.0)
    k_coords = torch.arange(k_size)[None, :] * max(q_size / k_size, 1.0)
    relative_coords = (q_coords - k_coords) + (k_size - 1) * max(q_size / k_size, 1.0)
    return rel_pos[relative_coords.long()]


def add_decomposed_rel_pos(attn, q, rel_pos_h, rel_pos_w, q_size, k_size):
    q_h, q_w = q_size
    k_h, k_w = k_size
    Rh = get_rel_pos(q_h, k_h, rel_pos_h)
    Rw = get_rel_pos(q_w, k_w, rel_pos_w)
    B, _, dim = q.shape
    r_q = q.reshape(B, q_h, q_w, dim)
    rel_h = torch.einsum("bhwc,hkc->bhwk", r_q, Rh)
    rel_w = torch.einsum("bhwc,wkc->bhwk", r_q, Rw)
    attn = (attn.view(B, q_h, q_w, k_h, k_w) + rel_h[:, :, :, :, None] + rel_w[:, :, :, None, :]).view(
        B, q_h * q_w, k_h * k_w)
    return attn


class DropPath(nn.Module):
    def __init__(self, drop_prob=0.0):
        super().__init__()
        self.drop_prob = drop_prob

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1 - self.drop_prob
        mask = x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep)
        return x * mask / keep


def install():
    ref_stub.install()
    _m = ref_stub._mod
    tl = _m("timm.models.layers", trunc_normal_=lambda t, mean=0.0, std=1.0, a=-2.0, b=2.0:
            nn.init.trunc_normal_(t, mean=mean, std=std, a=a, b=b), DropPath=DropPath)
    d2 = _m("detectron2")
    d2.__path__ = []
    mod = _m("detectron2.modeling", Backbone=type("Backbone", (nn.Module,), {}))
    mod.__path__ = []
    bb = _m("detectron2.modeling.backbone")
    bb.__path__ = []
    _m("detectron2.modeling.backbone.utils", window_partition=window_partition, window_unpartition=window_unpartition,
       add_decomposed_rel_pos=add_decomposed_rel_pos)
    ut = _m("detectron2.utils")
    ut.__path__ = []
    _m("detectron2.utils.comm", get_rank=lambda: 0)
    fs = _m("fairscale")
    fs.__path__ = []
    fn = _m("fairscale.nn")
    fn.__path__ = []
    _m("fairscale.nn.checkpoint", checkpoint_wrapper=lambda m, *a, **k: m)
    return tl
