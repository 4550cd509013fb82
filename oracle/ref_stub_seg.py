"""TEST INFRASTRUCTURE — not product code.  Stubs for the imports of
one_peace_vision/seg/mmseg_custom/models/backbones/{onepeace_adapter,adapter_modules,onepeace}.py, on top of
oracle/ref_stub.py's shells; only oracle/make_golden_seg.py uses it, where the reference tree exists.

  timm.models.layers.trunc_normal_ / DropPath     -> torch.nn.init.trunc_normal_ / identity (drop_path_rate 0)
  mmcv.runner.BaseModule / _load_checkpoint / get_dist_info -> nn.Module with init_cfg / torch.load / (0, 1)
  mmcv.cnn.build_norm_layer                       -> ("ln", nn.LayerNorm(dim)) for type LN, mmcv's default eps
  mmcv.cnn.utils.weight_init                      -> constant_init / kaiming_init / trunc_normal_
  mmseg.utils.get_root_logger                     -> a logging.Logger
  mmseg.models.builder.BACKBONES                  -> a registry whose register_module() returns the class unchanged
  ops.modules.MSDeformAttn                        -> the reference's own module, its CUDA function routed to its own
                                                     ms_deform_attn_core_pytorch (oracle/make_golden_msda.py)
  scipy.interpolate.interp2d                      -> oracle/make_golden_grounding.py's gridded-data stand-in
"""
import importlib
import logging
import os
import sys
import types

import torch
import torch.nn as nn

import ref_stub
import ref_stub_video

BACKBONES_DIR = os.path.join(ref_stub.REF_ROOT, "one_peace_vision", "seg", "mmseg_custom", "models", "backbones")


class _BaseModule(nn.Module):
    def __init__(self, init_cfg=None):
        super().__init__()
        self.init_cfg = init_cfg


def _build_norm_layer(cfg, num_features):
    assert cfg["type"] == "LN"
    return "ln", nn.LayerNorm(num_features)


def _constant_init(m, val, bias=0.0):
    if getattr(m, "weight", None) is not None:
        nn.init.constant_(m.weight, val)
    if getattr(m, "bias", None) is not None:
        nn.init.constant_(m.bias, bias)


def _kaiming_init(m, a=0, mode="fan_out", nonlinearity="relu", bias=0.0, distribution="normal"):
    nn.init.kaiming_normal_(m.weight, a=a, mode=mode, nonlinearity=nonlinearity)
    if getattr(m, "bias", None) is not None:
        nn.init.constant_(m.bias, bias)


def _trunc_normal(t, mean=0.0, std=1.0, a=-2.0, b=2.0):
    return nn.init.trunc_normal_(t, mean=mean, std=std, a=a, b=b)


def install():
    """-> the reference's backbones package (module ``ref_seg_backbones``)."""
    ref_stub_video.install()
    m = ref_stub._mod
    for pkg in ("mmcv.cnn", "mmcv.cnn.utils", "mmseg", "mmseg.models"):
        if pkg not in sys.modules:
            m(pkg).__path__ = []
    sys.modules["timm.models.layers"].DropPath = lambda p=0.0: nn.Identity()
    sys.modules["timm.models.layers"].trunc_normal_ = _trunc_normal
    runner = sys.modules["mmcv.runner"]
    runner.BaseModule = _BaseModule
    runner._load_checkpoint = lambda path, logger=None, map_location=None: torch.load(path, map_location=map_location,
                                                                                      weights_only=False)
    sys.modules["mmcv.cnn"].build_norm_layer = _build_norm_layer
    m("mmcv.cnn.utils.weight_init", constant_init=_constant_init, kaiming_init=_kaiming_init, trunc_normal_=_trunc_normal)
    m("mmseg.utils", get_root_logger=lambda *a, **k: logging.getLogger("mmseg"))
    m("mmseg.models.builder", BACKBONES=ref_stub_video._Registry())
    import make_golden_grounding
    from scipy import interpolate
    interpolate.interp2d = make_golden_grounding._Interp2dStandin
    import make_golden_msda
    make_golden_msda.load_reference()
    pkg = types.ModuleType("ref_seg_backbones")
    pkg.__path__ = [BACKBONES_DIR]
    sys.modules["ref_seg_backbones"] = pkg
    return importlib.import_module("ref_seg_backbones.onepeace_adapter")
