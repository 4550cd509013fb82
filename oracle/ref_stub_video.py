"""TEST INFRASTRUCTURE — not product code.  Stubs for the imports of
one_peace_vision/video/mmaction_custom/models/backbones/onepeace.py, on top of oracle/ref_stub.py's shells; only
oracle/make_golden_video.py uses it, where the reference tree exists.

  timm.models.layers.trunc_normal_          -> torch.nn.init.trunc_normal_ (timm's absolute cut-offs a=-2, b=2)
  mmcv.runner.get_dist_info                 -> (0, 1)
  mmaction.utils.get_root_logger            -> a logging.Logger
  mmaction.models.builder.BACKBONES         -> a registry whose register_module() returns the class unchanged
"""
import logging
import sys

import torch.nn as nn

import ref_stub


class _Registry:
    def __init__(self):
        self.module_dict = {}

    def register_module(self, *args, **kwargs):
        def deco(cls):
            self.module_dict[cls.__name__] = cls
            return cls
        return deco


def install():
    ref_stub.install()
    _m = ref_stub._mod
    for pkg in ("timm", "timm.models", "mmcv", "mmaction", "mmaction.models"):
        if pkg not in sys.modules:
            _m(pkg).__path__ = []
    _m("timm.models.layers", trunc_normal_=lambda t, mean=0.0, std=1.0, a=-2.0, b=2.0:
       nn.init.trunc_normal_(t, mean=mean, std=std, a=a, b=b))
    _m("mmcv.runner", get_dist_info=lambda: (0, 1))
    _m("mmaction.utils", get_root_logger=lambda *a, **k: logging.getLogger("mmaction"))
    _m("mmaction.models.builder", BACKBONES=_Registry())
