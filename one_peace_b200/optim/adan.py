"""Drop-in for ``adan`` (optim/adan.py:32-224): ``FairseqAdan`` (fairseq optimizer wrapper) and the inner ``Adan`` torch
optimizer whose ``step`` is ONE fused multi-tensor sm_90a kernel launch (``opb_adan_multi_step``, csrc/adam.cu).

Arithmetic = the reference's python ``Adan.step`` (:146-223): one step counter per param group, counted on every call
(:160-163); a parameter's first step, or any step at group step 1, takes diff = 0 (:197-198); the proximal weight decay
by default (:216-218).  With ``master_weights=True`` an fp32 copy of bf16 parameters is kept and updated; without it (the
reference's arithmetic) bf16 parameters are up-cast per step and rounded back (:175-177, :222-223), which drops every
update below half a bf16 ulp.

Two behaviours of ``FairseqAdan`` are mirrored as they are (INTEGRATION.md): it subclasses fairseq's FairseqOptimizer,
so ``set_lr`` gives every group the same lr and ignores ``lr_scale``; and ``optimizer_config`` never passes ``no_prox``,
so through fairseq the proximal form is always used.
"""
import ctypes
import math
from collections.abc import Collection
from dataclasses import dataclass, field
from typing import Any, List

import numpy as np
import torch
import torch.optim

from .. import _lib
from ..fairseq_compat import FairseqDataclass, FairseqOptimizer, register_optimizer
from .adam import _DT, _MAX_GROUPS, Layout, _ptr, _Table, grad_norm_and_scale

try:
    from omegaconf import II
except ImportError:            # fairseq (and with it omegaconf) is optional
    II = None

# AdanTensor (csrc/ops.h).  entry: (p, g, m, n, v, pre_grad, master_or_None, group_index, first)
ADAN_LAYOUT = Layout(
    np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("n", "<u8"), ("v", "<u8"), ("pre", "<u8"), ("master", "<u8"),
              ("numel", "<i8"), ("group", "<i4"), ("p_dtype", "<i4"), ("g_dtype", "<i4"), ("first", "<i4")]),
    lambda e: (e[0].data_ptr(), e[1].data_ptr(), e[2].data_ptr(), e[3].data_ptr(), e[4].data_ptr(), e[5].data_ptr(),
               _ptr(e[6]), e[0].numel(), e[7], _DT[e[0].dtype], _DT[e[1].dtype], int(e[8])))
assert ADAN_LAYOUT.dtype.itemsize == 80

_STATE = ("exp_avg", "exp_avg_diff", "exp_avg_sq", "pre_grad", "master")


class Adan(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.98, 0.92, 0.99), eps=1e-8, weight_decay=0.0, no_prox=False,
                 master_weights=False):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, no_prox=no_prox)
        super().__init__(params, defaults)
        self.master_weights = master_weights
        self._table = _Table(ADAN_LAYOUT)
        self._norm_table = _Table()

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("no_prox", False)

    @property
    def supports_memory_efficient_fp16(self):
        return True

    @property
    def supports_flat_params(self):
        return True

    def _entries(self):
        """Advances every group's step (adan.py:160-163, also for a group without gradients) and returns (entries,
        groups, betas, eps); `groups` are the param groups in order, one kernel group each."""
        if len(self.param_groups) > _MAX_GROUPS:
            raise NotImplementedError(f"more than {_MAX_GROUPS} param groups (the kernel's group table)")
        entries, groups = [], []
        betas = eps = None
        for group in self.param_groups:
            if betas is None:
                betas, eps = tuple(group["betas"]), group["eps"]
            elif tuple(group["betas"]) != betas or group["eps"] != eps:
                raise NotImplementedError("per-group betas / eps (the reference uses one setting for all groups)")
        for gi, group in enumerate(self.param_groups):
            b1, b2, b3 = group["betas"]
            t = group["step"] = int(group.get("step", 0)) + 1
            groups.append((group["lr"], group["weight_decay"], int(bool(group["no_prox"])), 1 - b1 ** t, 1 - b2 ** t,
                           math.sqrt(1 - b3 ** t)))
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("Adan does not support sparse gradients, please consider SparseAdam instead")
                if not p.is_cuda:
                    raise RuntimeError("one_peace_b200 Adan needs CUDA parameters (there is no CPU path)")
                st = self.state[p]
                if len(st) == 0:
                    for k in ("exp_avg", "exp_avg_sq", "exp_avg_diff"):
                        st[k] = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
                    if self.master_weights and p.dtype != torch.float32:
                        st["master"] = p.detach().float().clone()
                for k in _STATE:                # state restored from a checkpoint may be bf16 / on CPU
                    if k in st and (st[k].dtype != torch.float32 or st[k].device != p.device or not st[k].is_contiguous()):
                        st[k] = st[k].to(device=p.device, dtype=torch.float32).contiguous()
                first = "pre_grad" not in st or t == 1
                if "pre_grad" not in st:        # written by the kernel before it is ever read
                    st["pre_grad"] = torch.empty(p.shape, dtype=torch.float32, device=p.device)
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                if g is not p.grad:
                    p.grad = g
                entries.append((p.data, g, st["exp_avg"], st["exp_avg_diff"], st["exp_avg_sq"], st["pre_grad"],
                                st.get("master"), gi, first, p))
        return entries, groups, betas, eps

    @torch.no_grad()
    def step(self, closure=None, grad_scale=None):
        """grad_scale: optional fp32 device scalar multiplied into every gradient inside the kernel (the deferred
        multiply_grads * clip coefficient of MemoryEfficientBF16Optimizer); pre_grad keeps the scaled gradient, as the
        reference's in-place multiplied gradients leave it."""
        loss = closure() if closure is not None else None
        saved = [g.get("step") for g in self.param_groups]
        try:
            entries, groups, betas, eps = self._entries()
            if not entries:
                return loss
            dev = entries[0][0].device
            self._table.build([e[:9] for e in entries], dev)
            n = len(groups)
            arr = lambda k, ty=ctypes.c_float: ctypes.cast((ty * n)(*[g[k] for g in groups]), ctypes.c_void_p)
            t = self._table
            st = _lib.load().opb_adan_multi_step(t.tensors.data_ptr(), t.chunk_tensor.data_ptr(), t.chunk_off.data_ptr(),
                                                 t.n_chunks, arr(0), arr(1), arr(2, ctypes.c_int32), arr(3), arr(4), arr(5),
                                                 n, betas[0], betas[1], betas[2], eps,
                                                 0 if grad_scale is None else grad_scale.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream)
            _lib.check(st, "opb_adan_multi_step")
        except Exception:
            for g, s in zip(self.param_groups, saved):     # the step counts only advance once the step was accepted
                if s is None:
                    g.pop("step", None)
                else:
                    g["step"] = s
            raise
        params = [e[9] for e in entries]
        # the kernel wrote the parameters through raw pointers: tell autograd / PackCache (components.py) that they changed
        torch.autograd.graph.increment_version(params)
        return loss

    def load_state_dict(self, state_dict):
        """Loads an ``Adan`` state dict (the reference's or this class's).  torch's Optimizer.load_state_dict casts
        floating-point state to the PARAMETER dtype; with bf16 parameters that would round the moments and pre_grad to
        bf16, so the saved tensors are put back in fp32 afterwards."""
        super().load_state_dict(state_dict)
        _restore_fp32_state(self, state_dict, _STATE)
        for group in self.param_groups:
            group.setdefault("no_prox", False)
            if torch.is_tensor(group.get("step")):
                group["step"] = int(group["step"].item())

    @torch.no_grad()
    def grad_norm_and_scale(self, multiply_factor=1.0, max_norm=0.0):
        """Same contract as ``Adam.grad_norm_and_scale``: fp32 device tensor [2] {multiply_factor * ||g||_2, grad_scale}."""
        return grad_norm_and_scale(self.param_groups, self._norm_table, multiply_factor, max_norm)


def _restore_fp32_state(opt, state_dict, names):
    from itertools import chain
    saved_ids = chain(*(g["params"] for g in state_dict["param_groups"]))
    params = chain(*(g["params"] for g in opt.param_groups))
    id_map = dict(zip(saved_ids, params))
    for k, v in state_dict["state"].items():
        p = id_map.get(k)
        if p is None:
            continue
        st = dict(v)
        for name in names:
            if name in st and torch.is_tensor(st[name]):
                st[name] = st[name].detach().to(device=p.device, dtype=torch.float32).contiguous().clone()
        opt.state[p] = st


@dataclass
class FairseqAdanConfig(FairseqDataclass):
    """optim/adan.py:32-50: the reference's fields; ``tpu`` and ``lr`` are interpolated from common / optimization when
    omegaconf is present (as fairseq resolves them)."""
    adan_betas: Any = field(default=(0.98, 0.92, 0.99), metadata={"help": "betas for Adan optimizer"})
    adan_eps: float = field(default=1e-8, metadata={"help": "epsilon for Adam optimizer"})
    weight_decay: float = field(default=0.0, metadata={"help": "weight decay"})
    no_prox: bool = field(default=False, metadata={"help": "wether to perform prox operator"})
    fp16_adan_stats: bool = field(default=False, metadata={"help": "use FP16 stats (with automatic scaling)"})
    tpu: bool = II("common.tpu") if II is not None else False
    lr: List[float] = II("optimization.lr") if II is not None else field(default_factory=lambda: [1e-3])


@register_optimizer("adan", dataclass=FairseqAdanConfig)
class FairseqAdan(FairseqOptimizer):
    """optim/adan.py:53-111.  `cfg` needs: lr (float or list), adan_betas (sequence or a string such as
    "(0.98,0.92,0.99)"), adan_eps, weight_decay; fp16_adan_stats must be false, as in the reference (:66-78)."""

    def __init__(self, cfg, params):
        super().__init__(cfg)
        if bool(getattr(cfg, "fp16_adan_stats", False)):
            raise NotImplementedError("--fp16-adam-stats is only supported with FusedAdanV1")
        self._optimizer = Adan(params, master_weights=bool(getattr(cfg, "master_weights", False)),
                               **self.optimizer_config)

    @property
    def optimizer_config(self):
        """adan.py:82-98: no_prox is not passed, so the proximal weight decay is always used through fairseq."""
        lr, betas = self.cfg.lr, self.cfg.adan_betas
        return {"lr": lr[0] if isinstance(lr, Collection) else lr,
                "betas": eval(betas) if isinstance(betas, str) else tuple(betas),
                "eps": self.cfg.adan_eps, "weight_decay": self.cfg.weight_decay}

    @property
    def optimizer(self):
        return self._optimizer

    @property
    def param_groups(self):
        return self._optimizer.param_groups

    def set_lr(self, lr):
        """fairseq's FairseqOptimizer.set_lr: every group gets `lr`; a group's lr_scale is not applied (the reference's
        FairseqAdan does not derive from BaseOptimizer)."""
        for g in self.param_groups:
            g["lr"] = lr

    def get_lr(self):
        return self.param_groups[0]["lr"]

    def step(self, closure=None, scale=1.0, groups=None):
        """fairseq_optimizer.py:114-127: `scale` divides the gradients; here it is folded into the kernel's grad_scale."""
        gs = None
        if scale != 1.0:
            dev = next(p for g in self.param_groups for p in g["params"]).device
            gs = torch.full((1,), 1.0 / float(scale), dtype=torch.float32, device=dev)
        return self._optimizer.step(closure, grad_scale=gs)

    def zero_grad(self):
        for g in self.param_groups:
            for p in g["params"]:
                p.grad = None

    def state_dict(self):
        return self._optimizer.state_dict()

    def load_state_dict(self, state_dict, optimizer_overrides=None):
        self._optimizer.load_state_dict(state_dict)
        if optimizer_overrides:
            for g in self.param_groups:
                g.update(optimizer_overrides)
