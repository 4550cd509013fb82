"""Drop-in for ``adjust_adam`` (optim/adam.py:51-253): ``AdjustAdam`` (fairseq optimizer wrapper) and the inner
``Adam`` torch optimizer whose ``step`` is ONE fused multi-tensor sm_90a kernel launch.

Arithmetic = the reference's python ``Adam.step`` (:173-253): eps added to the un-bias-corrected sqrt(v),
decoupled weight decay, per-group ``lr`` already scaled by ``lr_scale`` (base_optimizer.py:8-13).  With
``master_weights=True`` an fp32 copy of bf16 parameters is kept and updated (what Apex FusedAdam does in
adam_fused.py:45-50,132-133); without it bf16 parameters are up-cast per step exactly like adam.py:197-199.
"""
import ctypes
import math

import numpy as np
import torch
import torch.optim

from .. import _lib
from ..fairseq_compat import FairseqOptimizer, register_optimizer

_DT = {torch.float32: 0, torch.bfloat16: 1}
_MAX_GROUPS = 128      # opb_adam_multi_step: n_groups <= 128 (include/onepeace_b200.h)


def _ptr(t):
    return 0 if t is None else t.data_ptr()


class Layout:
    """A record layout of the multi-tensor kernels: the numpy dtype of one record (mirroring the C struct) and
    ``pack(entry) -> tuple`` of its field values.  Every record has a ``numel`` field."""

    def __init__(self, dtype, pack):
        self.dtype, self.pack = dtype, pack


# AdamTensor (csrc/ops.h), also read by opb_grad_norm_clip.  entry: (p, g, m, v, master_or_None, group_index)
ADAM_LAYOUT = Layout(
    np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("v", "<u8"), ("master", "<u8"), ("numel", "<i8"),
              ("group", "<i4"), ("p_dtype", "<i4"), ("g_dtype", "<i4"), ("pad", "<i4")]),
    lambda e: (e[0].data_ptr(), e[1].data_ptr(), e[2].data_ptr(), e[3].data_ptr(), _ptr(e[4]), e[0].numel(), e[5],
               _DT[e[0].dtype], _DT[e[1].dtype], 0))
assert ADAM_LAYOUT.dtype.itemsize == 64


class _Table:
    """Device-resident tensor / chunk tables for the multi-tensor kernels; rebuilt only when a record changes (a moved
    pointer, a flag)."""

    def __init__(self, layout=ADAM_LAYOUT):
        self.layout = layout
        self.key = None
        self.shape_key = None

    def build(self, entries, device):
        """entries: what ``layout.pack`` takes (for Adam: (p, g, m, v, master_or_None, group_index)).  The chunk tables
        depend on the tensor sizes only and are kept while those do not change; a changed record (a re-allocated .grad)
        costs one small record upload."""
        key = tuple(self.layout.pack(e) for e in entries)
        if key == self.key:
            return
        rec = np.array(list(key), dtype=self.layout.dtype)
        self.tensors = torch.from_numpy(rec.view(np.uint8).copy()).to(device)
        numels = [int(x) for x in rec["numel"]]
        shape_key = (str(device),) + tuple(numels)
        if shape_key != self.shape_key:
            chunk = _lib.load().opb_adam_chunk_elems()
            ct, co = [], []
            for i, numel in enumerate(numels):
                offs = np.arange(0, numel, chunk, dtype=np.int64)
                ct.append(np.full(len(offs), i, dtype=np.int32))
                co.append(offs)
            self.chunk_tensor = torch.from_numpy(np.concatenate(ct)).to(device)
            self.chunk_off = torch.from_numpy(np.concatenate(co)).to(device)
            self.n_chunks = int(self.chunk_tensor.numel())
            self.partial = torch.empty(self.n_chunks, dtype=torch.float32, device=device)
            self.shape_key = shape_key
        self.key = key


class Adam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False,
                 master_weights=False):
        if amsgrad:
            raise NotImplementedError("amsgrad is not used by any ONE-PEACE config")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad)
        super().__init__(params, defaults)
        self.master_weights = master_weights
        self._table = _Table()
        self._norm_table = _Table()
        self._norm_out = None

    @property
    def supports_memory_efficient_fp16(self):
        return True

    @property
    def supports_flat_params(self):
        return True

    def _entries(self):
        """-> (entries, groups, betas, eps).  `groups` are VIRTUAL groups, one per (param group, step count): the
        reference keeps the step per parameter (adam.py:207-213), so a parameter that receives its first gradient later
        than its group-mates (an unused modality branch) gets its own bias correction."""
        entries, groups, vmap = [], [], {}
        betas = eps = None
        for gi, group in enumerate(self.param_groups):
            if betas is None:
                betas, eps = tuple(group["betas"]), group["eps"]
            elif tuple(group["betas"]) != betas or group["eps"] != eps:
                raise NotImplementedError("per-group betas / eps (the reference uses one setting for all groups)")
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("Adam does not support sparse gradients, please consider SparseAdam instead")
                if not p.is_cuda:
                    raise RuntimeError("one_peace_b200 Adam needs CUDA parameters (there is no CPU path)")
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
                    st["exp_avg_sq"] = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
                    if self.master_weights and p.dtype != torch.float32:
                        st["master"] = p.detach().float().clone()
                for k in ("exp_avg", "exp_avg_sq", "master"):      # state restored from a checkpoint may be bf16 / on CPU
                    if k in st and (st[k].dtype != torch.float32 or st[k].device != p.device):
                        st[k] = st[k].to(device=p.device, dtype=torch.float32)
                t = int(st["step"]) + 1
                vg = vmap.get((gi, t))
                if vg is None:
                    if len(groups) >= _MAX_GROUPS:
                        raise NotImplementedError("more (param group, step count) combinations than the kernel's group table")
                    vg = vmap[(gi, t)] = len(groups)
                    groups.append((group["lr"], group["weight_decay"], math.sqrt(1 - b2 ** t) / (1 - b1 ** t)))
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                if g is not p.grad:
                    p.grad = g
                entries.append((p.data, g, st["exp_avg"], st["exp_avg_sq"], st.get("master"), vg, p))
        return entries, groups, betas, eps

    @torch.no_grad()
    def step(self, closure=None, grad_scale=None):
        """grad_scale: optional fp32 device scalar multiplied into every gradient inside the kernel (the deferred
        multiply_grads * clip coefficient of MemoryEfficientFP16Optimizer, fp16_optimizer_memory_efficent.py:118-130)."""
        loss = closure() if closure is not None else None
        entries, groups, betas, eps = self._entries()
        if not entries:
            return loss
        dev = entries[0][0].device
        self._table.build([e[:6] for e in entries], dev)
        n = len(groups)
        lr = (ctypes.c_float * n)(*[g[0] for g in groups])
        wd = (ctypes.c_float * n)(*[g[1] for g in groups])
        bc = (ctypes.c_float * n)(*[g[2] for g in groups])
        t = self._table
        st = _lib.load().opb_adam_multi_step(t.tensors.data_ptr(), t.chunk_tensor.data_ptr(), t.chunk_off.data_ptr(),
                                             t.n_chunks, ctypes.cast(lr, ctypes.c_void_p), ctypes.cast(wd, ctypes.c_void_p),
                                             ctypes.cast(bc, ctypes.c_void_p), n, betas[0], betas[1], eps,
                                             0 if grad_scale is None else grad_scale.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream)
        _lib.check(st, "opb_adam_multi_step")       # state is only advanced once the launch was accepted
        params = [e[6] for e in entries]
        for p in params:
            self.state[p]["step"] += 1
        # the kernel wrote the parameters through raw pointers: tell autograd / PackCache (components.py) that they changed
        torch.autograd.graph.increment_version(params)
        return loss

    def load_state_dict(self, state_dict):
        """torch's Optimizer.load_state_dict casts floating-point state to the PARAMETER dtype; with bf16 parameters that
        would round exp_avg / exp_avg_sq / the fp32 master to bf16.  Put the saved fp32 tensors back afterwards, as the
        reference wrapper does (fp16_optimizer_memory_efficent.py:44-62)."""
        super().load_state_dict(state_dict)
        from itertools import chain
        saved_ids = chain(*(g["params"] for g in state_dict["param_groups"]))
        params = chain(*(g["params"] for g in self.param_groups))
        id_map = dict(zip(saved_ids, params))
        for k, v in state_dict["state"].items():
            p = id_map.get(k)
            if p is None:
                continue
            st = dict(v)
            for name in ("exp_avg", "exp_avg_sq", "master"):
                if name in st and torch.is_tensor(st[name]):
                    st[name] = st[name].detach().to(device=p.device, dtype=torch.float32).clone()
            if torch.is_tensor(st.get("step")):
                st["step"] = int(st["step"].item())
            self.state[p] = st

    @torch.no_grad()
    def grad_norm_and_scale(self, multiply_factor=1.0, max_norm=0.0):
        return grad_norm_and_scale(self.param_groups, self._norm_table, multiply_factor, max_norm)


@torch.no_grad()
def grad_norm_and_scale(param_groups, table, multiply_factor=1.0, max_norm=0.0):
    """-> fp32 device tensor [2]: {multiply_factor * ||g||_2, grad_scale}, or None without gradients.  One deterministic
    two-stage reduction over every gradient of ``param_groups`` (replaces utils.clip_grad_norm_'s per-tensor norms + stack
    + norm).  ``table``: the caller's ``_Table()`` (Adam layout), kept across steps."""
    entries = []
    for gi, group in enumerate(param_groups):
        for p in group["params"]:
            if p.grad is not None:
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                entries.append((p.data, g, g, g, None, gi))       # only .g / numel / dtype are read
    if not entries:
        return None
    dev = entries[0][0].device
    table.build(entries, dev)     # cached: rebuilding the chunk tables (184 k chunks for the 4B vision branch) every step cost
    #                               0.3 ms of host work + three synchronous uploads, as much as the reduction itself
    out = torch.empty(2, dtype=torch.float32, device=dev)
    st = _lib.load().opb_grad_norm_clip(table.tensors.data_ptr(), table.chunk_tensor.data_ptr(), table.chunk_off.data_ptr(),
                                        table.n_chunks, table.partial.data_ptr(), float(multiply_factor), float(max_norm),
                                        out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(st, "opb_grad_norm_clip")
    return out


@register_optimizer("adjust_adam")
class AdjustAdam(FairseqOptimizer):
    """optim/adam.py:51-110.  `cfg` needs: lr (list), adam_betas, adam_eps, weight_decay; the Apex branches
    (use_distributed_fused_adam / FusedAdam) are replaced by the first-party fused kernel."""

    def __init__(self, cfg, params):
        super().__init__(cfg)
        import torch.distributed as dist
        if bool(getattr(cfg, "use_distributed_fused_adam", False)) and dist.is_initialized() and dist.get_world_size() > 1:
            # adam.py:68-70 hands this case to Apex DistributedFusedAdam; here: first-party ZeRO-1 sharded step
            from .distributed_adam import DistributedAdam
            oc = self.optimizer_config
            oc.pop("master_weights")
            self._optimizer = DistributedAdam(params, **oc)
        else:
            self._optimizer = Adam(params, **self.optimizer_config)

    @property
    def optimizer_config(self):
        betas = self.cfg.adam_betas
        return {"lr": self.cfg.lr[0] if isinstance(self.cfg.lr, (list, tuple)) else self.cfg.lr,
                "betas": eval(betas) if isinstance(betas, str) else tuple(betas),
                "eps": self.cfg.adam_eps, "weight_decay": self.cfg.weight_decay,
                "master_weights": bool(getattr(self.cfg, "master_weights", False))}

    @property
    def optimizer(self):
        return self._optimizer

    @property
    def param_groups(self):
        return self._optimizer.param_groups

    def set_lr(self, lr):
        """optim/base_optimizer.py:8-13: per-group lr = lr * lr_scale."""
        for g in self.param_groups:
            g["lr"] = lr * g.get("lr_scale", 1.0)

    def get_lr(self):
        return self.param_groups[0]["lr"]

    def step(self, closure=None, scale=1.0, groups=None):
        """fairseq_optimizer.py:114-127: `scale` divides the gradients (FusedAdam-style optimizers take it as a kwarg);
        here it is folded into the kernel's grad_scale."""
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
