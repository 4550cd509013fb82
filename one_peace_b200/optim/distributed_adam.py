"""First-party replacement for Apex ``DistributedFusedAdam`` (reference: optim/distributed_fused_adam.py:14,
optim/adam.py:68-70 — ``use_distributed_fused_adam: true`` in every 4B recipe, finetune_3B.yaml:21; SURVEY.md 8f row 4):
ZeRO-1 style optimizer-state sharding over the data-parallel ranks, fused with the gradient exchange.

    step():   flat gradient buffer  --reduce-scatter (NCCL, mean)-->  this rank's 1/W shard
              shard grad-norm (two-stage fixed-order kernel) + one scalar all-reduce  ->  global norm, clip coefficient
              fused Adam on the shard (opb_adam_multi_step: fp32 master / m / v exist ONLY for the shard)
              updated shard  --all-gather (NCCL)-->  flat parameter buffer the model's parameters are views of

so the separate gradient all-reduce of LegacyDDP, the clip pass and the optimizer pass collapse into
reduce-scatter + one kernel + all-gather, and optimizer state costs 12 B/param / W instead of 12 B/param.
Arithmetic of the update = the reference's python ``Adam.step`` (optim/adam.py:173-253), as in ``optim/adam.py`` here.

The partitioning (``shard_layout`` / ``shard_segments``) is pure Python and unit-tested on CPU over gloo with the
oracle's ``adam_step`` standing in for the kernel (tests/test_distributed_gloo.py).
"""
import ctypes
import math

import torch
import torch.distributed as dist

from .. import _lib
from .adam import _MAX_GROUPS, _Table


def shard_layout(numels, world, align=8):
    """Flat layout of the parameters: every parameter starts at a multiple of `align` elements (16-byte vectors for
    bf16) and the total is padded to world * align.  -> (offsets, total, shard_size)"""
    offsets, off = [], 0
    for n in numels:
        offsets.append(off)
        off += (n + align - 1) // align * align
    q = world * align
    total = (off + q - 1) // q * q
    return offsets, total, total // world


def shard_segments(offsets, numels, lo, hi):
    """Intersections of the parameters with the flat range [lo, hi): list of (param index, start inside the parameter,
    length, start inside the shard)."""
    segs = []
    for i, (off, n) in enumerate(zip(offsets, numels)):
        a, b = max(off, lo), min(off + n, hi)
        if a < b:
            segs.append((i, a - off, b - a, a - lo))
    return segs


class DistributedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, process_group=None):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.pg = process_group
        self.world = dist.get_world_size(self.pg) if dist.is_initialized() else 1
        self.rank = dist.get_rank(self.pg) if dist.is_initialized() else 0
        self._plist = [(gi, p) for gi, g in enumerate(self.param_groups) for p in g["params"]]
        if not self._plist:
            raise ValueError("no parameters")
        p0 = self._plist[0][1]
        if any(p.dtype != p0.dtype or p.device != p0.device for _, p in self._plist):
            raise NotImplementedError("DistributedAdam shards one flat buffer: parameters must share dtype and device")
        if not p0.is_cuda:
            raise RuntimeError("one_peace_b200 DistributedAdam needs CUDA parameters (there is no CPU path)")
        self.dtype, self.device = p0.dtype, p0.device
        numels = [p.numel() for _, p in self._plist]
        self.offsets, self.total, self.shard = shard_layout(numels, self.world)
        self.lo, self.hi = self.rank * self.shard, (self.rank + 1) * self.shard
        # parameters become views of one flat buffer: the all-gather of the updated shards IS the parameter update
        self.flat_param = torch.zeros(self.total, dtype=self.dtype, device=self.device)
        with torch.no_grad():
            for (gi, p), off in zip(self._plist, self.offsets):
                self.flat_param[off:off + p.numel()].copy_(p.detach().reshape(-1))
                p.data = self.flat_param[off:off + p.numel()].view(p.shape)
        self.flat_grad = torch.zeros(self.total, dtype=self.dtype, device=self.device)
        self.gshard = torch.zeros(self.shard, dtype=self.dtype, device=self.device)
        self.pshard = self.flat_param[self.lo:self.hi].clone()
        self.master = self.pshard.float() if self.dtype != torch.float32 else None
        self.exp_avg = torch.zeros(self.shard, dtype=torch.float32, device=self.device)
        self.exp_avg_sq = torch.zeros(self.shard, dtype=torch.float32, device=self.device)
        self.segs = shard_segments(self.offsets, numels, self.lo, self.hi)
        self._table, self._norm_table = _Table(), _Table()
        # one step count per parameter, as the reference's python Adam keeps it (optim/adam.py:207-213): a parameter whose
        # first gradient comes later than its group-mates' gets its own bias correction
        self.steps = [0] * len(self._plist)
        self._pending = None
        self._has_grad = [True] * len(self._plist)

    @property
    def supports_memory_efficient_fp16(self):
        return True

    @property
    def supports_flat_params(self):
        return True

    def _entries(self):
        """Shard segments of the parameters that received a gradient this step (the reference's python Adam skips
        `p.grad is None`, adam.py:188-190; every data-parallel rank runs the same graph, so the set is rank-invariant).
        The last field is the parameter's (param group, step count) key: the kernel's group table holds one VIRTUAL group per
        key, as in ``Adam._entries``."""
        out = []
        for pi, _, ln, so in self.segs:
            if not self._has_grad[pi]:
                continue
            sl = slice(so, so + ln)
            out.append((self.pshard[sl], self.gshard[sl], self.exp_avg[sl], self.exp_avg_sq[sl],
                        None if self.master is None else self.master[sl], (self._plist[pi][0], self.steps[pi] + 1)))
        return out

    @torch.no_grad()
    def _exchange_grads(self):
        """flat gradient buffer -> reduce-scatter (mean) -> this rank's shard; then the global gradient norm from the
        shard norms (deterministic two-stage kernel + one scalar all-reduce).  -> fp32 device scalar ||g||_2."""
        self._has_grad = [p.grad is not None for _, p in self._plist]
        # one multi-tensor copy instead of ~1900 small launches (26 -> 13 ms of the step at 2.73 B parameters, where the
        # per-parameter loop was bound by Python and launch latency, not by the 11 GB it moves)
        if getattr(self, "_flat_views", None) is None:
            self._flat_views = [self.flat_grad[off:off + p.numel()].view(p.shape) for (_, p), off in zip(self._plist, self.offsets)]
        dsts, srcs = [], []
        for (gi, p), view in zip(self._plist, self._flat_views):
            if p.grad is None:
                view.zero_()
            else:
                dsts.append(view)
                srcs.append(p.grad if p.grad.dtype == view.dtype else p.grad.to(view.dtype))
        if dsts:
            torch._foreach_copy_(dsts, srcs)
        if self.world > 1:
            dist.reduce_scatter_tensor(self.gshard, self.flat_grad, op=dist.ReduceOp.AVG, group=self.pg)
        else:
            self.gshard.copy_(self.flat_grad)
        entries = self._entries()
        sq = torch.zeros(1, dtype=torch.float32, device=self.device)
        if entries:
            nt = self._norm_table
            nt.build([(e[0], e[1], e[1], e[1], None, 0) for e in entries], self.device)
            out2 = torch.empty(2, dtype=torch.float32, device=self.device)
            st = _lib.load().opb_grad_norm_clip(nt.tensors.data_ptr(), nt.chunk_tensor.data_ptr(), nt.chunk_off.data_ptr(),
                                                nt.n_chunks, nt.partial.data_ptr(), 1.0, 0.0, out2.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream)
            _lib.check(st, "opb_grad_norm_clip")
            sq = out2[0:1] * out2[0:1]
        if self.world > 1:
            dist.all_reduce(sq, group=self.pg)
        self._pending = (entries, sq.sqrt())
        return self._pending

    @torch.no_grad()
    def grad_norm_and_scale(self, multiply_factor=1.0, max_norm=0.0):
        """Same contract as optim/adam.py `Adam.grad_norm_and_scale` (used by MemoryEfficientBF16Optimizer.clip_grad_norm):
        fp32 device tensor [2] = {multiply_factor * ||mean-reduced g||_2, grad_scale}.  Performs the gradient exchange;
        the following step() re-uses it."""
        _, norm = self._exchange_grads()
        norm = norm * float(multiply_factor)
        scale = torch.full((1,), float(multiply_factor), dtype=torch.float32, device=self.device)
        if max_norm > 0:
            scale = scale * (max_norm / (norm + 1e-6)).clamp(max=1.0)
        return torch.cat([norm, scale])

    @torch.no_grad()
    def step(self, closure=None, max_norm=0.0, multiply_factor=1.0, grad_scale=None):
        """Returns the global gradient norm (fp32 device scalar, after `multiply_factor`); `max_norm` > 0 clips like
        fairseq's clip_grad_norm_ (coefficient max_norm / (norm + 1e-6), capped at 1).  `grad_scale` (fp32 device scalar)
        is the wrapper's deferred multiply_grads * clip coefficient (fp16_optimizer_memory_efficent.py:118-130); when it
        is given `max_norm` / `multiply_factor` are ignored."""
        loss = closure() if closure is not None else None
        entries, norm = self._pending if self._pending is not None else self._exchange_grads()
        self._pending = None
        norm = norm * multiply_factor
        if grad_scale is not None:
            scale = grad_scale.to(torch.float32).reshape(1)
        else:
            scale = torch.full((1,), float(multiply_factor), dtype=torch.float32, device=self.device)
            if max_norm > 0:
                scale = scale * (max_norm / (norm + 1e-6)).clamp(max=1.0)
        self.last_grad_norm = norm
        if not entries:
            return loss if loss is not None else norm
        lib = _lib.load()
        stream = torch.cuda.current_stream().cuda_stream
        b1, b2 = self.param_groups[0]["betas"]
        eps = self.param_groups[0]["eps"]
        if any(tuple(g["betas"]) != (b1, b2) or g["eps"] != eps for g in self.param_groups):
            raise NotImplementedError("per-group betas / eps (the reference uses one setting for all groups)")
        # virtual groups: one per (param group, step count) in first-seen order
        vmap = {}
        for *_, key in entries:
            vmap.setdefault(key, len(vmap))
        if len(vmap) > _MAX_GROUPS:
            raise NotImplementedError("more (param group, step count) combinations than the kernel's group table")
        keys = list(vmap)
        n = len(keys)
        lr = (ctypes.c_float * n)(*[self.param_groups[gi]["lr"] for gi, _ in keys])
        wd = (ctypes.c_float * n)(*[self.param_groups[gi]["weight_decay"] for gi, _ in keys])
        bcs = (ctypes.c_float * n)(*[math.sqrt(1 - b2 ** t) / (1 - b1 ** t) for _, t in keys])
        # fused Adam on the shard
        t = self._table
        t.build([e[:5] + (vmap[e[5]],) for e in entries], self.device)
        st = lib.opb_adam_multi_step(t.tensors.data_ptr(), t.chunk_tensor.data_ptr(), t.chunk_off.data_ptr(), t.n_chunks,
                                     ctypes.cast(lr, ctypes.c_void_p), ctypes.cast(wd, ctypes.c_void_p),
                                     ctypes.cast(bcs, ctypes.c_void_p), n, b1, b2, eps, scale.data_ptr(), stream)
        _lib.check(st, "opb_adam_multi_step")       # step counts advance only once the launch was accepted
        for pi, has in enumerate(self._has_grad):
            if has:
                self.steps[pi] += 1
        if self.world > 1:
            dist.all_gather_into_tensor(self.flat_param, self.pshard, group=self.pg)
        else:
            self.flat_param.copy_(self.pshard)
        # parameters are views of flat_param written by a collective / raw pointers: bump their version counters so
        # cached kernel-ready packs (components.PackCache) are rebuilt
        torch.autograd.graph.increment_version([p for _, p in self._plist])
        return loss if loss is not None else norm

    def state_bytes_per_rank(self):
        per = 8 + (4 if self.master is not None else 0)
        return self.shard * per

    # ---- checkpointing: rank-local shard state (Apex DistributedFusedAdam also saves per-rank shards) ----
    def state_dict(self):
        groups = [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]
        return {"distributed_adam": {"world": self.world, "rank": self.rank, "total": self.total, "shard": self.shard,
                                     "steps": list(self.steps), "exp_avg": self.exp_avg.clone(),
                                     "exp_avg_sq": self.exp_avg_sq.clone(),
                                     "master": None if self.master is None else self.master.clone()},
                "param_groups": groups}

    def load_state_dict(self, state_dict):
        st = state_dict["distributed_adam"]
        if (st["world"], st["rank"], st["total"], st["shard"]) != (self.world, self.rank, self.total, self.shard):
            raise ValueError("DistributedAdam state was saved with a different world size / rank / parameter layout")
        if "steps" in st:
            if len(st["steps"]) != len(self.steps):
                raise ValueError("DistributedAdam state was saved for a different number of parameters")
            self.steps = [int(t) for t in st["steps"]]
        else:       # a checkpoint from before per-parameter step counts: one step count for every parameter
            self.steps = [int(st["step"])] * len(self.steps)
        self.exp_avg.copy_(st["exp_avg"].to(torch.float32))
        self.exp_avg_sq.copy_(st["exp_avg_sq"].to(torch.float32))
        if self.master is not None:
            if st["master"] is None:
                raise ValueError("state has no fp32 master shard")
            self.master.copy_(st["master"].to(torch.float32))
            self.pshard.copy_(self.master)
        for g, saved in zip(self.param_groups, state_dict["param_groups"]):
            g.update(saved)
