"""Optimizer state and gradients sharded across ranks: drop-ins for the two fairscale classes behind the reference's
`--shard_optim --shard_grads` (`OSS` in src/util.py:173-178, `ShardedDataParallel` in train.py:199-208), without
fairscale.

Layout, decided once by `OSS.__init__` (oracle/shard_oracle.py states it in numpy):
  * the optimizer's parameters, in `params` order, become views of ONE flat buffer of their common dtype (a mix of
    dtypes raises: cast the model first, as `--precision` does), zero-padded to a multiple of W * 64 elements;
  * rank r owns the contiguous elements [r * S, (r + 1) * S), S = padded / W, and keeps the fp32 copy and both AdamW
    moments for those S elements only: 12 bytes per parameter / W instead of 12;
  * a segment is a parameter intersected with the rank's shard.  The update is the kernel of `AdamWFP32Copy`
    (`atlas_b200_adamw_fp32copy`) with one descriptor per segment, every pointer offset to the segment's first element,
    one launch per param group: each element comes out bit for bit as `AdamWFP32Copy` computes it from the same gradient.

Gradients (`ShardedDataParallel`): every forward with grad mode on installs each parameter's `.grad` as a view of a flat
gradient buffer laid out like the parameters, zeroing it first, unless the views are already in place.  Autograd then
accumulates in place across backward calls (`--accumulation_steps`); `zero_grad()` (set to None) starts a new
accumulation.  The first `clip_grad_norm` or `step` after a forward divides the buffer by W in place and runs ONE
`reduce_scatter_tensor` into the rank's shard, which gives DDP's average.  This communication starts after the backward:
it is not overlapped with it.  `step` updates the shard, then ONE in-place `all_gather_into_tensor` of the flat
parameter buffer gives every rank the new weights.

With one rank or without a process group there is no communication and both classes behave like `AdamWFP32Copy` and
the plain module.  `OSS` without `ShardedDataParallel` reads the gradients from `p.grad` (already averaged by DDP, or
a single rank's) and updates its shard from them.

Checkpoints: `consolidate_state_dict(recipient_rank)` gathers the shards to host memory on the recipient, whose
`state_dict()` then returns `AdamWFP32Copy`'s format (`state[i] = {step, float32copy, exp_avg, exp_avg_sq}` per global
parameter index, plus `param_groups`); `load_state_dict(full_dict)` on every rank keeps that rank's part of such a dict
(written by `AdamWFP32Copy`, by `OSS` at any world size, or by the reference) in fp32.  src/model_io.py:244 frees the
consolidated copy with `optimizer._all_states = []`, as with fairscale.
"""
import numpy as np
import torch
import torch.distributed as dist

from ._lib import AtlasB200Error
from .optim import AdamWFP32Copy, _kind, adamw_launch, bias_corrections, grad_stats_launch

ALIGN = 64          # shard boundaries fall on multiples of 64 elements


def _world(group):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


class OSS(torch.optim.Optimizer):
    """fairscale's `OSS(params, optim=AdamWFP32Copy, ...)`: `AdamWFP32Copy` whose state lives only for the rank's
    shard of the flat parameter buffer.  `param_groups` has torch's shape, so LR schedulers adjust `lr` as usual."""

    def __init__(self, params, optim=AdamWFP32Copy, group=None, force_broadcast_object=False, lr=1e-3,
                 betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, maximize=False):
        # force_broadcast_object only steers how fairscale moves state objects; the state here moves as tensors
        if optim is not AdamWFP32Copy:
            raise AtlasB200Error(f"OSS: optim={optim!r} is not implemented (only atlas_b200.optim.AdamWFP32Copy)")
        if amsgrad or maximize:
            raise AtlasB200Error("OSS: amsgrad / maximize are not implemented")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False,
                                      maximize=False))
        self.group = group
        self.world_size, self.rank = _world(group)
        self._params = [p for g in self.param_groups for p in g["params"]]
        dtypes = sorted({str(p.dtype) for p in self._params})
        if len(dtypes) != 1:
            raise AtlasB200Error(f"OSS: the parameters mix dtypes {dtypes}; one flat buffer needs one dtype")
        dtype = self._params[0].dtype
        _kind(self._params[0], "OSS parameter")
        devices = {p.device for p in self._params}
        if len(devices) != 1 or next(iter(devices)).type != "cuda":
            raise AtlasB200Error(f"OSS: parameters must live on one CUDA device (no CPU path), got {devices}")
        numels = np.array([p.numel() for p in self._params], dtype=np.int64)
        self._offsets = np.concatenate([[0], np.cumsum(numels)[:-1]]).astype(np.int64)
        self._numels = numels
        unit = self.world_size * ALIGN
        self._padded = -(-int(numels.sum()) // unit) * unit
        self._shard_size = self._padded // self.world_size
        self._flat = torch.zeros(self._padded, dtype=dtype, device=next(iter(devices)))
        with torch.no_grad():
            for p, o, n in zip(self._params, self._offsets.tolist(), numels.tolist()):
                view = self._flat[o:o + n]
                view.copy_(p.detach().reshape(-1))
                p.data = view.view(p.shape)
        lo, hi = self.rank * self._shard_size, (self.rank + 1) * self._shard_size
        self._group_index, self._segments, self._segment_of = [], [], {}
        first = 0
        for g in self.param_groups:
            idx = list(range(first, first + len(g["params"])))
            first += len(idx)
            segs = []
            for i in idx:
                o, n = int(self._offsets[i]), int(numels[i])
                a, b = max(o, lo), min(o + n, hi)
                if a < b:
                    segs.append((i, a, b))
                    self._segment_of[i] = (a, b)
            self._group_index.append(idx)
            self._segments.append(segs)
        self._steps = np.zeros(len(self._params), dtype=np.int64)
        self._master = self._exp_avg = self._exp_avg_sq = None     # fp32 [S], created at the first step or load
        self._grad_flat = None        # set up by ShardedDataParallel: the flat local gradient buffer
        self._grad_shard = None       # the rank's reduced gradient ([S] of the flat dtype)
        self._pending_reduce = False
        self._all_states = []         # the consolidated state dict, on the recipient rank

    def add_param_group(self, param_group):
        if hasattr(self, "_flat"):
            raise AtlasB200Error("OSS: the flat layout is fixed at construction; add_param_group is not supported")
        super().add_param_group(param_group)

    # ---- gradients ------------------------------------------------------------------------------------------------
    def _grads_are_views(self):
        if self._grad_flat is None:
            return False
        base, es = self._grad_flat.data_ptr(), self._grad_flat.element_size()
        return all(p.grad is not None and p.grad.data_ptr() == base + o * es
                   for p, o in zip(self._params, self._offsets.tolist()))

    def _prepare_grads(self):
        """Called by ShardedDataParallel.forward: (re)install the gradient views when they are not in place."""
        if not self._grads_are_views():
            if self._grad_flat is None:
                self._grad_flat = torch.zeros_like(self._flat)
                lo = self.rank * self._shard_size
                self._grad_shard = (self._grad_flat[lo:lo + self._shard_size] if self.world_size == 1
                                    else torch.empty(self._shard_size, dtype=self._flat.dtype, device=self._flat.device))
            else:
                self._grad_flat.zero_()
            for p, o, n in zip(self._params, self._offsets.tolist(), self._numels.tolist()):
                p.grad = self._grad_flat[o:o + n].view(p.shape)
        self._pending_reduce = True

    def _reduce(self):
        if not self._pending_reduce:
            return
        self._pending_reduce = False
        if self.world_size > 1:
            self._grad_flat.div_(self.world_size)
            dist.reduce_scatter_tensor(self._grad_shard, self._grad_flat, group=self.group)

    def _segment_grads(self, segs):
        """[(segment, grad pointer of its first element, grad kind)] for the segments whose parameter has a gradient,
        plus the tensors to keep alive."""
        out, keep = [], []
        lo = self.rank * self._shard_size
        sharded = self._grad_flat is not None
        es = self._flat.element_size()
        for i, a, b in segs:
            g = self._params[i].grad
            if g is None:
                continue
            if sharded:
                if g.data_ptr() != self._grad_flat.data_ptr() + int(self._offsets[i]) * es:
                    raise AtlasB200Error("OSS: a gradient under ShardedDataParallel was replaced; call zero_grad() "
                                         "and run the forward through the wrapped module")
                out.append(((i, a, b), self._grad_shard.data_ptr() + (a - lo) * es, _kind(self._flat, "gradient")))
            else:
                g = g if g.is_contiguous() else g.contiguous()
                keep.append(g)
                out.append(((i, a, b), g.data_ptr() + (a - int(self._offsets[i])) * g.element_size(),
                            _kind(g, "gradient")))
        return out, keep

    @torch.no_grad()
    def clip_grad_norm(self, max_norm, norm_type=2.0):
        """fairscale's `OSS.clip_grad_norm` (= torch.nn.utils.clip_grad_norm_'s rule): total = sqrt(all_reduce(sum of
        the shard's squared gradients)) in fp32; the shard gradient is multiplied in place by
        min(1, max_norm / (total + 1e-6)).  Returns `total` as a device tensor; nothing is read back to the host."""
        if float(norm_type) != 2.0:
            raise AtlasB200Error("OSS.clip_grad_norm: only the 2-norm is implemented")
        self._reduce()
        segs, _ = self._segment_grads([s for group in self._segments for s in group])
        device = self._flat.device
        if segs:
            stats = grad_stats_launch([(ptr, b - a, kind, 0) for (_, a, b), ptr, kind in segs], device)
            sq = (stats[:, 3] * stats[:, 3]).sum()
        else:
            sq = torch.zeros((), dtype=torch.float32, device=device)
        if self.world_size > 1:
            dist.all_reduce(sq, group=self.group)
        total = sq.sqrt()
        coef = (float(max_norm) / (total + 1e-6)).clamp(max=1.0)
        if self._grad_flat is not None:
            self._grad_shard.mul_(coef)
        elif segs:
            views = [self._params[i].grad.view(-1)[a - int(self._offsets[i]):b - int(self._offsets[i])]
                     for (i, a, b), _, _ in segs]
            torch._foreach_mul_(views, coef)
        return total

    # ---- update ---------------------------------------------------------------------------------------------------
    def _init_state(self):
        lo = self.rank * self._shard_size
        self._master = self._flat[lo:lo + self._shard_size].to(torch.float32, copy=True)
        self._exp_avg = torch.zeros_like(self._master)
        self._exp_avg_sq = torch.zeros_like(self._master)

    @torch.no_grad()
    def step(self, closure=None, scale=1.0):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self._reduce()
        if self._master is None:
            self._init_state()
        lo = self.rank * self._shard_size
        es = self._flat.element_size()
        pkind = _kind(self._flat, "parameter")
        fp, mp, ap, vp = (t.data_ptr() for t in (self._flat, self._master, self._exp_avg, self._exp_avg_sq))
        live = []
        for group, idx, segs in zip(self.param_groups, self._group_index, self._segments):
            if group.get("amsgrad", False) or group.get("maximize", False):
                raise AtlasB200Error("OSS: amsgrad / maximize are not implemented")
            for i in idx:                     # step counts are global: every rank counts every parameter
                if self._params[i].grad is not None:
                    self._steps[i] += 1
            grads, keep = self._segment_grads(segs)
            rows = [(fp + a * es, mp + (a - lo) * 4, ap + (a - lo) * 4, vp + (a - lo) * 4, gptr, b - a, pkind, gkind)
                    + bias_corrections(group, int(self._steps[i])) for (i, a, b), gptr, gkind in grads]
            if rows:
                live.append((adamw_launch(rows, group, scale, self._flat.device), keep))
        self._live = live             # the tables are read asynchronously: keep them until the next step
        if self.world_size > 1:
            dist.all_gather_into_tensor(self._flat, self._flat[lo:lo + self._shard_size], group=self.group)
        from .retrievers import _bump_weights_epoch

        _bump_weights_epoch()          # the kernel and the all-gather wrote the parameters behind autograd
        return loss

    # ---- checkpoints ----------------------------------------------------------------------------------------------
    def _global_rank(self, r):
        return r if self.group is None else dist.get_global_rank(self.group, r)

    def _gather_state(self, recipient_rank):
        """{key: fp32 host [padded]} on the recipient (None elsewhere, or before the first step)."""
        if self._master is None:
            return None
        S = self._shard_size
        out = {} if self.rank == recipient_rank else None
        for key, buf in (("float32copy", self._master), ("exp_avg", self._exp_avg), ("exp_avg_sq", self._exp_avg_sq)):
            full = torch.empty(self._padded, dtype=torch.float32) if out is not None else None
            tmp = torch.empty_like(buf) if self.world_size > 1 else None
            for r in range(self.world_size):       # one shard at a time: a rank holds at most one extra shard
                src = buf if r == self.rank else tmp
                if self.world_size > 1:
                    dist.broadcast(src, src=self._global_rank(r), group=self.group)
                if full is not None:
                    full[r * S:(r + 1) * S].copy_(src)
            if out is not None:
                out[key] = full
        return out

    def _full_state_dict(self, full):
        groups = []
        for g, idx in zip(self.param_groups, self._group_index):
            d = {k: v for k, v in g.items() if k != "params"}
            d["params"] = list(idx)
            groups.append(d)
        state = {}
        if full is not None:
            for i, p in enumerate(self._params):
                if self._steps[i] == 0:
                    continue
                o, n = int(self._offsets[i]), int(self._numels[i])
                state[i] = {"step": int(self._steps[i])}
                for key in ("float32copy", "exp_avg", "exp_avg_sq"):
                    state[i][key] = full[key][o:o + n].view(p.shape)
        return {"state": state, "param_groups": groups}

    def consolidate_state_dict(self, recipient_rank=0):
        """Collective: gathers every rank's shard to host memory on `recipient_rank`."""
        full = self._gather_state(recipient_rank)
        self._all_states = [self._full_state_dict(full)] if self.rank == recipient_rank else []

    def state_dict(self):
        """`AdamWFP32Copy`'s format.  With more than one rank, only on the recipient of `consolidate_state_dict`."""
        if self.world_size == 1:
            return self._full_state_dict(self._gather_state(0))
        if not self._all_states:
            raise RuntimeError("OSS: call consolidate_state_dict() on every rank first; state_dict() is available "
                               "on the recipient rank only")
        return self._all_states[0]

    def load_state_dict(self, state_dict):
        """Keeps this rank's part of a full (consolidated or `AdamWFP32Copy`) state dict; any saving world size."""
        saved_groups = state_dict["param_groups"]
        if len(saved_groups) != len(self.param_groups) or any(
                len(sg["params"]) != len(g["params"]) for sg, g in zip(saved_groups, self.param_groups)):
            raise ValueError("loaded state dict has a different number of parameter groups or parameters")
        ids = {}
        for sg, g, idx in zip(saved_groups, self.param_groups, self._group_index):
            g.update({k: v for k, v in sg.items() if k != "params"})
            ids.update(zip(sg["params"], idx))
        self._steps[:] = 0
        state = state_dict["state"]
        if not state:
            self._master = self._exp_avg = self._exp_avg_sq = None
            return
        self._init_state()
        lo = self.rank * self._shard_size
        for sid, st in state.items():
            i = ids[int(sid)]
            self._steps[i] = int(st["step"])
            if i not in self._segment_of:
                continue
            a, b = self._segment_of[i]
            o = int(self._offsets[i])
            for key, buf in (("float32copy", self._master), ("exp_avg", self._exp_avg), ("exp_avg_sq", self._exp_avg_sq)):
                buf[a - lo:b - lo].copy_(st[key].reshape(-1)[a - o:b - o])


class ShardedDataParallel(torch.nn.Module):
    """fairscale's `ShardedDataParallel(module, optimizer, auto_refresh_trainable=False)`: gradients accumulate in the
    optimizers' flat buffers and are reduce-scattered to their owners by the first `clip_grad_norm` / `step`.
    Attributes the module has (`encoder`, `generate`, ...) are reachable through the wrapper.  `auto_refresh_trainable`
    is accepted and ignored: the set of parameters is the one fixed by the optimizers."""

    def __init__(self, module, sharded_optimizer, process_group=None, sync_models_at_startup=True,
                 auto_refresh_trainable=True):
        super().__init__()
        self.module = module
        optims = list(sharded_optimizer) if isinstance(sharded_optimizer, (list, tuple)) else [sharded_optimizer]
        if not optims or not all(isinstance(o, OSS) for o in optims):
            raise AtlasB200Error("ShardedDataParallel: needs atlas_b200.sharded.OSS optimizers")
        mine = {id(p) for p in module.parameters()}
        if any(id(p) not in mine for o in optims for p in o._params):
            raise AtlasB200Error("ShardedDataParallel: the optimizer holds parameters that are not the module's")
        self._optims = optims
        if sync_models_at_startup:      # the replicas start from rank 0's weights, as fairscale's do
            with torch.no_grad():
                for o in optims:
                    if o.world_size > 1:
                        dist.broadcast(o._flat, src=o._global_rank(0), group=o.group)

    def forward(self, *args, **kwargs):
        if torch.is_grad_enabled():
            for o in self._optims:
                o._prepare_grads()
        return self.module(*args, **kwargs)

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self._modules["module"], name)
