"""Optimiser step and gradient statistics of the training loop as multi-tensor kernels (csrc/optim.cu).

Drop-ins for `src/AdamWFP32Copy.py` (`AdamWFP32Copy`, selected by `--precision bf16` in `src/util.py:158-166`) and
`src/util.py:200-222` (`compute_grad_stats`).  Same constructor, same `step(closure=None, scale=1.0)`, same state-dict
keys (`step`, `float32copy`, `exp_avg`, `exp_avg_sq`), so checkpoints written by the reference resume here and vice versa.

One kernel launch updates every parameter of a group (the reference runs torch's foreach AdamW on the fp32 copies plus
one `p.copy_(float32copy)` per parameter); the statistics come back as ONE [n, 4] device tensor instead of four `.item()`
synchronisations per parameter.  After a step the 16-bit weight caches of the models are marked stale
(`retrievers._WEIGHTS_EPOCH`), which the reference does not need.

No CPU path: parameters must live on a CUDA device; `amsgrad`, `maximize` and sparse gradients raise.
"""
import math

import numpy as np
import torch

from ._lib import AtlasB200Error, check, current_stream_ptr, lib

CHUNK = 65536          # elements per (tensor, chunk) work item

_ADAM_DESC = np.dtype([("param", "<u8"), ("master", "<u8"), ("exp_avg", "<u8"), ("exp_avg_sq", "<u8"), ("grad", "<u8"),
                       ("numel", "<i8"), ("param_kind", "<i4"), ("grad_kind", "<i4"), ("bc1", "<f4"), ("bc2s", "<f4")])
_GRAD_DESC = np.dtype([("grad", "<u8"), ("numel", "<i8"), ("grad_kind", "<i4"), ("pad", "<i4")])
assert _ADAM_DESC.itemsize == 64 and _GRAD_DESC.itemsize == 24

_KIND = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def _kind(t, what):
    try:
        return _KIND[t.dtype]
    except KeyError:
        raise AtlasB200Error(f"{what}: dtype {t.dtype} is not supported (fp32 / bf16 / fp16)")


def _chunk_table(numels):
    """(tensor index, chunk index) int32 pairs covering every element of every tensor."""
    pairs = [np.stack([np.full(-(-n // CHUNK), i, dtype=np.int32), np.arange(-(-n // CHUNK), dtype=np.int32)], 1)
             for i, n in enumerate(numels) if n > 0]
    return np.concatenate(pairs, 0) if pairs else np.zeros((0, 2), dtype=np.int32)


def _to_device(arr, device):
    """Small host table -> device bytes through pinned memory (asynchronous on the current stream)."""
    host = torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1)).pin_memory()
    return host.to(device, non_blocking=True), host


def bias_corrections(group, t):
    """(lr / (1 - beta1^t), sqrt(1 - beta2^t)): derived in double precision like torch, rounded once to fp32 by the
    descriptor table."""
    beta1, beta2 = group["betas"]
    return group["lr"] / (1.0 - beta1 ** t), math.sqrt(1.0 - beta2 ** t)


def adamw_launch(rows, group, scale, device):
    """One `atlas_b200_adamw_fp32copy` launch over `_ADAM_DESC` rows of one param group.  A row is a whole parameter
    (`AdamWFP32Copy`) or a segment of one (`sharded.OSS`: every pointer offset to the segment's first element).  Returns
    the device tables and their pinned staging copies, which must stay alive until the kernel has run."""
    beta1, beta2 = group["betas"]
    descs = np.array(rows, dtype=_ADAM_DESC)
    chunks = _chunk_table([r[5] for r in rows])
    d_dev, h1 = _to_device(descs, device)
    c_dev, h2 = _to_device(chunks, device)
    with torch.cuda.device(device):
        # torch derives these scalars in double precision and rounds them once: do the same
        check(lib().atlas_b200_adamw_fp32copy(d_dev.data_ptr(), c_dev.data_ptr(), int(chunks.shape[0]), CHUNK,
                                              1.0 - float(group["lr"]) * float(group["weight_decay"]), float(beta2),
                                              1.0 - float(beta1), 1.0 - float(beta2), float(group["eps"]),
                                              1.0 / float(scale), current_stream_ptr()))
    return d_dev, c_dev, h1, h2


class AdamWFP32Copy(torch.optim.AdamW):
    """`src/AdamWFP32Copy.py:14-169`: AdamW whose moments and update live on an fp32 copy of every parameter; the
    (bf16) parameter receives the rounded copy after each step."""

    @torch.no_grad()
    def step(self, closure=None, scale=1.0):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            if group.get("amsgrad", False) or group.get("maximize", False):
                raise AtlasB200Error("AdamWFP32Copy (B200): amsgrad / maximize are not implemented")
            rows = []
            keep = []          # tensors that must stay alive until the launch has been enqueued
            device = None
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("AdamW does not support sparse gradients")
                if not p.is_cuda:
                    raise AtlasB200Error("AdamWFP32Copy (B200): parameters must be CUDA tensors (no CPU path)")
                if not p.is_contiguous():
                    raise AtlasB200Error("AdamWFP32Copy (B200): parameters must be contiguous")
                device = p.device
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    copy = p.detach().to(torch.float32, memory_format=torch.preserve_format)
                    state["float32copy"] = copy.clone() if copy.data_ptr() == p.data_ptr() else copy
                    state["exp_avg"] = torch.zeros_like(state["float32copy"], memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(state["float32copy"], memory_format=torch.preserve_format)
                for key in ("float32copy", "exp_avg", "exp_avg_sq"):      # a loaded checkpoint: torch cast the state to bf16
                    if state[key].dtype != torch.float32 or not state[key].is_contiguous():
                        state[key] = state[key].to(torch.float32).contiguous()
                state["step"] = int(state["step"]) + 1
                t = int(state["step"])
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                keep.append(g)
                rows.append((p.data_ptr(), state["float32copy"].data_ptr(), state["exp_avg"].data_ptr(),
                             state["exp_avg_sq"].data_ptr(), g.data_ptr(), p.numel(), _kind(p, "parameter"),
                             _kind(g, "gradient")) + bias_corrections(group, t))
            if not rows:
                continue
            # the tables are read by the kernel asynchronously: keep them (and the pinned staging copies) until the next step
            self._live = (adamw_launch(rows, group, scale, device), keep)
        from .retrievers import _bump_weights_epoch

        _bump_weights_epoch()          # the kernel wrote the parameters behind autograd's version counters
        return loss


def grad_stats_tensor(params):
    """[len(params), 4] fp32 device tensor: (min |g|, max |g|, mean |g|, ||g||_2) per parameter, zeros where p.grad is
    None.  One table upload + three launches, no device synchronisation."""
    params = list(params)
    device = next((p.device for p in params if p.grad is not None), None)
    if device is None or device.type != "cuda":
        if device is not None:
            raise AtlasB200Error("grad_stats: gradients must be CUDA tensors (no CPU path)")
        dev0 = params[0].device if params else torch.device("cuda")
        return torch.zeros((len(params), 4), dtype=torch.float32, device=dev0)
    rows, keep = [], []
    for p in params:
        g = p.grad
        if g is None:
            rows.append((0, 0, 0, 0))
            continue
        g = g if g.is_contiguous() else g.contiguous()
        keep.append(g)
        rows.append((g.data_ptr(), g.numel(), _kind(g, "gradient"), 0))
    out = grad_stats_launch(rows, device)
    out._atlas_keep = (out._atlas_keep, keep)
    return out


def grad_stats_launch(rows, device):
    """[len(rows), 4] fp32 device tensor of (min |g|, max |g|, mean |g|, ||g||_2) for `_GRAD_DESC` rows (grad pointer,
    numel, kind, 0): whole gradients or segments of them (a null pointer or numel 0 gives zeros).  No synchronisation;
    the result keeps the uploaded tables alive."""
    descs = np.array(rows, dtype=_GRAD_DESC)
    chunks = _chunk_table([r[1] for r in rows])
    d_dev, h1 = _to_device(descs, device)
    c_dev, h2 = _to_device(chunks, device)
    out = torch.empty((len(rows), 4), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        check(lib().atlas_b200_grad_stats(d_dev.data_ptr(), len(rows), c_dev.data_ptr(), int(chunks.shape[0]), CHUNK,
                                          out.data_ptr(), current_stream_ptr()))
    out._atlas_keep = (d_dev, c_dev, h1, h2)
    return out


def compute_grad_stats(model):
    """`src/util.py:200-222`: {"skip_example", "min", "max", "mean"} over the reader's parameters (summed over ranks like the
    reference's all_reduce).  ONE host synchronisation (the final read-back) instead of four per parameter.

    With the reader wrapped in `sharded.ShardedDataParallel` each parameter's `.grad` is its view of the flat gradient
    buffer, which holds the rank's LOCAL gradient until the reduce-scatter of the next `clip_grad_norm` / `step`: the
    statistics are those of the W local gradients, summed.  Under DDP every rank holds the averaged gradient, so the
    sum is W copies of the averaged gradient's statistics instead.  The two agree when the local gradients are equal."""
    with torch.no_grad():
        inner = model.module if hasattr(model, "module") else model
        stats = grad_stats_tensor(p for _, p in inner.reader.named_parameters())
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.all_reduce(stats)
        bad = torch.isinf(stats).any() | torch.isnan(stats).any()
        packed = torch.stack([bad.float(), stats[:, 0].min(), stats[:, 1].max(), stats[:, 2].mean()]).cpu()
        return {"skip_example": bool(packed[0].item() != 0), "min": packed[1].item(), "max": packed[2].item(),
                "mean": packed[3].item()}
