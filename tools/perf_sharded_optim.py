"""Sharded optimizer step (atlas_b200/sharded.py) at the reader sizes Atlas trains, per rank:
  * the step split into the reduce-scatter of the gradients, the AdamW update of the shard and the all-gather of the
    parameters (CUDA events; the update is the time of `OSS.step` minus that of an all-gather timed on its own);
  * the update's bytes (28 per shard element: fp32 copy and both moments read and written, 16-bit gradient read and
    parameter written) over the H100 SXM's 3.35 TB/s, the time that bounds it;
  * the peak memory of the step (parameters, gradients, state) against unsharded `AdamWFP32Copy`, measured where it fits
    on the device and computed (16 bytes per parameter) where it does not.
Synthetic bf16 parameters with the parameter counts of the T5 v1.1 / lm-adapt xl and xxl readers (about 2.85 and 11.1
billion), split into tensors of 2^26 elements.  A size that does not fit on the device is reported, not run.  Prints the
card and its power limit with the numbers; one JSON line per size.

    python tools/perf_sharded_optim.py --gpus N [--sizes xl,xxl] [--steps K] [--warmup W] [--out FILE]
With N > 1 the script runs itself under torchrun, one rank per GPU."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = {"xl": 2_850_000_000, "xxl": 11_100_000_000}
PIECE = 1 << 26
HBM = 3.35e12
GB = 1e9


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"{torch.cuda.get_device_name(0)} (power limit not read)"


def params_of(numel, dev):
    sizes = [PIECE] * (numel // PIECE) + ([numel % PIECE] if numel % PIECE else [])
    return [torch.nn.Parameter(torch.empty(n, dtype=torch.bfloat16, device=dev).normal_(0, 0.02)) for n in sizes]


def event_time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps / 1e3


def sharded(numel, world, dev, steps, warmup):
    from atlas_b200.sharded import OSS

    S = -(-numel // (world * 64)) * 64
    need = numel * 2 * 2 + S * 12 + (S * 2 if world > 1 else 0) + PIECE * 2
    free = torch.cuda.mem_get_info(dev)[0]
    fits = torch.tensor([need <= 0.95 * free], dtype=torch.int32, device=dev)
    if world > 1:
        dist.all_reduce(fits, op=dist.ReduceOp.MIN)
    if not bool(fits):
        return {"fits": False, "needs_gb_per_rank": round(need / GB, 2)}
    ps = params_of(numel, dev)
    opt = OSS(ps, lr=1e-4, weight_decay=0.01, betas=(0.9, 0.999), eps=1e-6)
    opt._prepare_grads()                        # the flat gradient views a ShardedDataParallel forward installs
    opt._grad_flat.normal_(0, 1e-3)
    opt.step()                                  # allocate the state
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)

    def rs():
        opt._pending_reduce = True
        opt._reduce()

    def ag():
        if world > 1:
            lo = opt.rank * opt._shard_size
            dist.all_gather_into_tensor(opt._flat, opt._flat[lo:lo + opt._shard_size])

    t_rs = event_time(rs, steps, warmup) if world > 1 else 0.0
    t_step = event_time(opt.step, steps, warmup)
    t_ag = event_time(ag, steps, warmup) if world > 1 else 0.0
    t_upd = t_step - t_ag
    bound = 28 * opt._shard_size / HBM
    return {"fits": True, "reduce_scatter_ms": round(t_rs * 1e3, 3), "update_ms": round(t_upd * 1e3, 3),
            "all_gather_ms": round(t_ag * 1e3, 3), "update_hbm_bound_ms": round(bound * 1e3, 3),
            "update_share_of_hbm_bound": round(bound / t_upd, 3) if t_upd > 0 else None,
            "peak_gb_per_rank": round(torch.cuda.max_memory_allocated(dev) / GB, 2)}


def unsharded(numel, dev, steps, warmup):
    from atlas_b200.optim import AdamWFP32Copy

    need = numel * 16 + PIECE * 4
    if need > 0.95 * torch.cuda.mem_get_info(dev)[0]:
        return {"measured": False, "peak_gb_computed": round(numel * 16 / GB, 2)}
    ps = params_of(numel, dev)
    for p in ps:
        p.grad = torch.empty_like(p).normal_(0, 1e-3)
    opt = AdamWFP32Copy(ps, lr=1e-4, weight_decay=0.01, betas=(0.9, 0.999), eps=1e-6)
    opt.step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    t = event_time(opt.step, steps, warmup)
    return {"measured": True, "update_ms": round(t * 1e3, 3),
            "peak_gb": round(torch.cuda.max_memory_allocated(dev) / GB, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--sizes", default="xl,xxl")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.gpus > 1 and "RANK" not in os.environ:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={a.gpus}",
               "--master-addr", "127.0.0.1", "--master-port", "29911", os.path.abspath(__file__)] + sys.argv[1:]
        sys.exit(subprocess.run(cmd).returncode)
    assert torch.cuda.is_available(), "perf_sharded_optim needs a GPU"
    world = 1
    if "RANK" in os.environ:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
        world = dist.get_world_size()
    rank = dist.get_rank() if world > 1 else 0
    dev = torch.device("cuda", torch.cuda.current_device())
    gpu = card()
    lines = []
    for name in a.sizes.split(","):
        numel = SIZES[name]
        res = {"size": name, "params": numel, "world": world, "rank": rank, "gpu": gpu,
               "sharded": sharded(numel, world, dev, a.steps, a.warmup)}
        torch.cuda.empty_cache()
        if rank == 0:
            res["unsharded_adamw_fp32copy"] = unsharded(numel, dev, a.steps, a.warmup)
            torch.cuda.empty_cache()
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)
        if world > 1:
            dist.barrier()
    if a.out and rank == 0:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
