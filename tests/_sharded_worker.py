"""torchrun worker for tests/test_sharded_gpu.py::test_sharded_ranks_nccl (one rank per GPU).

Every rank's local gradient is a multiple of 2^-12 below 2^-6 in magnitude, so the pre-division by W (a power of two)
and every sum of the reduce-scatter are exact whatever NCCL's order: the sharded run must then be bit for bit a
single-process `AdamWFP32Copy` run on the averaged gradient, on every rank.  Then the consolidated state dict must equal
that run's, and loading it into a sub-group of W / 2 ranks must resume identically."""
import copy
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from atlas_b200.optim import AdamWFP32Copy  # noqa: E402
from atlas_b200.sharded import OSS, ShardedDataParallel  # noqa: E402

SHAPES = [(97, 33), (5,), (1000,), (64, 64), (1,), (300, 7), (129,)]


class Bag(torch.nn.Module):
    def __init__(self, dev):
        super().__init__()
        g = torch.Generator().manual_seed(11)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter((torch.randn(*s, generator=g) * 0.1).to(torch.bfloat16).to(dev))
                                          for s in SHAPES])

    def forward(self, cs):
        return sum((p * c).sum() for p, c in zip(self.ps, cs))


def groups(params):
    params = list(params)
    return [{"params": params[0::2], "lr": 3e-3, "weight_decay": 0.1}, {"params": params[1::2], "lr": 1e-3, "weight_decay": 0.0}]


def local_grads(step, rank, dev):
    g = torch.Generator().manual_seed(1000 * step + rank)
    return [(torch.randint(-63, 64, s, generator=g).float() * 2.0 ** -12).to(torch.bfloat16).to(dev) for s in SHAPES]


def bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def run_reference(ref, ref_opt, world, steps, dev):
    for step in steps:
        avg = [sum(c.float() for c in cs) / world for cs in zip(*(local_grads(step, r, dev) for r in range(world)))]
        ref.zero_grad(set_to_none=True)
        ref([a.to(torch.bfloat16) for a in avg]).backward()
        ref_opt.step(scale=2.0)


def main():
    backend = sys.argv[1]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group(backend)

    ref = Bag(dev)
    ref_opt = AdamWFP32Copy(groups(ref.parameters()), betas=(0.9, 0.98), eps=1e-6)
    mod = Bag(dev)
    opt = OSS(groups(mod.parameters()), optim=AdamWFP32Copy, betas=(0.9, 0.98), eps=1e-6, force_broadcast_object=True)
    assert opt.world_size == world and opt._shard_size * world == opt._padded
    sdp = ShardedDataParallel(mod, opt, auto_refresh_trainable=False)
    run_reference(ref, ref_opt, world, (1, 2, 3), dev)
    for step in (1, 2, 3):
        sdp.zero_grad(set_to_none=True)
        sdp(local_grads(step, rank, dev)).backward()
        total = opt.clip_grad_norm(1e9)                 # coefficient 1: the norm is collective, the gradient unchanged
        assert torch.isfinite(total)
        opt.step(scale=2.0)
    for i, (a, b) in enumerate(zip(ref.parameters(), mod.parameters())):
        assert torch.equal(bits(a), bits(b)), f"rank {rank}: parameter {i} differs"

    opt.consolidate_state_dict(recipient_rank=0)
    want = ref_opt.state_dict()
    if rank == 0:
        got = opt.state_dict()
        assert sorted(got["state"]) == sorted(want["state"])
        for i, st in want["state"].items():
            assert int(got["state"][i]["step"]) == int(st["step"]) == 3
            for key in ("float32copy", "exp_avg", "exp_avg_sq"):
                assert torch.equal(bits(got["state"][i][key]), bits(st[key])), f"state {i} {key} differs"
        shared = [got]
    else:
        assert opt._all_states == []
        shared = [None]
    dist.broadcast_object_list(shared, src=0)
    full = shared[0]

    # resume at another world size: the first half of the ranks
    half = max(world // 2, 1)
    sub = dist.new_group(list(range(half)))
    if rank < half:
        mod2 = copy.deepcopy(mod)
        opt2 = OSS(groups(mod2.parameters()), group=sub, betas=(0.9, 0.98), eps=1e-6)
        assert opt2.world_size == half
        opt2.load_state_dict(full)
        sdp2 = ShardedDataParallel(mod2, opt2, process_group=sub)
        # the sub-group's local gradients average to the full world's step-4 average
        avg = [sum(c.float() for c in cs) / world for cs in zip(*(local_grads(4, r, dev) for r in range(world)))]
        sdp2([a.to(torch.bfloat16) for a in avg]).backward()
        opt2.step(scale=2.0)
        run_reference(ref, ref_opt, world, (4,), dev)
        for i, (a, b) in enumerate(zip(ref.parameters(), mod2.parameters())):
            assert torch.equal(bits(a), bits(b)), f"rank {rank}: resumed parameter {i} differs"
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank}: ok")


if __name__ == "__main__":
    main()
