"""Step time of the padding-compacted FiD encoder (ATLAS_B200_ENC_PACKED) against the padded one, bf16, on bench.py's passage
lengths (20 query + U[128, 256] passage tokens, padded to text_maxlength):
  * FiD-base training step, n_context 40, bsz 2, 32 target tokens, dropout 0.1, at text_maxlength 384 and 512;
  * the Atlas-xl reader (T5 v1.1-xl dims) training step with gradient checkpointing at 512, bsz 1, dropout 0.1;
  * the FiD-base no-grad forward at 512, bsz 2;
  * at 384, the no-grad encoder attention alone (FiD-base heads, 80 passages): the persistent kernel against the resident
    kernel on the same packed rows (forced by asking for the log-sum-exp, which only the resident kernel writes).
Packed and padded alternate within every round in one process; each pair is printed as the medians and the median and range
of the per-round ratio.  The card's name and power limit are read in the same run.
    python tools/perf_packed_train.py [--rounds 7] [--steps 3] [--no-xl] [--json out.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from atlas_b200 import ops  # noqa: E402
from atlas_b200.fid import FiD, T5ConfigLite  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--no-xl", action="store_true")
ap.add_argument("--json", help="also write the per-round times to this file")
args = ap.parse_args()

dev = torch.device("cuda:0")
name = torch.cuda.get_device_name(dev)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print(f"{name}, power limit {power}", flush=True)

N_CTX, QUERY_TOKENS, T = 40, 20, 32


def inputs(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.clamp(QUERY_TOKENS + torch.randint(128, 257, (B, N_CTX), generator=g), max=L)
    mask = (torch.arange(L)[None, None, :] < lens[..., None]).reshape(B, N_CTX * L)
    ids = torch.randint(2, 32000, (B, N_CTX * L), generator=g) * mask
    labels = torch.randint(2, 32000, (B, T), generator=g)
    return ids.to(dev), mask.to(dev), labels.to(dev)


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def model_leg(model, B, L, train, ckpt=False):
    ids, mask, labels = inputs(B, L, L + B)

    def run(packed):
        ops._ENC_PACKED = packed
        model.encoder.config.n_context, model.encoder.config.bsz = N_CTX, B
        model.train(train)
        model.gradient_checkpointing_enable() if ckpt else model.gradient_checkpointing_disable()
        model._graphs.clear()

        def once():
            if train:
                model.zero_grad(set_to_none=True)
                model(input_ids=ids, attention_mask=mask, labels=labels)[0].backward()
            else:
                with torch.no_grad():
                    model(input_ids=ids, attention_mask=mask, labels=labels)

        try:
            return timed(once, args.steps)
        finally:
            ops._ENC_PACKED = True
            model._graphs.clear()
    return run


def attention_leg(L=384, S=80, H=12):
    g = torch.Generator().manual_seed(7)
    lens = torch.clamp(QUERY_TOKENS + torch.randint(128, 257, (S,), generator=g), max=L)
    mask = ((torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0).to(dev)
    keep, off, _, count = ops.segment_tile_scan(ops.key_block_live(mask))
    rows = int(count)
    qkv = (torch.randn(rows, 3 * H * 64, generator=g) * 0.35).to(torch.bfloat16).to(dev)
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev)
    out = torch.empty(rows, H * 64, dtype=torch.bfloat16, device=dev)

    def run(persistent):
        return timed(lambda: [ops.attention_packed(qkv, keep, off, S, H, L, mask, bias, out=out, lse=not persistent)
                              for _ in range(20)], args.steps) / 20
    return run


torch.manual_seed(0)
base = FiD(T5ConfigLite(dropout_rate=0.1)).to(torch.bfloat16).to(dev)
LEGS = [("FiD-base train step, 40 x 384, bsz 2, dropout 0.1", model_leg(base, 2, 384, True)),
        ("FiD-base train step, 40 x 512, bsz 2, dropout 0.1", model_leg(base, 2, 512, True)),
        ("FiD-base no-grad forward, 40 x 512, bsz 2", model_leg(base, 2, 512, False)),
        ("no-grad encoder attention, 80 x 384, 12 heads", attention_leg())]
if not args.no_xl:
    xl = FiD(T5ConfigLite(d_model=2048, d_ff=5120, num_layers=24, num_decoder_layers=24, num_heads=32, dropout_rate=0.1))
    xl = xl.to(torch.bfloat16).to(dev)
    LEGS.insert(2, ("Atlas-xl reader train step, checkpointing, 40 x 512, bsz 1, dropout 0.1", model_leg(xl, 1, 512, True, True)))

# (first, second) of every leg: packed / padded, or for the attention leg persistent / resident
times = {label: ([], []) for label, _ in LEGS}
for _ in range(args.rounds):
    for label, run in LEGS:
        times[label][0].append(run(True))
        times[label][1].append(run(False))

result = {"device": name, "power_limit": power, "rounds": args.rounds, "steps": args.steps, "legs": {}}
for label, _ in LEGS:
    a, b = times[label]
    r = [x / y for x, y in zip(a, b)]
    names = ("persistent", "resident") if "attention" in label else ("packed", "padded")
    print(f"{label}: {names[0]} median {statistics.median(a):.3f} ms (range {min(a):.3f}-{max(a):.3f}), {names[1]} median "
          f"{statistics.median(b):.3f} ms (range {min(b):.3f}-{max(b):.3f}); per-round ratio {names[0]} / {names[1]} median "
          f"{statistics.median(r):.3f} (range {min(r):.3f}-{max(r):.3f}), {len(r)} rounds of {args.steps}", flush=True)
    result["legs"][label] = {names[0] + "_ms": a, names[1] + "_ms": b, "ratio_median": statistics.median(r),
                             "ratio_min": min(r), "ratio_max": max(r)}
if args.json:
    with open(args.json, "w") as f:
        json.dump(result, f, indent=1)
