"""Cost of the padded decoder cross-attention key range (fid._cross_split) on FiD-base, bf16, one query.

Training step, 32 target tokens:
  * 30 x 200 with --dropout 0.1 (6000 keys: no split that is a multiple of 32, padded to 6144) against 32 x 200
    (6400 keys, a regular 320-key split), the comparison of two shapes;
  * 30 x 200 without dropout on its regular 375-key split against the same step padded on purpose: the pad's cost alone.
No-grad forward at 128 target tokens (the split-KV kernel; at 64 or fewer the stream kernel takes any key range unpadded):
  * 30 x 200 on its regular split against the same forward padded on purpose.
The configurations alternate within every round in one process; each comparison is printed as the median and range of
its per-round ratio.
    python tools/perf_cross_pad.py [--rounds 7] [--steps 10]"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from atlas_b200 import fid  # noqa: E402
from atlas_b200.fid import FiD, T5ConfigLite  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=10)
args = ap.parse_args()

dev = torch.device("cuda:0")
name = torch.cuda.get_device_name(dev)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print(f"{name}, power limit {power}", flush=True)

torch.manual_seed(0)
model = FiD(T5ConfigLite(dropout_rate=0.1)).to(torch.bfloat16).to(dev)
L, B = 200, 1
regular_split = fid._cross_split


def inputs(n_ctx, T):
    g = torch.Generator().manual_seed(n_ctx)
    lens = torch.randint(L * 3 // 5, L + 1, (B, n_ctx), generator=g)         # passages padded to text_maxlength
    mask = (torch.arange(L)[None, None, :] < lens[..., None]).reshape(B, n_ctx * L)
    ids = torch.randint(2, 32000, (B, n_ctx * L), generator=g) * mask
    labels = torch.randint(2, 32000, (B, T), generator=g)
    return ids.to(dev), mask.to(dev), labels.to(dev)


def run(n_ctx, train, dropout, pad, T):
    ids, mask, labels = inputs(n_ctx, T)
    fid._cross_split = (lambda Lk, dropout=False: regular_split(Lk, dropout, force_pad=True)) if pad else regular_split
    model.config.dropout_rate = dropout
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    model.train(train)
    model._graphs.clear()          # the captured forward graphs are keyed by shape, not by the key split

    def once():
        if train:
            model.zero_grad(set_to_none=True)
            model(input_ids=ids, attention_mask=mask, labels=labels)[0].backward()
        else:
            with torch.no_grad():
                model(input_ids=ids, attention_mask=mask, labels=labels)

    for _ in range(2):
        once()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        once()
    e1.record()
    torch.cuda.synchronize()
    fid._cross_split = regular_split
    return e0.elapsed_time(e1) / args.steps


# (label, n_context, train, dropout, padded on purpose, target tokens)
CONFIGS = [("train 30x200 dropout 0.1 (padded)", 30, True, 0.1, False, 32),
           ("train 32x200 dropout 0.1 (regular)", 32, True, 0.1, False, 32),
           ("train 30x200 dropout 0 (regular)", 30, True, 0.0, False, 32),
           ("train 30x200 dropout 0 (padded on purpose)", 30, True, 0.0, True, 32),
           ("no-grad fwd 30x200 T128 (regular)", 30, False, 0.0, False, 128),
           ("no-grad fwd 30x200 T128 (padded on purpose)", 30, False, 0.0, True, 128)]
times = {c[0]: [] for c in CONFIGS}
for _ in range(args.rounds):
    for label, *cfg in CONFIGS:
        times[label].append(run(*cfg))
for label, n_ctx, train, dropout, pad, T in CONFIGS:
    split, Lk_pad = fid._cross_split(n_ctx * L, dropout=dropout > 0, force_pad=pad)
    t = times[label]
    print(f"{label:44s} keys {n_ctx * L} -> {Lk_pad} (split {split}): median {statistics.median(t):8.2f} ms "
          f"(min {min(t):.2f}, max {max(t):.2f}, {len(t)} rounds of {args.steps})")
for num, den, note in ((0, 1, "padded keys 6144 / 6400 = 0.960, real keys 6000 / 6400 = 0.938"),
                       (3, 2, "padded keys 6144 / 6000 = 1.024"), (5, 4, "padded keys 6144 / 6000 = 1.024")):
    r = [a / b for a, b in zip(times[CONFIGS[num][0]], times[CONFIGS[den][0]])]
    print(f"{CONFIGS[num][0]} / {CONFIGS[den][0]}: per-round ratio median {statistics.median(r):.3f} "
          f"(min {min(r):.3f}, max {max(r):.3f}); {note}")
