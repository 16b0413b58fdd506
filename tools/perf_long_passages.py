"""FiD-base reader on long passages: text_maxlength 512 (the resident attention kernel) against 1024 and 2048 (the K / V
streaming kernel, ops.attention_long), with n_context chosen so that every setting encodes the same number of tokens
per example.  For each setting: the no-grad forward time, the training-step time (forward + backward), and the encoder
self-attention forward kernel on its own (CUDA events over repeated launches on the encoder's shapes) with its FLOPs
computed from the shapes and their share of the H100 SXM's dense bf16 peak (989 TFLOP/s at 700 W).  Every passage is
fully live (no padded 64-key blocks), so the attention does its dense work.  Random bf16 weights.
    python tools/perf_long_passages.py [--tokens 20480] [--batch 1] [--steps 5]"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from atlas_b200 import ops  # noqa: E402
from atlas_b200.fid import FiD, T5ConfigLite, bias_by_delta  # noqa: E402

BF16_DENSE_PEAK = 989e12


def timed(fn, n, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def device_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=20480, help="encoder tokens per example (n_context x text_maxlength)")
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--target", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_long_passages: needs a CUDA device")
    dev = torch.device("cuda:0")
    print("device:", device_line(), flush=True)
    torch.manual_seed(0)
    cfg = T5ConfigLite()
    model = FiD(cfg).to(torch.bfloat16).to(dev)
    H, B, T = cfg.num_heads, args.batch, args.target
    results = []
    for L in (512, 1024, 2048):
        n_ctx = args.tokens // L
        model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
        ids = torch.randint(2, cfg.vocab_size, (B, n_ctx * L), device=dev)
        mask = torch.ones(B, n_ctx * L, dtype=torch.bool, device=dev)
        labels = torch.randint(2, cfg.vocab_size, (B, T), device=dev)

        model.eval()

        def fwd():
            with torch.no_grad():
                model(input_ids=ids, attention_mask=mask, labels=labels)

        t_fwd = timed(fwd, args.steps)
        model.train()

        def step():
            model.zero_grad(set_to_none=True)
            model(input_ids=ids, attention_mask=mask, labels=labels)[0].backward()

        t_step = timed(step, args.steps)
        model.zero_grad(set_to_none=True)

        # the encoder self-attention forward as _encode_rows calls it: S = B * n_ctx segments of L tokens
        S = B * n_ctx
        qkv = (torch.randn(S * L, 3 * H * 64, device=dev) * 0.5).to(torch.bfloat16)
        out = torch.empty(S * L, H * 64, dtype=torch.bfloat16, device=dev)
        add_mask = torch.zeros(S, L, device=dev)
        W = model.encoder.block[0].layer[0].SelfAttention.relative_attention_bias.weight
        bias = bias_by_delta(W, L, L, True, cfg.relative_attention_num_buckets)
        live = ops.key_block_live(add_mask)
        fn = ops.encoder_attention(L)

        def attn():
            fn(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=add_mask, bias_delta=bias, scale=1.0, out=out,
               block_live=live)

        t_attn = timed(attn, 20, warm=3)
        flops = 4.0 * S * H * L * L * 64
        r = dict(text_maxlength=L, n_context=n_ctx, batch=B, kernel="attention" if fn is ops.attention else "attention_long",
                 forward_ms=round(t_fwd, 2), train_step_ms=round(t_step, 2), attention_fwd_ms=round(t_attn, 3),
                 attention_fwd_tflops=round(flops / (t_attn * 1e-3) / 1e12, 1),
                 attention_fwd_share_of_bf16_peak=round(flops / (t_attn * 1e-3) / BF16_DENSE_PEAK, 3),
                 attention_fwd_share_of_forward=round(cfg.num_layers * t_attn / t_fwd, 3))
        results.append(r)
        print(json.dumps(r), flush=True)
    print("device:", device_line(), flush=True)
    assert all(math.isfinite(r["forward_ms"]) for r in results)


if __name__ == "__main__":
    main()
