"""T5 v1.0 (ReLU feed-forward, tied LM head) against T5 v1.1 (gated GELU) readers at the benchmark's reader shape: FiD-base,
n_context 40 x text_maxlength 384, 32 target tokens, bf16, random-init weights and synthetic tokens.
  * the no-grad forward (batch 8, the bench's forward step) of a t5-base-shaped v1.0 reader next to the v1.1 base reader;
  * one training step (forward + backward, batch 2, the bench's train leg) of each;
  * the feed-forward input GEMM alone at the forward's encoder rows: wi with the ReLU epilogue (768 -> 3072) next to the
    interleaved wi_0 | wi_1 with the gated-GELU epilogue (768 -> 2 x 2048), achieved TFLOP/s.
The two feed-forward blocks have equal FLOPs (768 x 6144 multiply-adds per token), so the readers should take about the same
time.  CUDA-event timing; the A / B pairs alternate within one process.  Prints the GPU, its power limit and SM clocks.
    python tools/perf_t5v10.py"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from atlas_b200 import ops  # noqa: E402
from atlas_b200.fid import FiD, T5ConfigLite  # noqa: E402

N_CTX, L, T, B_FWD, B_TRAIN = 40, 384, 32, 8, 2


def timed(fn, n, warm=1):
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


def alternate(fns, n, rounds):
    """{name: [ms per round]}: the candidates timed in turn, `rounds` times (shared-host noise hits both alike)."""
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            out[k].append(timed(fn, n, warm=0))
    return out


def med(xs):
    return sorted(xs)[len(xs) // 2]


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e!r})"


def main():
    assert torch.cuda.is_available(), "tools/perf_t5v10.py measures on a GPU"
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    print(f"GPU: {gpu_info()}  [name, power limit, max SM clock, SM clock at start]", flush=True)
    readers = {
        "v1.1": FiD(T5ConfigLite()),
        "v1.0": FiD(T5ConfigLite(feed_forward_proj="relu", d_ff=3072, tie_word_embeddings=True)),
    }
    for m in readers.values():
        m.to(torch.bfloat16).to(dev)
        with torch.no_grad():
            m.shared.weight.mul_(0.05)           # keep the tied head's logits O(1) on random weights
    g = torch.Generator().manual_seed(7)

    # ---- no-grad forward, batch 8 ----
    ids = torch.randint(2, 32000, (B_FWD, N_CTX * L), generator=g).to(dev)
    mask = torch.ones(B_FWD, N_CTX * L, dtype=torch.bool, device=dev)
    dec = torch.randint(2, 32000, (B_FWD, T), generator=g).to(dev)

    def fwd(m):
        def run():
            with torch.no_grad():
                m(input_ids=ids, attention_mask=mask, decoder_input_ids=dec)
        return run

    for m in readers.values():
        m.eval()
        m.encoder.config.n_context, m.encoder.config.bsz = N_CTX, B_FWD
        timed(fwd(m), 2)                          # graph capture + warm-up
    res = alternate({k: fwd(m) for k, m in readers.items()}, n=5, rounds=5)
    f11, f10 = med(res["v1.1"]), med(res["v1.0"])
    print(f"forward (no grad, CUDA graph) B={B_FWD} x {N_CTX} x {L}: v1.1 {f11:.2f} ms, v1.0 {f10:.2f} ms, "
          f"v1.0 / v1.1 = {f10 / f11:.3f}  (per-round ms v1.1 {[round(x, 2) for x in res['v1.1']]}, "
          f"v1.0 {[round(x, 2) for x in res['v1.0']]})", flush=True)
    del ids, mask, dec
    for m in readers.values():
        m._graphs.clear()
    torch.cuda.empty_cache()

    # ---- training step, batch 2 ----
    ids = torch.randint(2, 32000, (B_TRAIN, N_CTX * L), generator=g).to(dev)
    mask = torch.ones(B_TRAIN, N_CTX * L, dtype=torch.bool, device=dev)
    labels = torch.randint(2, 32000, (B_TRAIN, T), generator=g).to(dev)

    def step(m):
        def run():
            m.zero_grad(set_to_none=True)
            m(input_ids=ids, attention_mask=mask, labels=labels)[0].backward()
        return run

    for m in readers.values():
        m.train()
        m.encoder.config.n_context, m.encoder.config.bsz = N_CTX, B_TRAIN
        timed(step(m), 1)
    res = alternate({k: step(m) for k, m in readers.items()}, n=2, rounds=5)
    s11, s10 = med(res["v1.1"]), med(res["v1.0"])
    print(f"train step (fwd + bwd) B={B_TRAIN} x {N_CTX} x {L}: v1.1 {s11:.1f} ms, v1.0 {s10:.1f} ms, "
          f"v1.0 / v1.1 = {s10 / s11:.3f}  (per-round ms v1.1 {[round(x, 1) for x in res['v1.1']]}, "
          f"v1.0 {[round(x, 1) for x in res['v1.0']]})", flush=True)
    for m in readers.values():
        m.zero_grad(set_to_none=True)
    del readers, ids, mask, labels
    torch.cuda.empty_cache()

    # ---- the feed-forward input GEMM at the forward's encoder rows ----
    M, d = B_FWD * N_CTX * L, 768
    x = (torch.randn(M, d, generator=g) * 0.5).bfloat16().to(dev)
    w_relu = (torch.randn(3072, d, generator=g) * 0.03).bfloat16().to(dev)
    w_gated = (torch.randn(4096, d, generator=g) * 0.03).bfloat16().to(dev)
    out_relu = torch.empty(M, 3072, dtype=torch.bfloat16, device=dev)
    out_gated = torch.empty(M, 2048, dtype=torch.bfloat16, device=dev)
    gemms = {"EPI_RELU  wi 768->3072": (lambda: ops.linear(x, w_relu, epilogue=ops.EPI_RELU, out=out_relu), 3072),
             "EPI_GATED wi_0|wi_1 768->2x2048": (lambda: ops.linear(x, w_gated, epilogue=ops.EPI_GATED, out=out_gated), 4096)}
    for fn, _ in gemms.values():
        timed(fn, 3)
    res = alternate({k: v[0] for k, v in gemms.items()}, n=20, rounds=5)
    for k, (_, N) in gemms.items():
        ms = med(res[k])
        print(f"GEMM {k}, M={M}: {ms:.3f} ms = {2 * M * N * d / ms / 1e9:.0f} TFLOP/s", flush=True)
    print(f"GPU after: {gpu_info()}", flush=True)


if __name__ == "__main__":
    main()
