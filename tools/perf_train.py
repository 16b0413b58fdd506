"""Training-step diagnostics on one GPU: (1) per-parameter relative L2 error of the kernels' gradients against the CPU
gradient oracle on the tiny models, (2) FiD-base forward + backward time at n_context 40 x 384 tokens with the share of
the GEMM / attention-backward kernels, (3) single-op timings of the backward kernels at FiD-base shapes.
    python tools/perf_train.py [diag] [step] [ops]"""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from atlas_b200 import grad_ops, ops  # noqa: E402
from atlas_b200._lib import lib  # noqa: E402
from atlas_b200.fid import FiD, T5ConfigLite  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(0)
what = set(sys.argv[1:]) or {"diag", "step", "ops"}


def timed(fn, n=5, warm=2):
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


if "diag" in what:
    import grad_oracle
    import model_synth

    kw = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    ids, mask, labels = model_synth.fid_inputs()
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        model = FiD(T5ConfigLite(**kw))
        sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
        model.load_state_dict(sd)
        model = model.to(dt).to(dev).train()
        model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
        out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))
        out[0].backward()
        _, ref = grad_oracle.fid_grads(sd, model_synth.T5_CFG, ids, mask, labels, 3, model._shift_right)
        errs = sorted(((float((p.grad.float().cpu() - ref[n]).norm() / ref[n].norm()), n)
                       for n, p in model.named_parameters()), reverse=True)
        print(f"FiD tiny {dt}: loss {float(out[0]):.4f}; worst relative L2 gradient errors vs the fp32 oracle:")
        for e, n in errs[:6]:
            print(f"    {e:.4f}  {n}")
        print(f"    median {errs[len(errs) // 2][0]:.4f}", flush=True)

if "step" in what:
    L_ = lib()
    model = FiD(T5ConfigLite()).to(torch.bfloat16).to(dev).train()
    n_ctx, L, T = 40, 384, 32
    for B in (1, 2):
        model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
        ids = torch.randint(2, 32000, (B, n_ctx * L), device=dev)
        mask = torch.ones(B, n_ctx * L, dtype=torch.bool, device=dev)
        labels = torch.randint(2, 32000, (B, T), device=dev)

        def step():
            model.zero_grad(set_to_none=True)
            out = model(input_ids=ids, attention_mask=mask, labels=labels)
            out[0].backward()

        def fwd_only():
            with torch.no_grad():
                model(input_ids=ids, attention_mask=mask, labels=labels)

        def fwd_grad():
            model(input_ids=ids, attention_mask=mask, labels=labels)

        t_step = timed(step, n=3, warm=2)
        t_fg = timed(fwd_grad, n=3, warm=1)
        t_f = timed(fwd_only, n=3, warm=2)
        torch.cuda.synchronize()
        mem = torch.cuda.max_memory_allocated() / 2 ** 30
        shares = {}
        for kind, name in ((2, "gemm"), (3, "attention fwd"), (4, "attention bwd")):
            L_.atlas_b200_profile_enable(kind)
            step()
            work = L_.atlas_b200_profile_work()
            ms, n = ctypes.c_double(0), ctypes.c_int32(0)
            L_.atlas_b200_profile_collect(ctypes.byref(ms), ctypes.byref(n))
            L_.atlas_b200_profile_enable(0)
            shares[name] = (ms.value, n.value, work / max(ms.value, 1e-9) / 1e9)
        tok = B * n_ctx * L
        print(f"FiD-base train B={B}: fwd+bwd {t_step:.1f} ms ({tok / t_step * 1e3:.0f} reader tokens/s), with-grad fwd "
              f"{t_fg:.1f} ms, no-grad fwd (graph) {t_f:.1f} ms, peak mem {mem:.1f} GiB")
        for k, (ms, n, tf) in shares.items():
            print(f"    {k:14s} {ms:8.2f} ms in {n:4d} launches = {tf:7.1f} TFLOP/s  ({100 * ms / t_step:.0f} % of the step)")
        sys.stdout.flush()

if "launchlist" in what:
    # one FiD-base training step (1 query) between cudaProfilerStart / Stop, for `ncu --profile-from-start off`
    model = FiD(T5ConfigLite()).to(torch.bfloat16).to(dev).train()
    n_ctx, L, T, B = 40, 384, 32, 1
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    ids = torch.randint(2, 32000, (B, n_ctx * L), device=dev)
    mask = torch.ones(B, n_ctx * L, dtype=torch.bool, device=dev)
    labels = torch.randint(2, 32000, (B, T), device=dev)
    # the backward kernels are launched from autograd's worker thread, outside any thread-scoped NVTX range of this
    # thread: bracket the step with cudaProfilerStart / Stop instead (ncu --profile-from-start off)
    for i in range(3):
        if i == 2:
            torch.cuda.synchronize()
            torch.cuda.profiler.start()
        model.zero_grad(set_to_none=True)
        model(input_ids=ids, attention_mask=mask, labels=labels)[0].backward()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()

if "ops" in what:
    M, d, dff, H, S, L = 30720, 768, 2048, 12, 80, 384
    x = torch.randn(M, d, device=dev).bfloat16() * 0.1
    dy = torch.randn(M, 3 * d, device=dev).bfloat16() * 0.1
    w = torch.randn(3 * d, d, device=dev).bfloat16() * 0.03
    t = timed(lambda: ops.transpose(dy))
    print(f"transpose [{M}, {3 * d}]: {t:.3f} ms = {2 * dy.numel() * 2 / t / 1e6:.0f} GB/s")
    t = timed(lambda: ops.linear_dgrad(dy, w))
    print(f"dgrad M={M} N={3 * d} K={d}: {t:.3f} ms = {2 * M * 3 * d * d / t / 1e9:.0f} TFLOP/s")
    t = timed(lambda: ops.linear_wgrad(dy, x))
    print(f"wgrad M={M} N={3 * d} K={d} (MN-major GEMM): {t:.3f} ms = {2 * M * 3 * d * d / t / 1e9:.0f} TFLOP/s")
    dyT, xT = ops.transpose(dy), ops.transpose(x)
    t = timed(lambda: ops.linear(dyT, xT))
    print(f"wgrad GEMM alone [{3 * d} x {M}] . [{M} x {d}]: {t:.3f} ms = {2 * M * 3 * d * d / t / 1e9:.0f} TFLOP/s")
    wn = torch.ones(d, device=dev).bfloat16()
    t = timed(lambda: ops.layernorm_bwd(x, x, wn, 1e-6, 1))
    print(f"rmsnorm bwd [{M}, {d}]: {t:.3f} ms = {3 * x.numel() * 2 / t / 1e6:.0f} GB/s")
    u = torch.randn(M, 2 * dff, device=dev).bfloat16()
    dg = torch.randn(M, dff, device=dev).bfloat16()
    t = timed(lambda: ops.gated_gelu(u, dg))
    print(f"gated-gelu bwd [{M}, {2 * dff}]: {t:.3f} ms = {(2 * u.numel() + dg.numel()) * 2 / t / 1e6:.0f} GB/s")
    qkv = torch.randn(S * L, 3 * H * 64, device=dev).bfloat16() * 0.2
    bias = torch.randn(H, 2 * L - 1, device=dev)
    am = torch.zeros(S, L, device=dev)
    out, lse = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=am, bias_delta=bias, return_lse=True)
    do = torch.randn_like(out)
    dqkv = torch.empty_like(qkv)
    for nb in (True, False):
        t = timed(lambda: ops.attention_bwd(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, out, do, dqkv, 0, dqkv, H * 64, dqkv,
                                            2 * H * 64, S, H, L, L, add_mask=am, bias_delta=bias, need_dbias=nb, lse=lse))
        print(f"attention bwd S={S} H={H} L={L} dbias={nb}: {t:.3f} ms = {14 * S * H * L * L * 64 / t / 1e9:.0f} TFLOP/s "
              f"(executed, 7 tile GEMMs), {10 * S * H * L * L * 64 / t / 1e9:.0f} (5-GEMM minimum)")
