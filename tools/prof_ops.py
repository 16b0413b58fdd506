"""Single-op drivers for ncu captures: python tools/prof_ops.py attention|gemm|gemm4|gemm_small|contriever|fid [reps]."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from atlas_b200 import ops
dev = torch.device("cuda:0")
torch.manual_seed(0)
what = sys.argv[1] if len(sys.argv) > 1 else "attention"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3

def timed(fn, n=10, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

def graph_timed(fn, n=20, reps=10):
    """Device time of one fn() call: n calls captured into a CUDA graph, replayed `reps` times (a launch that takes a few
    microseconds on the GPU takes longer than that to issue from Python, so timing eager calls measures the host)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3): fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n): fn()
    return timed(g.replay, reps) / n

if what == "attention":
    S, H, L = 160, 12, 384      # FiD-base encoder, 4 queries x 40 passages
    qkv = torch.randn(S * L, 3 * H * 64, device=dev).bfloat16() * 0.2
    bias = torch.randn(H, 2 * L - 1, device=dev)
    am = torch.zeros(S, L, device=dev)
    fn = lambda: ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=am, bias_delta=bias)
    ms = timed(fn, reps)
    print(f"attention S={S} H={H} L={L}: {ms:.3f} ms = {4 * S * H * L * L * 64 / ms / 1e9:.0f} TFLOP/s")
elif what == "gemm":
    M, N, K = 61440, 4096, 768  # FiD-base wi_0|wi_1 gated projection, 4 queries
    x = torch.randn(M, K, device=dev).bfloat16() * 0.1
    w = torch.randn(N, K, device=dev).bfloat16() * 0.03
    fn = lambda: ops.linear(x, w, epilogue=ops.EPI_GATED)
    ms = timed(fn, reps)
    print(f"gemm M={M} N={N} K={K} gated: {ms:.3f} ms = {2 * M * N * K / ms / 1e9:.0f} TFLOP/s")
elif what == "gemm4":
    # the four linear-layer shapes of a FiD-base encoder block at 4 queries x 40 passages x 384 tokens with their fused
    # epilogues, then the wo projection of the padding-compacted encoder (8 queries x 40 passages, U[148, 276] real tokens
    # padded to 384, as in `packed`): only the first `count` rows (device-side row count), residual + out_ss; each next to
    # cuBLAS (torch.matmul of the same computed rows, plain epilogue)
    S, L = 320, 384
    lens = torch.randint(148, 277, (S,), device=dev)
    mask = (torch.arange(L, device=dev)[None, :] >= lens[:, None]).float() * -10000.0
    count = ops.segment_tile_scan(ops.key_block_live(mask))[3]
    rows = int(count)
    for name, M, N, K, epi in (("qkv", 61440, 2304, 768, None), ("o-proj+res", 61440, 768, 768, "res"),
                               ("wi gated", 61440, 4096, 768, "gated"), ("wo+res", 61440, 768, 2048, "res"),
                               ("wo+res m_dev", S * L, 768, 2048, "res_rows")):
        x = torch.randn(M, K, device=dev).bfloat16() * 0.1
        w = torch.randn(N, K, device=dev).bfloat16() * 0.03
        r = torch.randn(M, N, device=dev).bfloat16() if epi in ("res", "res_rows") else None
        ss = torch.zeros(M, device=dev)
        if epi == "gated":
            fn = lambda: ops.linear(x, w, epilogue=ops.EPI_GATED)
        elif epi == "res":
            fn = lambda: ops.linear(x, w, None, residual=r, epilogue=ops.EPI_RESIDUAL)
        elif epi == "res_rows":
            fn = lambda: ops.linear(x, w, None, residual=r, epilogue=ops.EPI_RESIDUAL, out_ss=ss, rows=count)
        else:
            fn = lambda: ops.linear(x, w)
        ms = timed(fn, reps)
        m = rows if epi == "res_rows" else M
        xm, wt = x[:m], w.t().contiguous()
        ms_ref = timed(lambda: torch.matmul(xm, wt), reps)
        fl = 2 * m * N * K
        print(f"gemm {name:12s} M={m} N={N} K={K}: {ms:.3f} ms = {fl / ms / 1e9:.0f} TFLOP/s   cuBLAS plain: {ms_ref:.3f} ms = "
              f"{fl / ms_ref / 1e9:.0f} TFLOP/s")
elif what == "gemm_small":
    # both sides of the schedule selection (ping-pong from 2 x #SMs 128 x 128 tiles): the decoder's cross-attention K|V
    # projection over the packed encoder rows (device-side row count, ping-pong), then 256-row decoder-sized
    # launches (8 queries x 32 target tokens) with each epilogue: cooperative, except the LM head (2 x 251 tiles of
    # 128 x 128: ping-pong); each next to cuBLAS plain on the same rows, all timed inside CUDA graphs
    S, L = 320, 384
    lens = torch.randint(148, 277, (S,), device=dev)
    mask = (torch.arange(L, device=dev)[None, :] >= lens[:, None]).float() * -10000.0
    count = ops.segment_tile_scan(ops.key_block_live(mask))[3]
    rows = int(count)
    shapes = [("cross K|V", S * L, 1536, 768, "rows")]
    shapes += [(f"dec {nm}", 256, N, K, epi) for nm, N, K, epi in
               (("qkv", 2304, 768, None), ("o+res", 768, 768, "res"), ("wi gated", 4096, 768, "gated"),
                ("wo+res", 768, 2048, "res"), ("bias", 768, 768, "bias"), ("gelu", 3072, 768, "gelu"),
                ("lm_head", 32128, 768, None))]
    for name, M, N, K, epi in shapes:
        x = torch.randn(M, K, device=dev).bfloat16() * 0.1
        w = torch.randn(N, K, device=dev).bfloat16() * 0.03
        b = torch.randn(N, device=dev).bfloat16() * 0.1
        r = torch.randn(M, N, device=dev).bfloat16() if epi == "res" else None
        if epi == "rows":
            fn = lambda: ops.linear(x, w, rows=count)
        elif epi == "gated":
            fn = lambda: ops.linear(x, w, epilogue=ops.EPI_GATED)
        elif epi == "res":
            fn = lambda: ops.linear(x, w, b, residual=r, epilogue=ops.EPI_RESIDUAL)
        elif epi == "bias":
            fn = lambda: ops.linear(x, w, b, epilogue=ops.EPI_BIAS)
        elif epi == "gelu":
            fn = lambda: ops.linear(x, w, b, epilogue=ops.EPI_GELU)
        else:
            fn = lambda: ops.linear(x, w)
        ms = graph_timed(fn, reps=reps)
        m = rows if epi == "rows" else M
        xm, wt = x[:m], w.t().contiguous()
        ms_ref = graph_timed(lambda: torch.matmul(xm, wt), reps=reps)
        fl = 2 * m * N * K
        print(f"gemm {name:12s} M={m} N={N} K={K}: {ms * 1e3:.1f} us = {fl / ms / 1e9:.0f} TFLOP/s   cuBLAS plain: "
              f"{ms_ref * 1e3:.1f} us = {fl / ms_ref / 1e9:.0f} TFLOP/s")
elif what == "gemm_sched":
    # every encoder-sized GEMM shape of the bench step and of the index refresh, timed on the schedule the rule picks and on
    # both encoder-sized schedules forced (ATLAS_B200_GEMM_SCHEDULE, read once per process: one child process each)
    import subprocess
    for force in ("", "pingpong", "wide"):
        env = dict(os.environ, ATLAS_B200_GEMM_SCHEDULE=force)
        print(f"-- schedule: {force or 'selected by the rule'}", flush=True)
        subprocess.run([sys.executable, os.path.abspath(__file__), "gemm_sched1", str(reps)], env=env, check=True)
elif what == "gemm_sched1":
    # one process of gemm_sched: each shape at its bench size (8 queries x 40 passages x 384 tokens = 122,880 rows; the
    # packed encoder's launches run over the first `count` of them, a device-side row count) with its fused epilogue, the
    # schedule atlas_b200_linear_schedule reports for it, and cuBLAS plain on the same rows; then the mainloop alone
    # (K = 4096, plain epilogue), all timed inside CUDA graphs
    from atlas_b200._lib import lib
    names = {0: "coop128", 1: "coop256", 2: "pingpong", 3: "wide"}
    S, L = 320, 384
    lens = torch.randint(148, 277, (S,), device=dev)
    mask = (torch.arange(L, device=dev)[None, :] >= lens[:, None]).float() * -10000.0
    count = ops.segment_tile_scan(ops.key_block_live(mask))[3]
    rows = int(count)
    for name, M, N, K, epi in (("qkv", S * L, 2304, 768, "rows"), ("o-proj+res", S * L, 768, 768, "res"),
                               ("wi gated", S * L, 4096, 768, "gated"), ("wo+res+ss", S * L, 768, 2048, "res_ss"),
                               ("cross K|V", S * L, 1536, 768, "rows"), ("qkv+bias", S * L, 2304, 768, "bias"),
                               ("wi+gelu", S * L, 3072, 768, "gelu"), ("wi+relu", S * L, 3072, 768, "relu"),
                               ("mainloop", 61440, 2304, 4096, None)):
        x = torch.randn(M, K, device=dev).bfloat16() * 0.1
        w = torch.randn(N, K, device=dev).bfloat16() * 0.03
        b = torch.randn(N, device=dev).bfloat16() * 0.1
        r = torch.randn(M, N, device=dev).bfloat16() if epi in ("res", "res_ss") else None
        ss = torch.zeros(M, device=dev)
        e = {"gated": ops.EPI_GATED, "res": ops.EPI_RESIDUAL, "res_ss": ops.EPI_RESIDUAL, "bias": ops.EPI_BIAS,
             "gelu": ops.EPI_GELU, "relu": ops.EPI_RELU}.get(epi, ops.EPI_NONE)
        if epi is None:
            fn = lambda: ops.linear(x, w)
        else:
            fn = lambda: ops.linear(x, w, b if epi in ("bias", "gelu", "relu") else None, residual=r, epilogue=e,
                                    out_ss=ss if epi == "res_ss" else None, rows=count)
        m = M if epi is None else rows
        sched = names[lib().atlas_b200_linear_schedule(M, N, K, e)]
        ms = graph_timed(fn, n=5, reps=reps)
        xm, wt = x[:m], w.t().contiguous()
        ms_ref = graph_timed(lambda: torch.matmul(xm, wt), n=5, reps=reps)
        fl = 2 * m * N * K
        print(f"gemm {name:11s} M={m} N={N} K={K} {sched:8s}: {ms * 1e3:.1f} us = {fl / ms / 1e9:.0f} TFLOP/s   "
              f"cuBLAS plain: {ms_ref * 1e3:.1f} us = {fl / ms_ref / 1e9:.0f} TFLOP/s", flush=True)
elif what == "mips":
    # one 256-query top-40 search over a 4 Mi x 768 fp16 bank (BASELINE configs[1]): for `ncu --metrics gpu__time_duration.sum`
    n, nq, k = 4 * 1024 * 1024, 256, 40
    bank = torch.empty((n, 768), dtype=torch.float16, device=dev)
    for a in range(0, n, 1 << 19):
        bank[a:a + (1 << 19)] = (torch.randn((1 << 19, 768), device=dev) * 0.05).half()
    q = (torch.randn(nq, 768, device=dev) * 0.05).half()
    fn = lambda: ops.mips_topk(bank, q, k)
    ms = timed(fn, reps)
    print(f"mips n={n} nq={nq} k={k}: {ms:.3f} ms = {n * 768 * 2 / ms / 1e6:.0f} GB/s over the bank")
elif what == "packed":
    # the padding-compacted FiD-base encoder ops at the bench's length distribution (8 queries x 40 passages, U[148, 276] real
    # tokens padded to 384): packed attention vs the padded kernel with block skipping vs no skipping, and the gated
    # projection over the packed rows (device-side row count) vs all rows
    S, H, L = 320, 12, 384
    lens = torch.randint(148, 277, (S,), device=dev)
    mask = (torch.arange(L, device=dev)[None, :] >= lens[:, None]).float() * -10000.0
    live = ops.key_block_live(mask)
    keep, off, src, count = ops.segment_tile_scan(live)
    qkv = torch.randn(S * L, 3 * H * 64, device=dev).bfloat16() * 0.2
    bias = torch.randn(H, 2 * L - 1, device=dev)
    dense_fl = 4 * S * H * L * L * 64
    frac = float(keep.float().mean())
    ms_p = timed(lambda: ops.attention_packed(qkv, keep, off, S, H, L, mask, bias), reps)
    ms_s = timed(lambda: ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=mask, bias_delta=bias,
                                       block_live=live), reps)
    ms_d = timed(lambda: ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=mask, bias_delta=bias), reps)
    print(f"attention S={S} H={H} L={L}, kept tiles {frac:.3f}: packed {ms_p:.3f} ms | padded, dead key blocks skipped {ms_s:.3f} ms | "
          f"padded, every block {ms_d:.3f} ms = {dense_fl / ms_d / 1e9:.0f} TFLOP/s; packed executes "
          f"{dense_fl * float((keep.float().sum(1) ** 2).mean()) / 36 / ms_p / 1e9:.0f} TFLOP/s on kept x kept tiles")
    M, N, K = S * L, 4096, 768
    x = torch.randn(M, K, device=dev).bfloat16() * 0.1
    w = torch.randn(N, K, device=dev).bfloat16() * 0.03
    ms_r = timed(lambda: ops.linear(x, w, epilogue=ops.EPI_GATED, rows=count), reps)
    ms_a = timed(lambda: ops.linear(x, w, epilogue=ops.EPI_GATED), reps)
    rows = int(count)
    print(f"gemm gated M={M} N={N} K={K}: first {rows} rows (device-side count) {ms_r:.3f} ms = {2 * rows * N * K / ms_r / 1e9:.0f} "
          f"TFLOP/s | all rows {ms_a:.3f} ms = {2 * M * N * K / ms_a / 1e9:.0f} TFLOP/s")
elif what == "refresh":
    # one index-refresh embedder batch (bench.py refresh leg): 512 passages of U[64, 192] tokens padded to 192 through
    # Contriever-base with fp16 weight copies, pooled rows written into bank rows (Contriever.embed_into)
    from atlas_b200.retrievers import BertConfigLite, Contriever
    model = Contriever(BertConfigLite()).to(torch.bfloat16).to(dev).eval()
    nb, lmax = 512, 192
    g = torch.Generator().manual_seed(4242)
    lens = torch.randint(64, lmax + 1, (nb,), generator=g)
    lens[0] = lmax
    ids = torch.randint(1000, 30000, (nb, lmax), generator=g)
    mask = (torch.arange(lmax)[None, :] < lens[:, None]).to(torch.int64)
    ids, mask = (ids * mask).to(dev), mask.to(dev)
    rows = torch.zeros((nb, 768), dtype=torch.float16, device=dev)
    fn = lambda: model.embed_into(ids, mask, rows, dtype=torch.float16)
    ms = timed(fn, reps)
    print(f"refresh batch {nb} x {lmax} (kept tiles {float(((lens + 63) // 64).sum()) / (nb * 3):.3f}): {ms:.3f} ms = "
          f"{nb / ms * 1e3:.0f} passages/s")
elif what == "xattn":
    # FiD-base decoder cross-attention of the teacher-forced forward: 8 queries x 32 target tokens against 40 x 384 encoder keys,
    # passages of U[148, 276] real tokens padded to 384 (the bench's length distribution)
    B, H, T, n, Lp = 8, 12, 32, 40, 384
    Lk = n * Lp
    q = torch.randn(B * T, H * 64, device=dev).bfloat16() * 0.3
    kv = torch.randn(B * Lk, 2 * H * 64, device=dev).bfloat16() * 0.3
    lens = torch.randint(148, 277, (B, n), device=dev)
    valid = torch.arange(Lp, device=dev)[None, None, :] < lens[..., None]
    mask = ((~valid).reshape(B, Lk).float() * -1e9)
    live = ops.key_block_live(mask)
    fn = lambda: ops.cross_attention_split(q, 0, kv, 0, H * 64, B, H, T, Lk, add_mask=mask, scale=1.0, split=384, tile_live=live)
    ms = timed(fn, reps)
    frac = float(live.float().mean()) if live is not None else 1.0
    byt = B * Lk * 2 * H * 64 * 2
    print(f"cross-attention B={B} H={H} T={T} Lk={Lk}: {ms:.3f} ms (stream + combine); K/V {byt / 1e6:.0f} MB, live tiles {frac:.2f}: "
          f"{byt * frac / ms / 1e6:.0f} GB/s on the live bytes, {byt / ms / 1e6:.0f} GB/s dense-equivalent")
elif what == "attn_bwd":
    S, H, L = 80, 12, 384       # FiD-base encoder, 2 queries x 40 passages (the bench's training leg)
    qkv = torch.randn(S * L, 3 * H * 64, device=dev).bfloat16() * 0.2
    bias = torch.randn(H, 2 * L - 1, device=dev)
    am = torch.zeros(S, L, device=dev)
    out, lse = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=am, bias_delta=bias, return_lse=True)
    do = torch.randn_like(out)
    dqkv = torch.empty_like(qkv)
    fn = lambda: ops.attention_bwd(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, out, do, dqkv, 0, dqkv, H * 64, dqkv, 2 * H * 64,
                                   S, H, L, L, add_mask=am, bias_delta=bias, need_dbias=True, lse=lse)
    ms = timed(fn, reps)
    print(f"attention bwd S={S} H={H} L={L} (lse from the forward, dbias): {ms:.3f} ms = "
          f"{14 * S * H * L * L * 64 / ms / 1e9:.0f} TFLOP/s executed (7 tile GEMMs), {10 * S * H * L * L * 64 / ms / 1e9:.0f} useful")
elif what == "wgrad":
    M, N, K = 30720, 4096, 768  # dW of the interleaved wi_0|wi_1 projection, 2 queries
    x = torch.randn(M, K, device=dev).bfloat16() * 0.1
    dy = torch.randn(M, N, device=dev).bfloat16() * 0.1
    fn = lambda: ops.linear_wgrad(dy, x)
    ms = timed(fn, reps)
    print(f"wgrad tokens={M} N={N} K={K} (MN-major wgmma): {ms:.3f} ms = {2 * M * N * K / ms / 1e9:.0f} TFLOP/s")
