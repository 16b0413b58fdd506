"""GPU diagnostic for the MIPS path.  Prints detailed mismatch information."""
import os, sys, time, json
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import synth, mips_oracle
from atlas_b200 import ops

dev = torch.device("cuda:0")
print("device", torch.cuda.get_device_name(0), flush=True)


def run_case(n, nq, k, dist="grid", bseed=1, qseed=2, exhaustive=False, verbose=True):
    bank = synth.make_bank(n, seed=bseed, dist=dist)
    q = synth.make_queries(nq, seed=qseed, dist=dist)
    S = mips_oracle.scores_fp16(q, bank)
    ov, oi = mips_oracle.canonical_topk(S, k)
    b = torch.from_numpy(bank).to(dev)
    qt = torch.from_numpy(q).to(dev)
    t0 = time.time()
    s, i, st = ops.mips_topk(b, qt, k, exhaustive=exhaustive)
    torch.cuda.synchronize()
    dt = time.time() - t0
    s = s.cpu().numpy(); i = i.cpu().numpy(); st = int(st.item())
    ok_s = np.array_equal(s.view(np.uint16), ov.view(np.uint16))
    ok_i = np.array_equal(i, oi)
    print(f"case n={n} nq={nq} k={k} {dist} exh={exhaustive}: status={st} scores_equal={ok_s} ids_equal={ok_i} ({dt*1e3:.1f} ms)", flush=True)
    if verbose and not (ok_s and ok_i):
        print(" oracle row0 scores", ov[0][:8], "ids", oi[0][:8])
        print(" kernel row0 scores", s[0][:8], "ids", i[0][:8])
        if k == n:
            # reconstruct the kernel's score matrix
            M = np.full((nq, n), np.nan, dtype=np.float32)
            for r in range(nq):
                for c in range(k):
                    if 0 <= i[r, c] < n:
                        M[r, i[r, c]] = s[r, c]
            diff = (M != S.astype(np.float32))
            print(" matrix mismatches:", int(diff.sum()), "of", diff.size)
            rows = np.where(diff.any(axis=1))[0]
            cols = np.where(diff.any(axis=0))[0]
            print(" bad rows", rows[:20], "count", len(rows))
            print(" bad cols", cols[:40], "count", len(cols))
            print(" kernel M[0,:16]", M[0, :16])
            print(" oracle S[0,:16]", S[0, :16].astype(np.float32))
    return ok_s and ok_i


results = {}
try:
    results["single_small"] = run_case(128, 4, 128)
    results["single_c1"] = run_case(10000, 64, 40)
    results["tiny_full"] = run_case(128, 4, 128)          # whole matrix, single tile
    results["tiny_full_2tiles"] = run_case(256, 130, 256) # two tiles, both query halves
    results["ragged"] = run_case(257, 3, 5)
    results["c1"] = run_case(10000, 64, 40)
    results["c1_k80"] = run_case(10000, 64, 80)
    results["c1_gauss"] = run_case(10000, 64, 40, dist="gauss", verbose=False)
    results["sampled_200k"] = run_case(200000, 256, 40)
    results["sampled_200k_exh"] = run_case(200000, 256, 40, exhaustive=True)
    results["nq300"] = run_case(50000, 300, 40)
except Exception as e:
    import traceback; traceback.print_exc()
print(json.dumps(results), flush=True)

# quick timing at C2
try:
    n = 4 * 1024 * 1024
    g = torch.Generator(device=dev).manual_seed(0)
    bank = (torch.randn(n, 768, device=dev, generator=g, dtype=torch.float32) / 27.7).half() if False else None
    bank = torch.empty(n, 768, device=dev, dtype=torch.float16)
    for s0 in range(0, n, 1 << 18):
        bank[s0:s0 + (1 << 18)] = (torch.randn(1 << 18, 768, device=dev, generator=g) / 27.7).half()
    q = torch.randn(256, 768, device=dev, generator=g)
    for _ in range(3):
        s, i, st = ops.mips_topk(bank, q, 40)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(10):
        s, i, st = ops.mips_topk(bank, q, 40)
    ev[1].record(); torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / 10
    print(f"C2 mips_topk: {ms:.3f} ms/search  -> {n*1536/ms/1e6:.1f} GB/s  status={int(st.item())}", flush=True)
    # reference torch path on GPU for comparison
    bt = bank.T  # [768, n] view
    qh = q.half()
    for _ in range(2):
        sc = torch.matmul(qh, bt); v, ix = torch.topk(sc, 40, dim=1)
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(3):
        sc = torch.matmul(qh, bt); v, ix = torch.topk(sc, 40, dim=1)
    ev[1].record(); torch.cuda.synchronize()
    print(f"C2 torch matmul+topk: {ev[0].elapsed_time(ev[1])/3:.3f} ms", flush=True)
    print("values equal to torch.topk:", bool((v == s).all().item()))
except Exception as e:
    import traceback; traceback.print_exc()
