"""The product-quantized index (`--index_mode faiss`, atlas_b200.index.DistributedFAISSIndex) on one GPU, at the shard size
of bench.py (4 Mi passages of 768-d fp16 per GPU, BASELINE configs[1]).  Prints one JSON line with:
  train_index_s               train + encode of every row (host rows staged through the device)
  value / ms_per_search       search queries/s at 256 queries / top-40, CUDA events, device-resident queries
  flat                        the exact flat scan (ops.mips_topk) on the same bank, same timing
  sweep                       code bytes per search (computed from shapes) over the main code-sweep kernel time, against the
                              HBM peak
  device_bytes_per_passage    codes + list ids + codebooks + coarse centroids, over the rows
  recall_at_40                against the exact flat search, on a synthetic Gaussian bank: says little about real embeddings
  refine                      with --refine-factor R > 1 only: the same search re-ranked by exact score over the top
                              k' = 40 R PQ candidates (refine_factor = R): queries/s, recall_at_40 refined vs unrefined, the
                              refine kernel's time and the host-row bytes it reads per search (nq k' 1536, from shapes) over
                              that time
    python tools/perf_pq_index.py [--index-type ivfpq] [--code-size 16] [--rows N] [--steps 20] [--warmup 3]
                                  [--refine-factor 1]
Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import DIM, N_LOCAL, NQ, TOPK, make_bank, make_queries, peaks  # noqa: E402


def measure(args):
    import ctypes

    import torch

    from atlas_b200 import ops
    from atlas_b200._lib import lib
    from atlas_b200.index import DistributedFAISSIndex

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = lib()
    rows, M = args.rows, args.code_size
    steps, warmup = args.steps, args.warmup
    bank = make_bank(rows, dev, seed=1)
    q = make_queries().to(dev)

    def timed(fn):
        for _ in range(warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps, out

    flat_ms, (_, exact, st) = timed(lambda: ops.mips_topk(bank, q, TOPK))
    assert int(st.item()) == 0
    exact = exact.cpu().numpy()
    index = DistributedFAISSIndex(args.index_type, M)
    index._bank = index._host_rows(rows)
    index._bank.copy_(bank)
    del bank
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    index.train_index()
    torch.cuda.synchronize()
    train_s = time.perf_counter() - t0
    p = index._pq
    dev_bytes = sum(t.numel() * t.element_size() for t in (p["codes"], p["list_ids"], p["codebooks"], p["coarse"])
                    if t is not None)
    L.atlas_b200_profile_enable(1)
    ms, (_, ids, st) = timed(lambda: index.search_device(q, TOPK, return_status=True))
    kms, kn = ctypes.c_double(0), ctypes.c_int32(0)
    L.atlas_b200_profile_collect(ctypes.byref(kms), ctypes.byref(kn))
    L.atlas_b200_profile_enable(0)
    assert int(st.item()) == 0, "fast search path overflowed"
    ids = ids.cpu().numpy()
    recall_of = lambda ids: float(sum(len(set(a) & set(b)) for a, b in zip(ids.tolist(), exact.tolist())) / (NQ * TOPK))
    recall = recall_of(ids)
    list_bytes = 0 if p["list_ids"] is None else p["list_ids"].element_size()
    groups = kn.value // (steps + warmup) if kn.value else 0
    kernel_ms = kms.value / (steps + warmup)
    sweep_bytes = rows * (M + list_bytes)
    peak, peak_src = peaks("hbm")
    achieved = sweep_bytes / (kernel_ms * 1e-3) / 1e9 if kernel_ms > 0 else 0.0
    refine = None
    if args.refine_factor > 1:
        index.refine_factor = args.refine_factor
        k_cand = min(TOPK * args.refine_factor, rows)
        rms, (_, rids, st) = timed(lambda: index.search_device(q, TOPK, return_status=True))
        assert int(st.item()) == 0, "fast search path overflowed"
        L.atlas_b200_profile_enable(7)     # the refine kernel (csrc/pq_refine.cu)
        timed(lambda: index.search_device(q, TOPK, return_status=True))
        L.atlas_b200_profile_collect(ctypes.byref(kms), ctypes.byref(kn))
        L.atlas_b200_profile_enable(0)
        refine_kernel_ms = kms.value / (steps + warmup)
        host_bytes = NQ * k_cand * DIM * 2
        refine = {"refine_factor": args.refine_factor, "candidates_per_query": k_cand,
                  "value": NQ / (rms * 1e-3), "unit": "queries/s", "ms_per_search": rms,
                  "recall_at_40": recall_of(rids.cpu().numpy()), "recall_at_40_unrefined": recall,
                  "kernel": "pq_refine_kernel (zero-copy reads of the pinned host rows)",
                  "kernel_ms_per_search": refine_kernel_ms, "host_bytes_per_search": host_bytes,
                  "host_link_GBps": host_bytes / (refine_kernel_ms * 1e-3) / 1e9 if refine_kernel_ms > 0 else 0.0}
    try:
        smi = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        smi = None
    return {
        "metric": f"{args.index_type} index search queries/sec (top-{TOPK}, {NQ}-query batches, code_size {M})",
        "value": NQ / (ms * 1e-3), "unit": "queries/s", "ms_per_search": ms, "steps": steps, "rows": rows,
        "index_type": args.index_type, "code_size": M, "n_list": p["n_list"], "train_index_s": train_s,
        "flat": {"value": NQ / (flat_ms * 1e-3), "unit": "queries/s", "ms_per_search": flat_ms,
                 "call": "ops.mips_topk (exact fp16 bank scan, device-resident bank)"},
        "sweep": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                  "frac": achieved / peak if peak else None, "peak_source": peak_src,
                  "kernel": "pq_scan_kernel (main sweep; codes re-read once per query group, so real traffic is higher)",
                  "kernel_ms_per_search": kernel_ms, "kernel_launches_per_search": groups,
                  "code_bytes_per_search": sweep_bytes},
        "device_bytes_per_passage": dev_bytes / rows, "flat_device_bytes_per_passage": DIM * 2,
        "recall_at_40": recall, "recall_note": "against the exact flat search on a synthetic Gaussian bank; not "
                                               "representative of real embeddings",
        "gpu": smi,
    } | ({"refine": refine} if refine else {})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--index-type", choices=["pq", "ivfpq"], default="ivfpq")
    ap.add_argument("--code-size", type=int, default=16, help="bytes of PQ code per passage")
    ap.add_argument("--rows", type=int, default=N_LOCAL)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--refine-factor", type=int, default=1,
                    help="also time the search re-ranked over refine-factor x 40 PQ candidates (1 = off)")
    print(json.dumps(measure(ap.parse_args())))


if __name__ == "__main__":
    main()
