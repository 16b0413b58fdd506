"""The product-quantized index (`--index_mode faiss`, atlas_b200.index.DistributedFAISSIndex) on one GPU, at the shard size
of bench.py (4 Mi passages of 768-d fp16 per GPU, BASELINE configs[1]).  Prints one JSON line with:
  train_index_s               train + encode of every row (host rows staged through the device)
  value / ms_per_search       search queries/s at 256 queries / top-40, CUDA events, device-resident queries
  flat                        the exact flat scan (ops.mips_topk) on the same bank, same timing
  sweep                       code bytes per search (computed from shapes) over the main code-sweep kernel time, against the
                              HBM peak
  device_bytes_per_passage    every device tensor of the trained index (codes, list ids or slot rows, codebooks or
                              ranges, coarse centroids), over the rows
  recall_at_40                against the exact flat search, on a synthetic Gaussian bank: says little about real embeddings
  refine                      with --refine-factor R > 1 only: the same search re-ranked by exact score over the top
                              k' = 40 R PQ candidates (refine_factor = R): queries/s, recall_at_40 refined vs unrefined, the
                              refine kernel's time and the host-row bytes it reads per search (nq k' 1536, from shapes) over
                              that time
  at_8_queries                the same search, and the flat scan, at 8 queries per search (bench.py's per-rank batch)
  ivfsq / ivfflat             with --index-type ivfsq or ivfflat only: each sweep's kernel time (256 and 8 queries) against
                              the larger of its two bounds from shapes: the code (ivfflat: fp16 row) bytes over the HBM
                              peak, and 2 x 768 x slots x queries FLOPs over the dense fp16 tensor peak
    python tools/perf_pq_index.py [--index-type ivfpq] [--code-size 16] [--rows N] [--steps 20] [--warmup 3]
                                  [--refine-factor 1]
With --nprobe 8,32,128 it measures the probed search instead, for ivfpq (--code-size) and ivfsq (or, with --index-type
ivfflat, for ivfflat alone, and the flat scan beside it at both batch sizes) on a seeded CLUSTERED
bank (a Gaussian mixture: on an isotropic bank IVF recall means nothing; this is still not real embeddings): per index
type, nprobe (and "all", the full scan) and batch of 8 and 256 queries, queries/s, recall@40 against the exact flat
search, the fast path's overflow flag (`fast_path_status`; the timed search includes the exhaustive retry when it is
set), and the sweep's kernel time against the HBM bound of the code bytes of the lists it had to read (the union of
the block's probe sets, computed on the host from the coarse terms; the probe-set extension for small lists is ignored,
it does not trigger at this shard size; a probed ivfpq row costs its 4-byte list position and a 32-byte sector per
scattered code read).
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
    rows = args.rows
    M = None if args.index_type in ("ivfsq", "ivfflat") else args.code_size
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
    flat8_ms, _ = timed(lambda: ops.mips_topk(bank, q[:8], TOPK))
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
    dev_bytes = sum(t.numel() * t.element_size() for t in p.values() if torch.is_tensor(t))

    def profiled(queries):
        L.atlas_b200_profile_enable(1)
        ms, out = timed(lambda: index.search_device(queries, TOPK, return_status=True))
        kms, kn = ctypes.c_double(0), ctypes.c_int32(0)
        L.atlas_b200_profile_collect(ctypes.byref(kms), ctypes.byref(kn))
        L.atlas_b200_profile_enable(0)
        return ms, out, kms, kn

    ms, (_, ids, st), kms, kn = profiled(q)
    assert int(st.item()) == 0, "fast search path overflowed"
    ids = ids.cpu().numpy()
    recall_of = lambda ids, nq=NQ: float(sum(len(set(a) & set(b)) for a, b in zip(ids.tolist(), exact[:nq].tolist()))
                                         / (nq * TOPK))
    recall = recall_of(ids)
    list_bytes = 0 if p.get("list_ids") is None else p["list_ids"].element_size()
    groups = kn.value // (steps + warmup) if kn.value else 0
    kernel_ms = kms.value / (steps + warmup)
    slot_bytes = DIM * 2 if args.index_type == "ivfflat" else ops.SQ_CODE_BYTES
    sweep_bytes = rows * (M + list_bytes) if M else p["slot_rows"].numel() * slot_bytes
    peak, peak_src = peaks("hbm")
    achieved = sweep_bytes / (kernel_ms * 1e-3) / 1e9 if kernel_ms > 0 else 0.0
    ms8, (_, ids8, st8), kms8, _ = profiled(q[:8])
    assert int(st8.item()) == 0, "fast search path overflowed"
    recall8 = recall_of(ids8.cpu().numpy(), 8)
    ivfsq = None
    if args.index_type in ("ivfsq", "ivfflat"):
        slots = p["slot_rows"].shape[0]
        tflops, tensor_src = 989.0, "H100 SXM data sheet, dense fp16"

        def bounds(nq, kernel_ms):
            hbm_ms = slots * slot_bytes / (peak * 1e9) * 1e3
            tensor_ms = 2.0 * DIM * slots * nq / (tflops * 1e12) * 1e3
            bound_ms = max(hbm_ms, tensor_ms)
            return {"queries": nq, "kernel_ms_per_search": kernel_ms, "hbm_bound_ms": hbm_ms, "tensor_bound_ms": tensor_ms,
                    "binding": "hbm" if hbm_ms >= tensor_ms else "tensor",
                    "frac_of_binding_bound": bound_ms / kernel_ms if kernel_ms > 0 else None}

        ivfsq = {"slots": slots, "padding_frac": slots / rows - 1.0, "tensor_peak_tflops": tflops,
                 "tensor_peak_source": tensor_src,
                 "at_256": {"value": NQ / (ms * 1e-3), "unit": "queries/s", "ms_per_search": ms} | bounds(NQ, kernel_ms),
                 "at_8": bounds(8, kms8.value / (steps + warmup))}
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
        "at_8_queries": {"value": 8 / (ms8 * 1e-3), "unit": "queries/s", "ms_per_search": ms8, "recall_at_40": recall8,
                         "flat_value": 8 / (flat8_ms * 1e-3), "flat_ms_per_search": flat8_ms},
        "flat": {"value": NQ / (flat_ms * 1e-3), "unit": "queries/s", "ms_per_search": flat_ms,
                 "call": "ops.mips_topk (exact fp16 bank scan, device-resident bank)"},
        "sweep": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                  "frac": achieved / peak if peak else None, "peak_source": peak_src,
                  "kernel": {"ivfsq": "ivfsq_scan_kernel (main sweep; codes read once per 128 queries)",
                             "ivfflat": "ivfflat_scan_kernel (main sweep; rows read once per 256 queries)"}.get(
                                 args.index_type,
                                 "pq_scan_kernel (main sweep; codes re-read once per query group, so real traffic is higher)"),
                  "kernel_ms_per_search": kernel_ms, "kernel_launches_per_search": groups,
                  "code_bytes_per_search": sweep_bytes},
        "device_bytes_per_passage": dev_bytes / rows, "flat_device_bytes_per_passage": DIM * 2,
        "recall_at_40": recall, "recall_note": "against the exact flat search on a synthetic Gaussian bank; not "
                                               "representative of real embeddings",
        "gpu": smi,
    } | ({"refine": refine} if refine else {}) | ({args.index_type: ivfsq} if ivfsq else {})


def clustered_bank(rows, dev, centers=4096, spread=0.35, seed=3):
    """Seeded Gaussian mixture, rows and queries drawn alike, scaled like bench.make_bank's rows."""
    import torch

    g = torch.Generator(device=dev).manual_seed(seed)
    c = torch.randn((centers, DIM), generator=g, device=dev)
    bank = torch.empty((rows, DIM), dtype=torch.float16, device=dev)
    for a in range(0, rows, 1 << 20):
        b = min(rows, a + (1 << 20))
        pick = torch.randint(0, centers, (b - a,), generator=g, device=dev)
        bank[a:b] = ((c[pick] + spread * torch.randn((b - a, DIM), generator=g, device=dev)) / DIM ** 0.5).half()
    pick = torch.randint(0, centers, (NQ,), generator=g, device=dev)
    q = ((c[pick] + spread * torch.randn((NQ, DIM), generator=g, device=dev)) / DIM ** 0.5).half()
    return bank, q


def measure_nprobe(args):
    import ctypes

    import torch

    from atlas_b200 import ops
    from atlas_b200._lib import lib
    from atlas_b200.index import DistributedFAISSIndex

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = lib()
    rows, steps, warmup = args.rows, args.steps, args.warmup
    nprobes = [int(v) for v in args.nprobe.split(",")]
    bank, q = clustered_bank(rows, dev)
    _, exact, st = ops.mips_topk(bank, q, TOPK)
    assert int(st.item()) == 0
    exact = exact.cpu().numpy()
    host = None
    peak, peak_src = peaks("hbm")
    out = {"metric": "probed IVF search (nprobe), top-40", "rows": rows, "steps": steps,
           "bank": "seeded Gaussian mixture (4096 centres, spread 0.35): clustered, still not real embeddings",
           "hbm_peak_GBps": peak, "peak_source": peak_src, "results": []}
    kinds = ("ivfflat",) if args.index_type == "ivfflat" else ("ivfpq", "ivfsq")
    if args.index_type == "ivfflat":
        # the exact flat scan of the same bank (ops.mips_topk, device-resident), for comparison
        out["flat"] = []
        for nq in (8, NQ):
            fn = lambda: ops.mips_topk(bank, q[:nq], TOPK)
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / steps
            out["flat"].append({"queries": nq, "value": nq / (ms * 1e-3), "unit": "queries/s", "ms_per_search": ms,
                                "hbm_bound_ms": rows * DIM * 2 / (peak * 1e9) * 1e3})
    for kind in kinds:
        index = DistributedFAISSIndex(kind, args.code_size if kind == "ivfpq" else None)
        if host is None:
            host = index._host_rows(rows)
            host.copy_(bank)
            del bank
            torch.cuda.empty_cache()
        index._bank = host
        index.train_index()
        p = index._pq
        n_list = p["n_list"]
        if kind in ("ivfsq", "ivfflat"):
            tl = p["tile_lists"].to(torch.int64)
            slot_bytes = ops.SQ_CODE_BYTES if kind == "ivfsq" else DIM * 2
            list_bytes = torch.bincount(tl, minlength=n_list).double() * ops.SQ_TILE * slot_bytes
        else:
            # a probed ivfpq sweep reads each probed row's list position (4 B, in order) and then its codes through that
            # permutation: scattered reads that each move whole 32-byte sectors
            sector_bytes = (args.code_size + 31) // 32 * 32
            list_bytes = torch.bincount(p["list_ids"].to(torch.int64), minlength=n_list).double() * (sector_bytes + 4)
        T = q.float() @ p["coarse"].t()          # the coarse terms, up to the fp32 summation order
        for nq in (8, NQ):
            for nprobe in nprobes + [None]:
                index.nprobe = nprobe
                # the fast path's overflow flag, then the timed search: the final result, i.e. with the exhaustive retry
                # (and the host synchronisation that reads the flag) whenever the flag is set, as search_knn runs it
                status = int(index.search_device(q[:nq], TOPK, return_status=True)[2].item())
                fn = lambda: index.search_device(q[:nq], TOPK)
                for _ in range(warmup):
                    fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                L.atlas_b200_profile_enable(1)
                e0.record()
                for _ in range(steps):
                    _, ids = fn()
                e1.record()
                torch.cuda.synchronize()
                kms, kn = ctypes.c_double(0), ctypes.c_int32(0)
                L.atlas_b200_profile_collect(ctypes.byref(kms), ctypes.byref(kn))
                L.atlas_b200_profile_enable(0)
                ms = e0.elapsed_time(e1) / steps
                kernel_ms = kms.value / steps
                if nprobe is None or nprobe >= n_list:
                    read = float(list_bytes.sum()) if kind != "ivfpq" else float(rows * (args.code_size + 2))
                else:
                    union = torch.zeros(n_list, dtype=torch.bool, device=dev)
                    union[torch.topk(T[:nq], nprobe, dim=1).indices.flatten()] = True
                    read = float(list_bytes[union].sum())
                    if kind == "ivfsq" and nq > 128:     # each 128-query group reads the lists its queries probe
                        read = sum(float(list_bytes[torch.unique(torch.topk(T[g:g + 128], nprobe, dim=1).indices)].sum())
                                   for g in range(0, nq, 128))
                hbm_ms = read / (peak * 1e9) * 1e3
                rec = float(sum(len(set(a) & set(b)) for a, b in zip(ids.cpu().numpy().tolist(), exact[:nq].tolist()))
                            / (nq * TOPK))
                out["results"].append({
                    "index_type": kind, "n_list": n_list, "nprobe": nprobe if nprobe is not None else "all",
                    "queries": nq, "value": nq / (ms * 1e-3), "unit": "queries/s", "ms_per_search": ms,
                    "recall_at_40": rec, "fast_path_status": status, "sweep_kernel_ms": kernel_ms,
                    "code_bytes_read": read, "hbm_bound_ms": hbm_ms,
                    "frac_of_hbm_bound": hbm_ms / kernel_ms if kernel_ms > 0 else None})
        index.nprobe = None
        del index, p
        torch.cuda.empty_cache()
    try:
        out["gpu"] = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out["gpu"] = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--index-type", choices=["pq", "ivfpq", "ivfsq", "ivfflat"], default="ivfpq")
    ap.add_argument("--code-size", type=int, default=16, help="bytes of PQ code per passage (ivfsq: always 4 bits per dim)")
    ap.add_argument("--rows", type=int, default=N_LOCAL)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--refine-factor", type=int, default=1,
                    help="also time the search re-ranked over refine-factor x 40 PQ candidates (1 = off)")
    ap.add_argument("--nprobe", default=None,
                    help="comma-separated nprobe values: measure the probed search of ivfpq and ivfsq (of ivfflat with "
                         "--index-type ivfflat) instead")
    args = ap.parse_args()
    print(json.dumps(measure_nprobe(args) if args.nprobe else measure(args)))


if __name__ == "__main__":
    main()
