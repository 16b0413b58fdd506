"""TEST INFRASTRUCTURE - CPU restatement of the probed IVF search (`nprobe`, csrc/ivf_probe.cu) for ivfpq and ivfsq.

Only tests and `__graft_entry__.smoke()` import it, as the checker.

Parity status: NOT pinned to the reference.  The reference probes every list (nprobe = n_list, src/index.py:212,269);
the probe rule below is faiss's IVF `nprobe` with one stated difference, pinned on hand cases (tests/test_ivf_probe_cpu.py):
  * `probe_lists`   for query q, with T[q][l] the fp32 coarse term the scan adds (ivfpq: pq_oracle.coarse_terms, ivfsq:
                    T of sq_oracle.contract_scores): order(q) = lists by T descending, then list id ascending; P(q) = the
                    shortest prefix of order(q) with at least nprobe lists (empty lists count) that holds at least k rows.
                    faiss instead returns id -1 when its nprobe lists hold fewer than k rows.
  * `restricted_topk`  the canonical top-k (score desc, id asc) of the index's own scores over the rows whose list is in
                    P(q); `pq_probed_topk` / `sq_probed_topk` apply it to pq_oracle.adc_scores / sq_oracle.contract_scores.
"""
import numpy as np

import pq_oracle
import sq_oracle
from mips_oracle import canonical_topk


def probe_lists(T, nprobe, list_sizes, k):
    """bool [nq, n_list]: list l is in P(q).  T [nq, n_list] fp32, list_sizes [n_list] real rows, k <= sum(list_sizes)."""
    T = np.asarray(T, np.float32)
    sizes = np.asarray(list_sizes, np.int64)
    nq, n_list = T.shape
    if k > sizes.sum():
        raise ValueError(f"k={k} exceeds the {int(sizes.sum())} rows of all lists")
    out = np.zeros((nq, n_list), bool)
    ids = np.arange(n_list)
    for q in range(nq):
        order = np.lexsort((ids, -T[q].astype(np.float64)))     # T descending, then list id ascending
        held = np.cumsum(sizes[order])
        p = min(max(int(nprobe), 1), n_list)
        while held[p - 1] < k:
            p += 1
        out[q, order[:p]] = True
    return out


def restricted_topk(scores16, row_lists, probed, k):
    """Canonical top-k of fp16 scores [nq, n] over the rows whose list (row_lists [n]) is probed ([nq, n_list])."""
    s = np.asarray(scores16, np.float16).copy()
    keep = np.asarray(probed)[:, np.asarray(row_lists, np.int64)]
    s[~keep] = np.float16(-np.inf)
    return canonical_topk(s, k)


def pq_coarse_terms(queries, coarse):
    return pq_oracle.coarse_terms(queries, coarse)


def sq_coarse_terms(queries, coarse):
    """T of sq_oracle.contract_scores: fp32 of the float64 product."""
    q = np.asarray(queries).astype(np.float16).astype(np.float64)
    return (q @ np.asarray(coarse, np.float64).T).astype(np.float32)


def pq_probed_topk(queries, codes, codebooks, coarse, list_ids, nprobe, k, T=None):
    """(scores fp16 [nq, k], ids [nq, k], probed [nq, n_list]) of the probed ivfpq search."""
    lists = np.asarray(list_ids, np.int64)
    n_list = np.asarray(coarse).shape[0]
    T = pq_coarse_terms(queries, coarse) if T is None else T
    probed = probe_lists(T, nprobe, np.bincount(lists, minlength=n_list), k)
    s = pq_oracle.adc_scores(queries, codes, codebooks, coarse, lists)
    v, i = restricted_topk(s, lists, probed, k)
    return v, i, probed


def sq_probed_topk(queries, codes, vmin, vdiff, coarse, lists, nprobe, k, T=None):
    """(scores fp16 [nq, k], ids [nq, k], probed [nq, n_list]) of the probed ivfsq search, codes unpacked [n, 768]."""
    lists = np.asarray(lists, np.int64)
    n_list = np.asarray(coarse).shape[0]
    T = sq_coarse_terms(queries, coarse) if T is None else T
    probed = probe_lists(T, nprobe, np.bincount(lists, minlength=n_list), k)
    s = sq_oracle.contract_scores(queries, codes, vmin, vdiff, coarse, lists)
    v, i = restricted_topk(s, lists, probed, k)
    return v, i, probed
