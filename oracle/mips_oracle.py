"""CPU oracle for the exact MIPS + top-k path of Atlas' flat index.

TEST INFRASTRUCTURE ONLY.  Only `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` /
`--impl reference` legs of `bench.py` may import this file, and only as the checker or the
timed CPU baseline.  The product path (`atlas_b200/`) never imports `oracle/`; it raises if the
CUDA library is missing.

Parity status: PINNED.  `oracle/make_golden.py` runs the unmodified reference
(`/root/reference/src/index.py`, imported under `oracle/ref_shims.py`) on the same seeded
inputs and commits its outputs under `tests/golden/mips_*.npz`; `tests/test_oracle_golden.py`
checks this restatement against those files on every CPU run.

Restated reference code (numpy, no torch):
  * `scores_fp16`          <- `DistributedIndex._compute_scores_and_indices`, src/index.py:113-117
                              (`torch.matmul(allqueries.half(), self.embeddings)`: fp16 operands,
                              fp32 accumulation, ONE rounding of the result to fp16)
  * `canonical_topk`       <- `torch.topk(scores, topk, dim=1)`, src/index.py:118, with the tie
                              order pinned: stable sort by (score desc, id asc).
  * `search_knn_oracle`    <- `DistributedIndex.search_knn`, src/index.py:122-157, for a world of
                              W ranks holding round-robin shards (src/index_io.py:41).
"""
import numpy as np


def scores_fp16(queries, bank):
    """queries [nq, d] (any float dtype), bank [n, d] fp16 (row = passage) -> [nq, n] fp16.

    src/index.py:117 casts queries with `.half()` (round-to-nearest-even) and multiplies by the
    fp16 bank; products of two fp16 numbers are exact in fp32, accumulation is fp32, the result is
    rounded once to fp16.  numpy's float32 matmul (BLAS sgemm) has exactly those semantics up to
    the accumulation ORDER, which does not matter for the exact-grid inputs (oracle/synth.py)."""
    q = np.asarray(queries).astype(np.float16).astype(np.float32)
    b = np.asarray(bank)
    assert b.dtype == np.float16, "the reference bank is fp16 (src/index.py:51)"
    out = np.empty((q.shape[0], b.shape[0]), dtype=np.float16)
    step = 1 << 16
    for s in range(0, b.shape[0], step):
        out[:, s:s + step] = (q @ b[s:s + step].astype(np.float32).T).astype(np.float16)
    return out


def canonical_topk(scores, k, ids=None):
    """Row-wise top-k of an fp16 score matrix with the canonical tie rule.

    Returns (values [nq,k] fp16 descending, ids [nq,k] int64).  Order: score descending, then id
    ascending (-0.0 == +0.0, as in torch.topk's float comparison).  `ids` optionally maps column ->
    id (default: the column number, i.e. the reference's local index, src/index.py:118)."""
    scores = np.asarray(scores)
    nq, n = scores.shape
    if k > n:
        # torch.topk raises "selected index k out of range" (src/index.py:118)
        raise RuntimeError(f"selected index k out of range: k={k} > n={n}")
    col_ids = np.arange(n, dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    s32 = scores.astype(np.float32) + 0.0  # canonicalise -0.0
    out_v = np.empty((nq, k), dtype=np.float16)
    out_i = np.empty((nq, k), dtype=np.int64)
    for r in range(nq):
        order = np.lexsort((col_ids, -s32[r]))[:k]  # last key is primary
        out_v[r] = scores[r, order]
        out_i[r] = col_ids[order]
    return out_v, out_i


def shard_rows(n_total, rank, world_size):
    """Global line numbers held by `rank` (src/index_io.py:41): g = rank, rank+W, ..."""
    return np.arange(rank, n_total, world_size, dtype=np.int64)


def search_knn_oracle(bank, queries_per_rank, k):
    """Distributed exact search restated for W = len(queries_per_rank) ranks.

    bank: the FULL [n, d] fp16 bank in global line order; rank r holds rows r::W.
    queries_per_rank: list of [nq_r, d] arrays (nq_r may be 0, src/atlas.py:103-106).
    Returns per rank (scores [nq_r,k] fp16, global_ids [nq_r,k] int64).

    Follows src/index.py:127-157: every rank scores ALL gathered queries against its shard and
    keeps its local top-k (:131), the per-shard lists are gathered to the rank that owns the query
    and concatenated in rank order (:138-150), and a second top-k over the W*k candidates picks the
    result (:151-156).  Ties use the canonical rule on (score, global id)."""
    world = len(queries_per_rank)
    allq = np.concatenate([np.asarray(q, dtype=np.float32).reshape(-1, bank.shape[1]) for q in queries_per_rank])
    sizes = np.cumsum([0] + [len(q) for q in queries_per_rank])
    per_shard = []
    for r in range(world):
        rows = shard_rows(bank.shape[0], r, world)
        s = scores_fp16(allq, bank[rows])
        v, local = canonical_topk(s, k)
        per_shard.append((v, rows[local]))  # local index l -> global line l*W + r
    cat_v = np.concatenate([v for v, _ in per_shard], axis=1)  # [nq, W*k], rank order
    cat_i = np.concatenate([i for _, i in per_shard], axis=1)
    out = []
    for r in range(world):
        lo, hi = sizes[r], sizes[r + 1]
        vs = np.empty((hi - lo, k), dtype=np.float16)
        gs = np.empty((hi - lo, k), dtype=np.int64)
        for j, row in enumerate(range(lo, hi)):
            order = np.lexsort((cat_i[row], -(cat_v[row].astype(np.float32) + 0.0)))[:k]
            vs[j] = cat_v[row, order]
            gs[j] = cat_i[row, order]
        out.append((vs, gs))
    return out


def ids_match_tie_aware(scores_row, ids_a, ids_b):
    """True if two id lists for one query agree at every position whose score is unique in the
    row's top-k and differs from the k-th score (positions where torch.topk's unspecified tie order
    or the k-boundary cannot matter)."""
    s = np.asarray(scores_row, dtype=np.float32)
    ok = True
    for p in range(len(s)):
        unique = (s == s[p]).sum() == 1 and s[p] != s[-1]
        if unique and ids_a[p] != ids_b[p]:
            ok = False
    return ok
