"""TEST INFRASTRUCTURE - CPU restatement of the exact re-ranking of product-quantized candidates (csrc/pq_refine.cu,
`atlas_b200.ops.pq_refine_topk`, `DistributedFAISSIndex(refine_factor > 1)`; faiss's IndexRefineFlat).

Only tests import it, as the checker.  Pinned on hand-written cases in tests/test_pq_refine_cpu.py:
  * score(q, x) = fp32 dot product of the fp16-rounded query with the fp16 row, rounded ONCE to fp16 (the flat index's
    score, mips_oracle.scores_fp16, up to the fp32 summation order);
  * per query, the canonical top-k of its candidates (score desc, global id asc; pq_oracle.canonical_topk) with
    global id = id_base + id_stride * local row;
  * candidates outside [0, n) are skipped; fewer than k valid ones leave a (-inf, -1) tail.
"""
import numpy as np

from pq_oracle import canonical_topk


def refine_topk(queries, rows, cand_local, k, id_base=0, id_stride=1):
    """queries [nq, d], rows [n, d] fp16, cand_local [nq, k'] local rows -> (fp16 [nq, k] desc, int64 global ids [nq, k])."""
    q = np.asarray(queries).astype(np.float16).astype(np.float32)
    rows = np.asarray(rows)
    assert rows.dtype == np.float16
    cand = np.asarray(cand_local, dtype=np.int64)
    nq, n = q.shape[0], rows.shape[0]
    out_v = np.full((nq, k), -np.inf, dtype=np.float16)
    out_i = np.full((nq, k), -1, dtype=np.int64)
    for j in range(nq):
        c = cand[j][(cand[j] >= 0) & (cand[j] < n)]
        if len(c) == 0:
            continue
        s = (rows[c].astype(np.float32) @ q[j]).astype(np.float32).astype(np.float16)
        kk = min(k, len(c))
        v, i = canonical_topk(s[None, :], kk, ids=id_base + id_stride * c)
        out_v[j, :kk], out_i[j, :kk] = v[0], i[0]
    return out_v, out_i
