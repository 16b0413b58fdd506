"""TEST INFRASTRUCTURE - CPU restatement of the product-quantized index (csrc/pq.cu, atlas_b200.index.DistributedFAISSIndex).

Only tests and `__graft_entry__.smoke()` import it, as the checker.

Parity status: NOT pinned to the reference.  The reference delegates to faiss (IndexPQ / GpuIndexIVFPQ, src/index.py:163-381),
which is not available here, so nothing can be compared against faiss's output.  The rules below are pinned instead on
hand-written cases whose answers are known by construction (tests/test_pq_cpu.py):
  * `adc_scores`      score(q, x) = sum_m LUT[q][m][code_m] (m ascending, fp32) + T[q][list] (ivfpq), rounded ONCE to fp16;
                      LUT[q][m][j] = <q_m, cb[m][j]> and T[q][l] = <q, coarse[l]> in fp32 from the fp16-rounded queries
  * `encode`          code_m = argmin_j ||r_m - cb[m][j]||^2 (lowest j on ties) of the residual r = x - coarse[list] (fp32);
                      list = argmax_l <x, coarse[l]> (lowest l on ties)
  * `kmeans`          plain Lloyd iterations (the quality yardstick of the device k-means, not its bitwise twin)
  * `canonical_topk`  mips_oracle's top-k with the canonical tie order (score desc, id asc)
Dimensions are generic (d = M * dsub) so that hand cases can be small; the product uses d = 768.
"""
import numpy as np

from mips_oracle import canonical_topk  # noqa: F401  (re-exported: the selection rule is the flat index's)

KSUB = 256


def _q32(queries):
    return np.asarray(queries).astype(np.float16).astype(np.float32)


def lut(queries, codebooks):
    """queries [nq, d], codebooks [M, ksub, dsub] -> fp32 [nq, M, ksub]."""
    cb = np.asarray(codebooks, dtype=np.float32)
    M, _, dsub = cb.shape
    q = _q32(queries).reshape(-1, M, dsub)
    return np.einsum("qmd,mjd->qmj", q, cb).astype(np.float32)


def coarse_terms(queries, coarse):
    """queries [nq, d], coarse [n_list, d] -> fp32 [nq, n_list]."""
    return (_q32(queries) @ np.asarray(coarse, dtype=np.float32).T).astype(np.float32)


def adc_scores(queries, codes, codebooks, coarse=None, list_ids=None):
    """fp16 [nq, n] scores of the rows given by codes [n, M] (and list ids [n] for ivfpq)."""
    L = lut(queries, codebooks)
    codes = np.asarray(codes).astype(np.int64)
    nq = L.shape[0]
    acc = np.zeros((nq, codes.shape[0]), dtype=np.float32)
    for m in range(codes.shape[1]):
        acc += L[:, m, codes[:, m]]
    if coarse is not None:
        acc += coarse_terms(queries, coarse)[:, np.asarray(list_ids).astype(np.int64)]
    return acc.astype(np.float16)


def assign_lists(x, coarse):
    """Inner-product coarse assignment, lowest list on ties."""
    s = np.asarray(x, dtype=np.float32) @ np.asarray(coarse, dtype=np.float32).T
    return np.argmax(s, axis=1).astype(np.int64)


def sub_distances(r, codebooks):
    """Squared L2 distances [n, M, ksub] of the sub-vectors of r [n, d] to every centroid."""
    cb = np.asarray(codebooks, dtype=np.float32)
    M, _, dsub = cb.shape
    rs = np.asarray(r, dtype=np.float32).reshape(-1, M, dsub)
    return ((rs[:, :, None, :] - cb[None]) ** 2).sum(-1)


def encode(x, codebooks, coarse=None):
    """(codes uint8 [n, M], list ids [n] or None) of rows x [n, d]."""
    x32 = np.asarray(x).astype(np.float32)
    lists = None
    if coarse is not None:
        lists = assign_lists(x32, coarse)
        x32 = x32 - np.asarray(coarse, dtype=np.float32)[lists]
    codes = np.empty((x32.shape[0], np.asarray(codebooks).shape[0]), dtype=np.uint8)
    for a in range(0, x32.shape[0], 4096):
        codes[a:a + 4096] = np.argmin(sub_distances(x32[a:a + 4096], codebooks), axis=2)
    return codes, lists


def decode(codes, codebooks, coarse=None, list_ids=None):
    cb = np.asarray(codebooks, dtype=np.float32)
    M = cb.shape[0]
    out = np.concatenate([cb[m][np.asarray(codes)[:, m].astype(np.int64)] for m in range(M)], axis=1)
    if coarse is not None:
        out = out + np.asarray(coarse, dtype=np.float32)[np.asarray(list_ids).astype(np.int64)]
    return out


def quantization_mse(x, codes, codebooks, coarse=None, list_ids=None):
    return float(((np.asarray(x, dtype=np.float32) - decode(codes, codebooks, coarse, list_ids)) ** 2).sum(1).mean())


def kmeans(x, k, iters=25, seed=0, inner_product=False, init=None):
    """Plain Lloyd: k random rows (or the rows `init`) as the initial centroids, assignment by L2 (or inner product),
    centroids = means; an empty cluster keeps its centroid."""
    x = np.asarray(x, dtype=np.float32)
    rng = np.random.default_rng(seed)
    c = x[rng.choice(x.shape[0], k, replace=False) if init is None else np.asarray(init)].copy()
    for _ in range(iters):
        if inner_product:
            a = np.argmax(x @ c.T, axis=1)
        else:
            a = np.argmin((c * c).sum(1)[None, :] - 2.0 * (x @ c.T), axis=1)
        for j in range(k):
            sel = a == j
            if sel.any():
                c[j] = x[sel].mean(0)
    return c


def train(x, M, n_list=0, iters=25, seed=0):
    """Oracle pipeline: coarse IP k-means (ivfpq), then one L2 k-means of 256 centroids per sub-space of the residuals.
    Returns (codebooks [M, 256, d / M], coarse [n_list, d] or None)."""
    x = np.asarray(x, dtype=np.float32)
    coarse = None
    r = x
    if n_list:
        coarse = kmeans(x, n_list, iters, seed, inner_product=True)
        r = x - coarse[assign_lists(x, coarse)]
    dsub = x.shape[1] // M
    cb = np.stack([kmeans(r[:, m * dsub:(m + 1) * dsub], KSUB, iters, seed + 1 + m) for m in range(M)])
    return cb, coarse
