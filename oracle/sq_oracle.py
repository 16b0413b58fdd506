"""TEST INFRASTRUCTURE - CPU restatement of the IVF-SQ index (csrc/pq.cu, csrc/ivfsq.cu, DistributedFAISSIndex("ivfsq")).

Only tests and `__graft_entry__.smoke()` import it, as the checker.

Parity status: NOT pinned to the reference.  The reference delegates to faiss (GpuIndexIVFScalarQuantizer with QT_4bit,
encodeResidual=True and METRIC_INNER_PRODUCT, src/index.py:332-343), which is not available here.  The rules below are
faiss 1.7.2's, written out and pinned on hand cases whose answers are known by construction (tests/test_ivfsq_cpu.py):
  * `train_range`      per dim: vmin = min r_d, vdiff = max r_d - vmin over the training residuals (RS_minmax, rangestat_arg
                       = 0, one range per dimension), fp32
  * `encode`           xi = fp32((r_d - vmin_d) / vdiff_d), 0 when vdiff_d == 0, clamped to [0, 1];
                       code_d = (int)(xi * 15.0) with the product in double, as faiss multiplies a float by the double 15.0;
                       dim 2j in the low nibble of byte j, dim 2j + 1 in the high nibble (384 bytes per row)
  * `decode`           x^_d = vmin_d + (code_d + 0.5) / 15 * vdiff_d (+ the coarse centroid of the row's list)
  * `faiss_scores`     float64 <q, c_l> + sum_d q_d x^_d with the fp16-rounded queries: the faiss rule without its fp32
                       rounding (the reference rounds the result once to fp16, src/index.py:219)
  * `contract_scores`  what the device computes, restated exactly:
                         w^[q][d] = fp16(2^e_q * fp32(q_d * fp32(vdiff_d / 15))), e_q putting max_d |w^| in [2^14, 2^15)
                         C[q] = fp32(fp32 sum_d q_d (vmin_d + 0.5 vdiff_d / 15) + 2^-e_q * 8 sum_d w^[q][d])
                         T[q][l] = fp32 <q, c_l>
                         s = fp16(fp32(fp32(T + C) + 2^-e_q * sum_d w^[q][d] (code_d - 8))), the sums exact here (the
                         device accumulates them in fp32, the last one on the tensor cores, whose accumulation does
                         not round to nearest: centring the codes keeps that sum, and its error, small)
  * `contract_error_bound`  a worst-case bound on |contract - faiss| per (query, row): the fp16 rounding of w^ (half an
                       fp16 ulp of each w^, times 15), the fp32 products and sums of w^, C and T, and the final fp16
                       rounding.  It assumes every rounding error points the same way, so it is several fp16 ulps; the
                       gap itself is about one fp16 ulp of the largest score on clustered and Gaussian data.
  * `canonical_topk`   mips_oracle's top-k with the canonical tie order (score desc, id asc)
The product xi * 15.0 is taken in double as faiss does.  For the multiplier 15 the fp32 product truncates to the same
code for every fp32 xi in [0, 1] (checked exhaustively over all 2^30 of them), so it could not differ either.
"""
import numpy as np

from mips_oracle import canonical_topk  # noqa: F401  (re-exported: the selection rule is the flat index's)

DIM = 768
LEVELS = 15
U = 2.0 ** -24    # fp32 unit roundoff


def _q32(queries):
    return np.asarray(queries).astype(np.float16).astype(np.float32)


def residuals(x, coarse, lists):
    """fp32(x) - coarse[list] in fp32."""
    return np.asarray(x).astype(np.float32) - np.asarray(coarse, np.float32)[np.asarray(lists).astype(np.int64)]


def assign_lists(x, coarse):
    """Inner-product coarse assignment, lowest list on ties."""
    return np.argmax(np.asarray(x, np.float32) @ np.asarray(coarse, np.float32).T, axis=1).astype(np.int64)


def train_range(r):
    """(vmin, vdiff) fp32 [d] of residuals r [n, d]."""
    r = np.asarray(r, np.float32)
    vmin = r.min(0)
    return vmin, (r.max(0) - vmin).astype(np.float32)


def quantize(r, vmin, vdiff):
    """Unpacked codes uint8 [n, d] by faiss's rule."""
    r = np.asarray(r, np.float32)
    vmin = np.asarray(vmin, np.float32)
    vdiff = np.asarray(vdiff, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        xi = ((r - vmin) / vdiff).astype(np.float32)
    xi = np.where(vdiff == 0, np.float32(0), np.clip(xi, np.float32(0), np.float32(1)))
    return (xi.astype(np.float64) * 15.0).astype(np.int64).astype(np.uint8)


def pack(codes):
    """[n, d] nibbles -> [n, d / 2] bytes, dim 2j low, 2j + 1 high."""
    c = np.asarray(codes, np.uint8)
    return (c[:, 0::2] | (c[:, 1::2] << 4)).astype(np.uint8)


def unpack(packed):
    p = np.asarray(packed, np.uint8)
    out = np.empty((p.shape[0], 2 * p.shape[1]), np.uint8)
    out[:, 0::2] = p & 15
    out[:, 1::2] = p >> 4
    return out


def encode(r, vmin, vdiff):
    """Packed codes uint8 [n, d / 2] of residuals r [n, d]."""
    return pack(quantize(r, vmin, vdiff))


def decode(codes, vmin, vdiff, coarse=None, lists=None):
    """fp32 reconstruction of unpacked codes [n, d]."""
    c = np.asarray(codes).astype(np.float32)
    x = np.asarray(vmin, np.float32) + (c + np.float32(0.5)) / np.float32(LEVELS) * np.asarray(vdiff, np.float32)
    if coarse is not None:
        x = x + np.asarray(coarse, np.float32)[np.asarray(lists).astype(np.int64)]
    return x.astype(np.float32)


def faiss_scores(queries, codes, vmin, vdiff, coarse, lists):
    """float64 [nq, n] scores of the faiss rule (unrounded), codes unpacked [n, d]."""
    q = _q32(queries).astype(np.float64)
    c = np.asarray(codes).astype(np.float64)
    xh = np.asarray(vmin, np.float64) + (c + 0.5) / LEVELS * np.asarray(vdiff, np.float64)
    t = q @ np.asarray(coarse, np.float64).T
    return t[:, np.asarray(lists).astype(np.int64)] + q @ xh.T


def query_operand(queries, vdiff):
    """(w^ fp16 [nq, d], e_q int [nq]) as the device forms them."""
    q = _q32(queries)
    p = q * (np.asarray(vdiff, np.float32) / np.float32(LEVELS)).astype(np.float32)
    m = np.abs(p).max(1)
    e = np.zeros(len(q), np.int64)
    ok = (m > 0) & np.isfinite(m)
    e[ok] = 15 - np.frexp(m[ok])[1]
    w = np.ldexp(p, e[:, None].astype(np.int32)).astype(np.float32).astype(np.float16)
    return w, e


def contract_scores(queries, codes, vmin, vdiff, coarse, lists, return_fp32=False):
    """fp16 [nq, n] scores of the device contract, codes unpacked [n, d]."""
    q = _q32(queries)
    vmin = np.asarray(vmin, np.float32)
    vdiff = np.asarray(vdiff, np.float32)
    w, e = query_operand(queries, vdiff)
    center = (vmin + (np.float32(0.5) * vdiff) / np.float32(LEVELS)).astype(np.float32)
    C = ((q.astype(np.float64) @ center.astype(np.float64)).astype(np.float32).astype(np.float64)
         + np.ldexp(8.0 * w.astype(np.float64).sum(1), -e)).astype(np.float32)
    T = (q.astype(np.float64) @ np.asarray(coarse, np.float64).T).astype(np.float32)
    base = (T[:, np.asarray(lists).astype(np.int64)] + C[:, None]).astype(np.float32)
    acc = w.astype(np.float64) @ (np.asarray(codes).astype(np.float64) - 8).T    # exact: integer codes, fp16 w^
    s32 = (base.astype(np.float64) + np.ldexp(acc, -e[:, None])).astype(np.float32)
    return s32 if return_fp32 else s32.astype(np.float16)


def _ulp16(v):
    a = np.abs(np.asarray(v, np.float64)).astype(np.float16)
    return (np.nextafter(a, np.float16(np.inf)) - a).astype(np.float64)


def contract_error_bound(queries, codes, vmin, vdiff, coarse, lists):
    """Bound [nq, n] on |contract_scores - faiss_scores|."""
    q = _q32(queries).astype(np.float64)
    vmin64 = np.asarray(vmin, np.float64)
    vdiff64 = np.asarray(vdiff, np.float64)
    w, e = query_operand(queries, vdiff)
    scale = np.ldexp(1.0, -e)[:, None]
    # w^ rounding (half an fp16 ulp of each, times a code <= 15) and the two fp32 roundings inside it
    w_err = scale * (LEVELS * 0.5 * _ulp16(w)).sum(1, keepdims=True) + LEVELS * (np.abs(q) * vdiff64 / LEVELS).sum(
        1, keepdims=True) * 3 * U
    c_abs = (np.abs(q) * (np.abs(vmin64) + vdiff64)).sum(1, keepdims=True)
    t_abs = np.abs(q) @ np.abs(np.asarray(coarse, np.float64)).T
    n_terms = q.shape[1] + 3
    sum_err = n_terms * U * (c_abs + t_abs[:, np.asarray(lists).astype(np.int64)])
    contract32 = contract_scores(queries, codes, vmin, vdiff, coarse, lists, return_fp32=True).astype(np.float64)
    return w_err + sum_err + 2 * U * np.abs(contract32) + 0.5 * _ulp16(contract32)
