"""Thin torch-tensor wrappers over the C ABI (`include/atlas_b200.h`).

torch owns the device memory and the stream; the arithmetic happens in `lib/libatlas_b200.so`.
Nothing here falls back to torch ops: a missing library or a CPU tensor raises.
"""
import ctypes
import os

import torch

from . import _lib
from ._lib import AtlasB200Error, check, current_stream_ptr, lib, require_cuda

DIM = _lib.EMBEDDINGS_DIM


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


class Workspace:
    """Grow-only device scratch buffer reused across calls (kernels borrow it per launch)."""

    def __init__(self):
        self.buf = None

    def get(self, nbytes, device):
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            self.buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        return self.buf


_default_ws = Workspace()
_wgrad_ws = Workspace()


def _check_bank(bank):
    require_cuda(bank, "bank")
    if bank.dim() != 2 or bank.shape[1] != DIM or bank.stride(1) != 1:
        raise AtlasB200Error(f"bank must be [n, {DIM}] with unit inner stride, got {tuple(bank.shape)} {bank.stride()}")
    if bank.dtype not in (torch.float16, torch.bfloat16):
        raise AtlasB200Error("bank must be fp16 (reference dtype, src/index.py:51) or bf16")
    return 1 if bank.dtype == torch.bfloat16 else 0


def cast_queries(queries, dtype):
    """`allqueries.half()` (src/index.py:117) on the device through the library's cast kernel."""
    require_cuda(queries, "queries")
    if queries.dtype == dtype:
        return queries.contiguous()
    q32 = queries.float().contiguous()
    out = torch.empty(q32.shape, dtype=dtype, device=q32.device)
    check(lib().atlas_b200_cast_f32(_ptr(q32), _ptr(out), q32.numel(), 1 if dtype == torch.bfloat16 else 0,
                                    current_stream_ptr()))
    return out


def mips_topk(bank, queries, k, id_base=0, id_stride=1, workspace=None, exhaustive=False):
    """Exact top-k inner-product search of `queries` [nq, 768] in `bank` [n, 768] (one shard).

    Returns (scores [nq,k] bank dtype desc, ids [nq,k] int64, status int32[1] device tensor).
    `status != 0` means the fast path overflowed and the caller must retry with exhaustive=True
    (see `search_shard`, which does that)."""
    is_bf16 = _check_bank(bank)
    n = bank.shape[0]
    q = cast_queries(queries.reshape(-1, DIM), bank.dtype)
    nq = q.shape[0]
    ws = workspace or _default_ws
    nbytes = lib().atlas_b200_mips_workspace_bytes(n, nq, k)
    buf = ws.get(nbytes, bank.device)
    out_s = torch.empty((nq, k), dtype=bank.dtype, device=bank.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=bank.device)
    status = torch.zeros(1, dtype=torch.int32, device=bank.device)
    if exhaustive:
        check(lib().atlas_b200_mips_topk_exhaustive(
            _ptr(bank), n, bank.stride(0), is_bf16, _ptr(q), nq, k, _ptr(out_s), _ptr(out_i), id_base, id_stride,
            _ptr(buf), buf.numel(), current_stream_ptr()))
    else:
        check(lib().atlas_b200_mips_topk(
            _ptr(bank), n, bank.stride(0), is_bf16, _ptr(q), nq, k, _ptr(out_s), _ptr(out_i), id_base, id_stride,
            _ptr(status), _ptr(buf), buf.numel(), current_stream_ptr()))
    return out_s, out_i, status


def search_shard(bank, queries, k, id_base=0, id_stride=1, workspace=None):
    """mips_topk + the overflow fallback (one host sync to read the status word)."""
    s, i, status = mips_topk(bank, queries, k, id_base, id_stride, workspace)
    if queries.numel() and int(status.item()) != 0:
        s, i, _ = mips_topk(bank, queries, k, id_base, id_stride, workspace, exhaustive=True)
    return s, i


def topk_merge(scores_in, ids_in, world, nq_total, k, q_begin, nq_out, stride_s=None, stride_i=None):
    """Merge W per-shard lists [W, nq_total, k] -> rows [q_begin, q_begin+nq_out) merged [nq_out, k]."""
    require_cuda(scores_in, "scores_in")
    out_s = torch.empty((nq_out, k), dtype=scores_in.dtype, device=scores_in.device)
    out_i = torch.empty((nq_out, k), dtype=torch.int64, device=scores_in.device)
    ss = nq_total * k if stride_s is None else stride_s
    si = nq_total * k if stride_i is None else stride_i
    check(lib().atlas_b200_topk_merge(_ptr(scores_in), _ptr(ids_in), ss, si,
                                      1 if scores_in.dtype == torch.bfloat16 else 0, world, nq_total, k, q_begin,
                                      nq_out, _ptr(out_s), _ptr(out_i), current_stream_ptr()))
    return out_s, out_i


def search_host(bank, queries_host, k, id_base=0, id_stride=1, workspace=None):
    """The C-ABI end-to-end call with HOST buffers (H2D + cast + scan + select + D2H, synchronous).

    queries_host: CPU float32 tensor [nq, 768] (pinned or pageable).  Returns CPU tensors
    (scores float32 [nq,k] holding the 16-bit values, ids int64 [nq,k])."""
    is_bf16 = _check_bank(bank)
    if queries_host.is_cuda or queries_host.dtype != torch.float32:
        raise AtlasB200Error("search_host takes a CPU float32 query tensor")
    qh = queries_host.reshape(-1, DIM).contiguous()
    nq = qh.shape[0]
    n = bank.shape[0]
    ws = workspace or _default_ws
    nbytes = lib().atlas_b200_mips_workspace_bytes(n, nq, k)
    buf = ws.get(nbytes, bank.device)
    out_s = torch.empty((nq, k), dtype=torch.float32).pin_memory()
    out_i = torch.empty((nq, k), dtype=torch.int64).pin_memory()
    check(lib().atlas_b200_search_host(_ptr(bank), n, bank.stride(0), is_bf16, _ptr(qh), nq, k, _ptr(out_s),
                                       _ptr(out_i), id_base, id_stride, _ptr(buf), buf.numel(),
                                       current_stream_ptr()))
    return out_s, out_i


def pack_results(scores, ids, status=None):
    """One contiguous byte blob [scores (16-bit) | pad to 8 | ids (int64) | status (int64)] so that a SINGLE all-gather
    ships both lists AND the shard's overflow flag (replaces the 2*W gathers of src/index.py:138-141; the flag lets every
    rank learn, at the host sync it has anyway, whether any shard must be re-run exhaustively).
    Returns (blob uint8, ids offset, status offset)."""
    nbytes_s = scores.numel() * 2
    ids_off = (nbytes_s + 7) // 8 * 8
    st_off = ids_off + ids.numel() * 8
    blob = torch.empty(st_off + 8, dtype=torch.uint8, device=scores.device)
    blob[:nbytes_s].view(scores.dtype).copy_(scores.reshape(-1))
    blob[ids_off:st_off].view(torch.int64).copy_(ids.reshape(-1))
    if status is None:
        blob[st_off:].zero_()
    else:
        blob[st_off:].view(torch.int64).copy_(status.reshape(1))
    return blob, ids_off, st_off


def topk_merge_blob(blob_all, ids_off, world, nq_total, k, q_begin, nq_out, dtype):
    """Merge directly out of the all-gathered blobs `[W, blob_bytes]` (see pack_results)."""
    require_cuda(blob_all, "blob_all")
    blob_bytes = blob_all.shape[1]
    assert blob_bytes % 8 == 0 and blob_all.is_contiguous()
    out_s = torch.empty((nq_out, k), dtype=dtype, device=blob_all.device)
    out_i = torch.empty((nq_out, k), dtype=torch.int64, device=blob_all.device)
    base = blob_all.data_ptr()
    check(lib().atlas_b200_topk_merge(ctypes.c_void_p(base), ctypes.c_void_p(base + ids_off), blob_bytes // 2,
                                      blob_bytes // 8, 1 if dtype == torch.bfloat16 else 0, world, nq_total, k,
                                      q_begin, nq_out, _ptr(out_s), _ptr(out_i), current_stream_ptr()))
    return out_s, out_i


# ---------------------------------------------------------------------------------------------
# product-quantized index (csrc/pq.cu)
# ---------------------------------------------------------------------------------------------
PQ_OP_TRAIN, PQ_OP_ENCODE, PQ_OP_SEARCH, PQ_OP_SEARCH_PROBED = 0, 1, 2, 3
PQ_KSUB = 256
PQ_ITERS = 25   # faiss's k-means default


def pq_check_code_size(code_size):
    """code_size M: sub-quantizers of 8 bits; M must divide 768 with 768 / M >= 8."""
    if not isinstance(code_size, int) or code_size < 1 or DIM % code_size or DIM // code_size < 8:
        ok = [m for m in range(1, DIM + 1) if DIM % m == 0 and DIM // m >= 8]
        raise AtlasB200Error(f"code_size={code_size!r} is not supported: it must divide {DIM} into sub-vectors of at "
                             f"least 8 dimensions, one of {ok}")


def pq_list_dtype(n_list):
    """Storage type of the list ids: uint16 while every id fits, else int32."""
    return torch.uint16 if n_list <= 65535 else torch.int32


def pq_train(sample, code_size, n_list, iters=PQ_ITERS):
    """k-means on the device (atlas_b200_pq_train).  sample: CUDA fp16 [S, 768], rows in a seeded random order.
    Returns (codebooks fp32 [M, 256, 768 / M], coarse centroids fp32 [n_list, 768] or None)."""
    require_cuda(sample, "sample")
    pq_check_code_size(code_size)
    s = sample.reshape(-1, DIM).to(torch.float16).contiguous()
    dev = s.device
    cb = torch.empty((code_size, PQ_KSUB, DIM // code_size), dtype=torch.float32, device=dev)
    coarse = torch.empty((n_list, DIM), dtype=torch.float32, device=dev) if n_list else None
    ws = torch.empty(int(lib().atlas_b200_pq_workspace_bytes(PQ_OP_TRAIN, s.shape[0], code_size, n_list, 1)),
                     dtype=torch.uint8, device=dev)
    check(lib().atlas_b200_pq_train(_ptr(s), s.shape[0], code_size, n_list, iters, _ptr(cb),
                                    _ptr(coarse) if coarse is not None else None, _ptr(ws), ws.numel(),
                                    current_stream_ptr()))
    return cb, coarse


def pq_encode(rows, codebooks, coarse, codes, list_ids=None, workspace=None):
    """Codes (and list ids) of CUDA fp16 rows [n, 768] into `codes` uint8 [n, M] (and `list_ids` [n])."""
    require_cuda(rows, "rows")
    r = rows.reshape(-1, DIM)
    if r.dtype != torch.float16 or not r.is_contiguous():
        raise AtlasB200Error("pq_encode: rows must be contiguous fp16 [n, 768]")
    M = codebooks.shape[0]
    n_list = 0 if coarse is None else coarse.shape[0]
    if codes.shape != (r.shape[0], M) or codes.dtype != torch.uint8 or (n_list and list_ids is None):
        raise AtlasB200Error("pq_encode: codes must be uint8 [n, M] (and list ids are needed with a coarse quantizer)")
    buf = (workspace or _default_ws).get(lib().atlas_b200_pq_workspace_bytes(PQ_OP_ENCODE, r.shape[0], M, n_list, 1),
                                         r.device)
    check(lib().atlas_b200_pq_encode(_ptr(r), r.shape[0], M, _ptr(codebooks), _ptr(coarse) if n_list else None, n_list,
                                     _ptr(codes), _ptr(list_ids) if n_list else None, _ptr(buf), buf.numel(),
                                     current_stream_ptr()))
    return codes, list_ids


def check_nprobe(nprobe):
    """nprobe: None (every list) or an int >= 1 (not a bool)."""
    if nprobe is not None and (isinstance(nprobe, bool) or not isinstance(nprobe, int) or nprobe < 1):
        raise AtlasB200Error(f"nprobe={nprobe!r} must be None (every list) or an integer >= 1")
    return nprobe


def _probed(nprobe, n_list, what):
    """True when a search with `nprobe` scans only some lists (nprobe < n_list); None / >= n_list is the full scan."""
    check_nprobe(nprobe)
    if nprobe is not None and n_list == 0:
        raise AtlasB200Error(f"{what}: nprobe={nprobe} needs inverted lists (index type pq has none)")
    return nprobe is not None and nprobe < n_list


def _check_table(t, name, shape):
    require_cuda(t, name)
    if t.dtype != torch.int32 or tuple(t.shape) != shape or not t.is_contiguous():
        raise AtlasB200Error(f"{name} must be contiguous int32 {list(shape)}, got {t.dtype} {tuple(t.shape)}")


def ivfpq_list_tables(list_ids, n_list):
    """The list tables of a probed ivfpq search: (list_order int32 [n], the rows sorted by list id, stable;
    list_offsets int32 [n_list + 1], list l holding list_order[list_offsets[l]:list_offsets[l + 1]])."""
    lists = list_ids.to(torch.int64)
    order = torch.sort(lists, stable=True).indices.to(torch.int32)
    offsets = torch.zeros(n_list + 1, dtype=torch.int64, device=lists.device)
    offsets[1:] = torch.cumsum(torch.bincount(lists, minlength=n_list), 0)
    return order, offsets.to(torch.int32)


def pq_topk(codes, list_ids, codebooks, coarse, queries, k, id_base=0, id_stride=1, workspace=None, exhaustive=False,
            nprobe=None, list_order=None, list_offsets=None):
    """Top-k of the PQ / IVF-PQ scores of `queries` [nq, 768] over one shard's codes (atlas_b200_pq_topk).

    Returns (scores [nq, k] fp16 desc, ids [nq, k] int64, status int32[1] device tensor) like `mips_topk`.
    nprobe < n_list (ivfpq): only the rows of each query's best lists (atlas_b200_pq_topk_probed), with the tables of
    `ivfpq_list_tables`; None or >= n_list scans every row.  The probed search does not synchronise with the host when
    the tables are passed; built here (when not given) they cost a host synchronisation (torch.bincount) per call."""
    require_cuda(codes, "codes")
    n, M = codes.shape
    n_list = 0 if coarse is None else coarse.shape[0]
    probed = _probed(nprobe, n_list, "pq_topk")
    q = cast_queries(queries.reshape(-1, DIM).to(codes.device), torch.float16)
    nq = q.shape[0]
    op = PQ_OP_SEARCH_PROBED if probed else PQ_OP_SEARCH
    buf = (workspace or _default_ws).get(lib().atlas_b200_pq_workspace_bytes(op, n, M, n_list, k), codes.device)
    out_s = torch.empty((nq, k), dtype=torch.float16, device=codes.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=codes.device)
    status = torch.zeros(1, dtype=torch.int32, device=codes.device)
    lp = _ptr(list_ids) if n_list else None
    cp = _ptr(coarse) if n_list else None
    if probed:
        if list_order is None or list_offsets is None:
            list_order, list_offsets = ivfpq_list_tables(list_ids, n_list)
        _check_table(list_order, "list_order", (n,))
        _check_table(list_offsets, "list_offsets", (n_list + 1,))
        args = (_ptr(codes), lp, n, M, _ptr(codebooks), cp, n_list, _ptr(list_order), _ptr(list_offsets), nprobe, _ptr(q),
                nq, k, _ptr(out_s), _ptr(out_i), id_base, id_stride)
        if exhaustive:
            check(lib().atlas_b200_pq_topk_probed_exhaustive(*args, _ptr(buf), buf.numel(), current_stream_ptr()))
        else:
            check(lib().atlas_b200_pq_topk_probed(*args, _ptr(status), _ptr(buf), buf.numel(), current_stream_ptr()))
        return out_s, out_i, status
    if exhaustive:
        check(lib().atlas_b200_pq_topk_exhaustive(_ptr(codes), lp, n, M, _ptr(codebooks), cp, n_list, _ptr(q), nq, k,
                                                  _ptr(out_s), _ptr(out_i), id_base, id_stride, _ptr(buf), buf.numel(),
                                                  current_stream_ptr()))
    else:
        check(lib().atlas_b200_pq_topk(_ptr(codes), lp, n, M, _ptr(codebooks), cp, n_list, _ptr(q), nq, k, _ptr(out_s),
                                       _ptr(out_i), id_base, id_stride, _ptr(status), _ptr(buf), buf.numel(),
                                       current_stream_ptr()))
    return out_s, out_i, status


def pq_refine_topk(rows_host, queries, cand_local, k, id_base=0, id_stride=1, workspace=None):
    """Exact re-ranking of PQ candidates (atlas_b200_pq_refine_topk, faiss IndexRefineFlat).

    rows_host: PINNED CPU fp16 [n, 768] (the index's host rows), read zero-copy by the kernel; queries: [nq, 768], moved
    to cand_local's device and rounded to fp16 like `pq_topk`; cand_local: CUDA int64 [nq, k'] local row numbers
    (`pq_topk(..., k', 0, 1)`), distinct within a row; entries outside [0, n) are skipped.
    Returns (scores fp16 [nq, k] desc, ids int64 [nq, k] = id_base + id_stride * row) as CUDA tensors: the top k of the
    candidates by their exact inner product, accumulated in fp32 and rounded once to fp16."""
    if rows_host.is_cuda or rows_host.dtype != torch.float16 or rows_host.dim() != 2 or rows_host.shape[1] != DIM \
            or not rows_host.is_contiguous():
        raise AtlasB200Error(f"pq_refine_topk: rows_host must be a contiguous CPU fp16 [n, {DIM}] tensor, got "
                             f"{rows_host.dtype} {tuple(rows_host.shape)} on {rows_host.device}")
    if not rows_host.is_pinned():
        raise AtlasB200Error("pq_refine_topk: rows_host must be pinned host memory (tensor.pin_memory()): the kernel "
                             "reads it over the host link")
    require_cuda(cand_local, "cand_local")
    q = cast_queries(queries.reshape(-1, DIM).to(cand_local.device), torch.float16)
    nq = q.shape[0]
    if cand_local.dtype != torch.int64 or cand_local.dim() != 2 or cand_local.shape[0] != nq:
        raise AtlasB200Error(f"pq_refine_topk: cand_local must be int64 [nq={nq}, k'], got {cand_local.dtype} "
                             f"{tuple(cand_local.shape)}")
    cand = cand_local.contiguous()
    k_cand = cand.shape[1]
    if not 1 <= k <= k_cand:
        raise AtlasB200Error(f"pq_refine_topk: need 1 <= k <= k' (k={k}, k'={k_cand})")
    if k_cand > _lib.MAX_TOPK:
        raise AtlasB200Error(f"pq_refine_topk: k'={k_cand} candidates exceed MAX_TOPK={_lib.MAX_TOPK}")
    dev = q.device
    out_s = torch.empty((nq, k), dtype=torch.float16, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    if nq == 0:
        return out_s, out_i
    buf = (workspace or _default_ws).get(lib().atlas_b200_pq_refine_workspace_bytes(nq, k_cand), dev)
    check(lib().atlas_b200_pq_refine_topk(_ptr(rows_host), rows_host.shape[0], _ptr(q), nq, _ptr(cand), k_cand, k,
                                          _ptr(out_s), _ptr(out_i), id_base, id_stride, _ptr(buf), buf.numel(),
                                          current_stream_ptr()))
    return out_s, out_i


# ---------------------------------------------------------------------------------------------
# IVF-SQ index (csrc/pq.cu, csrc/ivfsq.cu)
# ---------------------------------------------------------------------------------------------
SQ_BITS = 4
SQ_CODE_BYTES = DIM * SQ_BITS // 8
SQ_TILE = 64                # slots per tile: every tile belongs to one inverted list
SQ_RANGE_MAX = 100000       # faiss ScalarQuantizer::train_residual's subsample
_SQ_CHUNK = 65536           # rows per step of the layout conversions


def sq_nibble_of_dim():
    """Nibble position (2 * byte + high) of every dim inside a device slot (csrc/ivfsq.cuh's permutation), int64 [768]."""
    d = torch.arange(DIM)
    kb, s, c = d // 64, (d % 64) // 16, d % 16
    j, e, hi = (c % 8) // 2, c % 2, c // 8
    byte = kb * 32 + j * 8 + (s // 2) * 4 + (s % 2) + 2 * e
    return 2 * byte + hi


def _sq_check_state(coarse, vmin, vdiff):
    for name, t in (("coarse", coarse), ("vmin", vmin), ("vdiff", vdiff)):
        require_cuda(t, name)
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise AtlasB200Error(f"ivfsq: {name} must be contiguous fp32")
    if coarse.dim() != 2 or coarse.shape[1] != DIM or coarse.shape[0] < 1 or vmin.shape != (DIM,) or vdiff.shape != (DIM,):
        raise AtlasB200Error(f"ivfsq: coarse must be [n_list >= 1, {DIM}] and vmin / vdiff [{DIM}], got "
                             f"{tuple(coarse.shape)}, {tuple(vmin.shape)}, {tuple(vdiff.shape)}")
    return coarse.shape[0]


def ivfsq_train(sample, n_list, iters=PQ_ITERS):
    """Coarse k-means + per-dim residual ranges on the device (atlas_b200_ivfsq_train).  sample: CUDA fp16 [S, 768] in a
    seeded random order, S >= n_list.  Returns (coarse fp32 [n_list, 768], vmin fp32 [768], vdiff fp32 [768])."""
    require_cuda(sample, "sample")
    s = sample.reshape(-1, DIM).to(torch.float16).contiguous()
    if n_list < 1 or s.shape[0] < n_list:
        raise AtlasB200Error(f"ivfsq_train: need 1 <= n_list <= sample rows (n_list={n_list}, rows={s.shape[0]})")
    dev = s.device
    coarse = torch.empty((n_list, DIM), dtype=torch.float32, device=dev)
    vmin = torch.empty(DIM, dtype=torch.float32, device=dev)
    vdiff = torch.empty(DIM, dtype=torch.float32, device=dev)
    ws = torch.empty(int(lib().atlas_b200_ivfsq_workspace_bytes(PQ_OP_TRAIN, s.shape[0], n_list, 1)), dtype=torch.uint8,
                     device=dev)
    check(lib().atlas_b200_ivfsq_train(_ptr(s), s.shape[0], n_list, iters, _ptr(coarse), _ptr(vmin), _ptr(vdiff), _ptr(ws),
                                       ws.numel(), current_stream_ptr()))
    return coarse, vmin, vdiff


def ivfsq_encode(rows, coarse, vmin, vdiff, list_ids=None, row_slot=None, codes=None, workspace=None):
    """For CUDA fp16 rows [n, 768]: the coarse list of each row into `list_ids` (int32 [n]) and/or its 384 code bytes
    into slot `row_slot[i]` (int32 [n]) of `codes` (uint8 [slots, 384], the device layout)."""
    require_cuda(rows, "rows")
    r = rows.reshape(-1, DIM)
    if r.dtype != torch.float16 or not r.is_contiguous():
        raise AtlasB200Error("ivfsq_encode: rows must be contiguous fp16 [n, 768]")
    n_list = _sq_check_state(coarse, vmin, vdiff)
    n = r.shape[0]
    if list_ids is None and codes is None:
        raise AtlasB200Error("ivfsq_encode: pass list_ids and/or codes")
    if list_ids is not None and (list_ids.dtype != torch.int32 or list_ids.shape != (n,) or not list_ids.is_contiguous()):
        raise AtlasB200Error(f"ivfsq_encode: list_ids must be contiguous int32 [{n}]")
    if codes is not None:
        if codes.dtype != torch.uint8 or codes.dim() != 2 or codes.shape[1] != SQ_CODE_BYTES or not codes.is_contiguous():
            raise AtlasB200Error(f"ivfsq_encode: codes must be contiguous uint8 [slots, {SQ_CODE_BYTES}]")
        if row_slot is None or row_slot.dtype != torch.int32 or row_slot.shape != (n,) or not row_slot.is_contiguous():
            raise AtlasB200Error(f"ivfsq_encode: codes need row_slot, contiguous int32 [{n}]")
    buf = (workspace or _default_ws).get(lib().atlas_b200_ivfsq_workspace_bytes(PQ_OP_ENCODE, n, n_list, 1), r.device)
    check(lib().atlas_b200_ivfsq_encode(_ptr(r), n, _ptr(coarse), n_list, _ptr(vmin), _ptr(vdiff),
                                        None if list_ids is None else _ptr(list_ids),
                                        None if codes is None else _ptr(row_slot), None if codes is None else _ptr(codes),
                                        _ptr(buf), buf.numel(), current_stream_ptr()))


def ivfsq_layout(list_ids, n_list):
    """The inverted-list slot layout of rows with list ids `list_ids` [n]: rows stable-sorted by list, each list padded
    to a multiple of SQ_TILE slots.  Returns (slot_rows int32 [slots] (-1 = padding), tile_lists int32 [slots / 64],
    row_slot int32 [n])."""
    lists = list_ids.to(torch.int64)
    dev, n = lists.device, lists.numel()
    if n and (int(lists.min()) < 0 or int(lists.max()) >= n_list):
        raise AtlasB200Error(f"ivfsq_layout: list ids must lie in [0, {n_list})")
    counts = torch.bincount(lists, minlength=n_list)
    padded = (counts + SQ_TILE - 1) // SQ_TILE * SQ_TILE
    start = torch.cumsum(padded, 0) - padded
    first = torch.cumsum(counts, 0) - counts
    order = torch.sort(lists, stable=True).indices
    ls = lists[order]
    slot = start[ls] + torch.arange(n, device=dev) - first[ls]
    n_slots = int(padded.sum())
    slot_rows = torch.full((n_slots,), -1, dtype=torch.int32, device=dev)
    slot_rows[slot] = order.to(torch.int32)
    row_slot = torch.empty(n, dtype=torch.int32, device=dev)
    row_slot[order] = slot.to(torch.int32)
    tile_lists = torch.repeat_interleave(torch.arange(n_list, dtype=torch.int32, device=dev), padded // SQ_TILE)
    return slot_rows, tile_lists, row_slot


def ivfsq_export(codes, slot_rows, tile_lists, n_rows):
    """Device layout -> row order: (codes uint8 [n_rows, 384] in faiss's packing - dim 2j in the low nibble of byte j,
    dim 2j + 1 in the high one - and list ids int32 [n_rows])."""
    dev = codes.device
    perm = sq_nibble_of_dim().to(dev)
    out = torch.empty((n_rows, SQ_CODE_BYTES), dtype=torch.uint8, device=dev)
    lists = torch.empty(n_rows, dtype=torch.int32, device=dev)
    slots = torch.nonzero(slot_rows >= 0).flatten()
    if slots.numel() != n_rows:
        raise AtlasB200Error(f"ivfsq_export: {slots.numel()} real slots for {n_rows} rows")
    for a in range(0, n_rows, _SQ_CHUNK):
        sl = slots[a:a + _SQ_CHUNK]
        c = codes[sl]
        nib = torch.stack([c & 15, c >> 4], dim=2).reshape(-1, 2 * SQ_CODE_BYTES)[:, perm]     # [rows, 768] by dim
        rows = slot_rows[sl].to(torch.int64)
        out[rows] = nib[:, 0::2] | (nib[:, 1::2] << 4)
        lists[rows] = tile_lists[sl // SQ_TILE]
    return out, lists


def ivfsq_import(codes_rows, list_ids, n_list):
    """Row order (ivfsq_export's format) -> device layout: (codes, slot_rows, tile_lists)."""
    dev = codes_rows.device
    n = codes_rows.shape[0]
    if codes_rows.dtype != torch.uint8 or codes_rows.shape != (n, SQ_CODE_BYTES) or list_ids.shape != (n,):
        raise AtlasB200Error(f"ivfsq_import: codes must be uint8 [n, {SQ_CODE_BYTES}] and list ids [n]")
    slot_rows, tile_lists, row_slot = ivfsq_layout(list_ids, n_list)
    perm = sq_nibble_of_dim().to(dev)
    codes = torch.zeros((slot_rows.numel(), SQ_CODE_BYTES), dtype=torch.uint8, device=dev)
    for a in range(0, n, _SQ_CHUNK):
        c = codes_rows[a:a + _SQ_CHUNK]
        by_dim = torch.stack([c & 15, c >> 4], dim=2).reshape(-1, DIM)
        nib = torch.empty_like(by_dim)
        nib[:, perm] = by_dim
        codes[row_slot[a:a + _SQ_CHUNK].to(torch.int64)] = nib[:, 0::2] | (nib[:, 1::2] << 4)
    return codes, slot_rows, tile_lists


def ivfsq_list_tables(slot_rows, tile_lists, n_list):
    """The list tables of a probed ivfsq search: (list_tile_off int32 [n_list + 1], list l owning tiles
    list_tile_off[l]:list_tile_off[l + 1]; list_rows int32 [n_list], its real rows)."""
    tl = tile_lists.to(torch.int64)
    off = torch.zeros(n_list + 1, dtype=torch.int64, device=tl.device)
    off[1:] = torch.cumsum(torch.bincount(tl, minlength=n_list), 0)
    real = (slot_rows.reshape(-1, SQ_TILE) >= 0).sum(1)
    rows = torch.zeros(n_list, dtype=torch.int64, device=tl.device).index_add_(0, tl, real)
    return off.to(torch.int32), rows.to(torch.int32)


def ivfsq_topk(codes, slot_rows, tile_lists, n_rows, coarse, vmin, vdiff, queries, k, id_base=0, id_stride=1,
               workspace=None, exhaustive=False, nprobe=None, list_tile_off=None, list_rows=None):
    """Top-k of the IVF-SQ scores of `queries` [nq, 768] over one shard's rows in the device layout
    (atlas_b200_ivfsq_topk).  Returns (scores [nq, k] fp16 desc, ids [nq, k] int64, status int32[1]) like `mips_topk`.
    nprobe < n_list: only the rows of each query's best lists (atlas_b200_ivfsq_topk_probed), with the tables of
    `ivfsq_list_tables`; None or >= n_list scans every slot.  The probed search does not synchronise with the host when
    the tables are passed; built here (when not given) they cost a host synchronisation (torch.bincount) per call."""
    require_cuda(codes, "codes")
    n_list = _sq_check_state(coarse, vmin, vdiff)
    probed = _probed(nprobe, n_list, "ivfsq_topk")
    if codes.dtype != torch.uint8 or codes.dim() != 2 or codes.shape[1] != SQ_CODE_BYTES or not codes.is_contiguous() \
            or codes.shape[0] % SQ_TILE or codes.data_ptr() % 16:
        raise AtlasB200Error(f"ivfsq_topk: codes must be contiguous, 16-byte aligned uint8 [64 * tiles, {SQ_CODE_BYTES}]")
    n_tiles = codes.shape[0] // SQ_TILE
    if slot_rows.dtype != torch.int32 or slot_rows.shape != (codes.shape[0],) or tile_lists.dtype != torch.int32 \
            or tile_lists.shape != (n_tiles,):
        raise AtlasB200Error("ivfsq_topk: slot_rows must be int32 [slots] and tile_lists int32 [tiles]")
    q = cast_queries(queries.reshape(-1, DIM).to(codes.device), torch.float16)
    nq = q.shape[0]
    op = PQ_OP_SEARCH_PROBED if probed else PQ_OP_SEARCH
    buf = (workspace or _default_ws).get(lib().atlas_b200_ivfsq_workspace_bytes(op, codes.shape[0], n_list, k), codes.device)
    out_s = torch.empty((nq, k), dtype=torch.float16, device=codes.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=codes.device)
    status = torch.zeros(1, dtype=torch.int32, device=codes.device)
    if probed:
        if list_tile_off is None or list_rows is None:
            list_tile_off, list_rows = ivfsq_list_tables(slot_rows, tile_lists, n_list)
        _check_table(list_tile_off, "list_tile_off", (n_list + 1,))
        _check_table(list_rows, "list_rows", (n_list,))
        args = (_ptr(codes), _ptr(slot_rows.contiguous()), _ptr(tile_lists.contiguous()), n_tiles, n_rows,
                _ptr(list_tile_off), _ptr(list_rows), _ptr(coarse), n_list, _ptr(vmin), _ptr(vdiff), nprobe, _ptr(q), nq, k,
                _ptr(out_s), _ptr(out_i), id_base, id_stride)
        if exhaustive:
            check(lib().atlas_b200_ivfsq_topk_probed_exhaustive(*args, _ptr(buf), buf.numel(), current_stream_ptr()))
        else:
            check(lib().atlas_b200_ivfsq_topk_probed(*args, _ptr(status), _ptr(buf), buf.numel(), current_stream_ptr()))
        return out_s, out_i, status
    args = (_ptr(codes), _ptr(slot_rows.contiguous()), _ptr(tile_lists.contiguous()), n_tiles, n_rows, _ptr(coarse),
            n_list, _ptr(vmin), _ptr(vdiff), _ptr(q), nq, k, _ptr(out_s), _ptr(out_i), id_base, id_stride)
    if exhaustive:
        check(lib().atlas_b200_ivfsq_topk_exhaustive(*args, _ptr(buf), buf.numel(), current_stream_ptr()))
    else:
        check(lib().atlas_b200_ivfsq_topk(*args, _ptr(status), _ptr(buf), buf.numel(), current_stream_ptr()))
    return out_s, out_i, status


# ---------------------------------------------------------------------------------------------
# IVF-Flat index (csrc/pq.cu, csrc/ivfflat.cu): ivfsq's slot layout with fp16 rows in place of codes
# ---------------------------------------------------------------------------------------------
def ivfflat_train(sample, n_list, iters=PQ_ITERS):
    """The coarse quantizer alone (atlas_b200_ivfsq_train with vmin = vdiff = NULL): bit-identical to the ivfpq / ivfsq
    one on the same sample.  sample: CUDA fp16 [S, 768] in a seeded random order, S >= n_list.  Returns fp32 [n_list, 768]."""
    require_cuda(sample, "sample")
    s = sample.reshape(-1, DIM).to(torch.float16).contiguous()
    if n_list < 1 or s.shape[0] < n_list:
        raise AtlasB200Error(f"ivfflat_train: need 1 <= n_list <= sample rows (n_list={n_list}, rows={s.shape[0]})")
    coarse = torch.empty((n_list, DIM), dtype=torch.float32, device=s.device)
    ws = torch.empty(int(lib().atlas_b200_ivfsq_workspace_bytes(PQ_OP_TRAIN, s.shape[0], n_list, 1)), dtype=torch.uint8,
                     device=s.device)
    check(lib().atlas_b200_ivfsq_train(_ptr(s), s.shape[0], n_list, iters, _ptr(coarse), None, None, _ptr(ws), ws.numel(),
                                       current_stream_ptr()))
    return coarse


def ivf_list_ids(rows, coarse, list_ids, workspace=None):
    """The coarse list (inner product, lowest list on ties) of every CUDA fp16 row [n, 768] into `list_ids` int32 [n]
    (atlas_b200_ivfsq_encode without codes)."""
    require_cuda(rows, "rows")
    require_cuda(coarse, "coarse")
    r = rows.reshape(-1, DIM)
    n = r.shape[0]
    if r.dtype != torch.float16 or not r.is_contiguous():
        raise AtlasB200Error("ivf_list_ids: rows must be contiguous fp16 [n, 768]")
    if coarse.dtype != torch.float32 or coarse.dim() != 2 or coarse.shape[1] != DIM or not coarse.is_contiguous():
        raise AtlasB200Error(f"ivf_list_ids: coarse must be contiguous fp32 [n_list, {DIM}]")
    if list_ids.dtype != torch.int32 or list_ids.shape != (n,) or not list_ids.is_contiguous():
        raise AtlasB200Error(f"ivf_list_ids: list_ids must be contiguous int32 [{n}]")
    n_list = coarse.shape[0]
    buf = (workspace or _default_ws).get(lib().atlas_b200_ivfsq_workspace_bytes(PQ_OP_ENCODE, n, n_list, 1), r.device)
    check(lib().atlas_b200_ivfsq_encode(_ptr(r), n, _ptr(coarse), n_list, None, None, _ptr(list_ids), None, None, _ptr(buf),
                                        buf.numel(), current_stream_ptr()))
    return list_ids


def ivfflat_topk(rows, slot_rows, tile_lists, n_rows, coarse, queries, k, id_base=0, id_stride=1, workspace=None,
                 exhaustive=False, nprobe=None, list_tile_off=None, list_rows=None):
    """Top-k of the exact inner products (the flat index's fp16 scores) of `queries` [nq, 768] over one shard's rows in
    the IVF-Flat slot layout (atlas_b200_ivfflat_topk): rows CUDA fp16 [64 * tiles, 768] (padding slots zero),
    slot_rows int32 [slots], tile_lists int32 [tiles] (`ivfsq_layout`).  Returns (scores [nq, k] fp16 desc, ids [nq, k]
    int64, status int32[1]) like `mips_topk`.
    coarse None is type flat: one list, always the full scan, and nprobe must be None.  nprobe < n_list: only the rows of
    each query's best lists, with the tables of `ivfsq_list_tables`; None or >= n_list scans every slot.  The probed
    search does not synchronise with the host when the tables are passed; built here (when not given) they cost a host
    synchronisation (torch.bincount) per call."""
    require_cuda(rows, "rows")
    check_nprobe(nprobe)
    if coarse is None:
        if nprobe is not None:
            raise AtlasB200Error(f"ivfflat_topk: nprobe={nprobe} needs inverted lists (index type flat has none)")
        n_list = 1
    else:
        require_cuda(coarse, "coarse")
        if coarse.dtype != torch.float32 or coarse.dim() != 2 or coarse.shape[1] != DIM or coarse.shape[0] < 1 \
                or not coarse.is_contiguous():
            raise AtlasB200Error(f"ivfflat_topk: coarse must be contiguous fp32 [n_list >= 1, {DIM}]")
        n_list = coarse.shape[0]
    probed = nprobe is not None and nprobe < n_list
    if rows.dtype != torch.float16 or rows.dim() != 2 or rows.shape[1] != DIM or not rows.is_contiguous() \
            or rows.shape[0] % SQ_TILE or rows.shape[0] == 0 or rows.data_ptr() % 16:
        raise AtlasB200Error(f"ivfflat_topk: rows must be contiguous, 16-byte aligned fp16 [64 * tiles, {DIM}]")
    n_tiles = rows.shape[0] // SQ_TILE
    if slot_rows.dtype != torch.int32 or slot_rows.shape != (rows.shape[0],) or tile_lists.dtype != torch.int32 \
            or tile_lists.shape != (n_tiles,):
        raise AtlasB200Error("ivfflat_topk: slot_rows must be int32 [slots] and tile_lists int32 [tiles]")
    q = cast_queries(queries.reshape(-1, DIM).to(rows.device), torch.float16)
    nq = q.shape[0]
    op = PQ_OP_SEARCH_PROBED if probed else PQ_OP_SEARCH
    buf = (workspace or _default_ws).get(lib().atlas_b200_ivfflat_workspace_bytes(op, rows.shape[0], n_list, k), rows.device)
    out_s = torch.empty((nq, k), dtype=torch.float16, device=rows.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=rows.device)
    status = torch.zeros(1, dtype=torch.int32, device=rows.device)
    lt = lr = None
    if probed:
        if list_tile_off is None or list_rows is None:
            list_tile_off, list_rows = ivfsq_list_tables(slot_rows, tile_lists, n_list)
        _check_table(list_tile_off, "list_tile_off", (n_list + 1,))
        _check_table(list_rows, "list_rows", (n_list,))
        lt, lr = _ptr(list_tile_off), _ptr(list_rows)
    args = (_ptr(rows), _ptr(slot_rows.contiguous()), n_tiles, n_rows, lt, lr, _ptr(coarse) if probed else None, n_list,
            nprobe if probed else 0, _ptr(q), nq, k, _ptr(out_s), _ptr(out_i), id_base, id_stride)
    if exhaustive:
        check(lib().atlas_b200_ivfflat_topk_exhaustive(*args, _ptr(buf), buf.numel(), current_stream_ptr()))
    else:
        check(lib().atlas_b200_ivfflat_topk(*args, _ptr(status), _ptr(buf), buf.numel(), current_stream_ptr()))
    return out_s, out_i, status


# ---------------------------------------------------------------------------------------------
# dense layers (csrc/gemm.cu)
# ---------------------------------------------------------------------------------------------
EPI_NONE, EPI_BIAS, EPI_GELU, EPI_RESIDUAL, EPI_GATED, EPI_RELU = 0, 1, 2, 3, 4, 5


def linear(x, weight, bias=None, residual=None, epilogue=None, out=None, row_ss=None, out_ss=None, rs_eps=1e-6, rows=None):
    """y = epilogue(x @ weight.T) on wgmma.  x [..., K], weight [N, K] (nn.Linear layout), 16-bit.

    epilogue: EPI_NONE / EPI_BIAS / EPI_GELU / EPI_RESIDUAL / EPI_GATED / EPI_RELU (see include/atlas_b200.h);
    default: EPI_RESIDUAL if `residual` is given, else EPI_BIAS if `bias` is given, else EPI_NONE.
    Fused T5 RMSNorm: `row_ss` fp32 [M] = sum of squares of the rows of x -> accumulator rows are
    scaled by rsqrt(row_ss / K + rs_eps) (x is the UN-normalised hidden state, the norm weight is folded into `weight`);
    `out_ss` fp32 [M] (pre-zeroed) receives the sum of squares of the stored output rows.
    `rows`: int32 [1] device tensor - only the first *rows rows are computed (static launch shape)."""
    require_cuda(x, "x")
    if x.dtype not in (torch.float16, torch.bfloat16) or weight.dtype != x.dtype:
        raise AtlasB200Error(f"linear: x and weight must both be fp16 or bf16 (got {x.dtype}, {weight.dtype})")
    K = x.shape[-1]
    N = weight.shape[0]
    if weight.shape[1] != K:
        raise AtlasB200Error(f"linear: weight {tuple(weight.shape)} does not match K={K}")
    x2 = x.reshape(-1, K)
    if x2.stride(-1) != 1:
        x2 = x2.contiguous()
    w = weight if weight.stride(-1) == 1 else weight.contiguous()
    M = x2.shape[0]
    if epilogue is None:
        epilogue = EPI_RESIDUAL if residual is not None else (EPI_BIAS if bias is not None else EPI_NONE)
    n_out = N // 2 if epilogue == EPI_GATED else N
    # the kernel reads these through raw pointers: a wrong dtype, length or layout would be read (or written) past its end
    if bias is not None and (bias.dtype != x.dtype or bias.device != x.device or not bias.is_contiguous()
                             or bias.numel() != N):
        raise AtlasB200Error(f"linear: bias must be a contiguous {x.dtype} tensor of {N} elements on {x.device} "
                             f"(got {bias.dtype} {tuple(bias.shape)} on {bias.device})")
    if out is None:
        out = torch.empty((M, n_out), dtype=x.dtype, device=x.device)
    elif (out.dtype != x.dtype or out.device != x.device or out.dim() != 2 or out.stride(-1) != 1
          or out.shape[0] < M or out.shape[1] < n_out):
        raise AtlasB200Error(f"linear: out must be a {x.dtype} [>= {M}, >= {n_out}] tensor on {x.device} with unit column "
                             f"stride (got {out.dtype} {tuple(out.shape)} stride {out.stride()} on {out.device})")
    r2 = None
    if residual is not None:
        r2 = residual.reshape(-1, residual.shape[-1])
        if r2.dtype != x.dtype or r2.device != x.device or tuple(r2.shape) != (M, N):
            raise AtlasB200Error(f"linear: residual must be a {x.dtype} [{M}, {N}] tensor on {x.device} "
                                 f"(got {residual.dtype} {tuple(residual.shape)} on {residual.device})")
        if r2.stride(-1) != 1:
            r2 = r2.contiguous()
    for t in (row_ss, out_ss):
        if t is not None and (t.dtype != torch.float32 or t.numel() != M or not t.is_contiguous() or not t.is_cuda):
            raise AtlasB200Error("linear: row_ss / out_ss must be contiguous CUDA fp32 tensors with one element per row")
    if rows is not None and (rows.dtype != torch.int32 or rows.numel() != 1 or rows.device != x.device):
        raise AtlasB200Error(f"linear: rows must be an int32 tensor of one element on {x.device} "
                             f"(got {rows.dtype} {tuple(rows.shape)} on {rows.device})")
    check(lib().atlas_b200_linear_rows(
        _ptr(x2), x2.stride(0), _ptr(w), w.stride(0), _ptr(bias) if bias is not None else None,
        _ptr(r2) if r2 is not None else None, r2.stride(0) if r2 is not None else 0, _ptr(out), out.stride(0),
        M, N, K, epilogue, 1 if x.dtype == torch.bfloat16 else 0, _ptr(row_ss) if row_ss is not None else None,
        _ptr(out_ss) if out_ss is not None else None, float(rs_eps), _ptr(rows) if rows is not None else None,
        current_stream_ptr()))
    return out[:M, :n_out].reshape(*x.shape[:-1], n_out)


# ---------------------------------------------------------------------------------------------
# normalisation / embedding / pooling (csrc/elementwise.cu) and attention (csrc/attention.cu)
# ---------------------------------------------------------------------------------------------
def _bf(t):
    return 1 if t.dtype == torch.bfloat16 else 0


def layernorm(x, weight, bias=None, eps=1e-12, kind=0, out=None):
    """kind 0: BertLayerNorm (uncentred 2nd moment, src/modeling_bert.py:104-114); kind 1: T5 RMSNorm."""
    require_cuda(x, "x")
    H = x.shape[-1]
    x2 = x.reshape(-1, H)
    if x2.stride(-1) != 1:
        x2 = x2.contiguous()
    if out is None:
        out = torch.empty_like(x2)
    check(lib().atlas_b200_layernorm(_ptr(x2), x2.stride(0), _ptr(weight), _ptr(bias) if bias is not None else None,
                                     _ptr(out), out.stride(0), x2.shape[0], H, float(eps), kind, _bf(x),
                                     current_stream_ptr()))
    return out.reshape(x.shape)


def bert_embed_ln(input_ids, token_type_ids, word_emb, type_emb, pos_emb, ln_weight, ln_bias, eps):
    require_cuda(input_ids, "input_ids")
    B, L = input_ids.shape
    H = word_emb.shape[1]
    y = torch.empty((B, L, H), dtype=word_emb.dtype, device=word_emb.device)
    ids = input_ids.contiguous()
    tt = token_type_ids.contiguous() if token_type_ids is not None else None
    check(lib().atlas_b200_bert_embed_ln(_ptr(ids), _ptr(tt) if tt is not None else None, _ptr(word_emb), _ptr(type_emb),
                                         _ptr(pos_emb), _ptr(ln_weight), _ptr(ln_bias), _ptr(y), B, L, H, float(eps),
                                         _bf(word_emb), current_stream_ptr()))
    return y


def masked_mean_pool(x, mask, out=None):
    """x [B, L, H] 16-bit, mask [B, L] int64 -> [B, H] (optionally written into `out` rows, e.g. the bank)."""
    require_cuda(x, "x")
    B, L, H = x.shape
    xc = x.contiguous()
    m = mask.to(torch.int64).contiguous()
    if out is None:
        out = torch.empty((B, H), dtype=x.dtype, device=x.device)
    check(lib().atlas_b200_masked_mean_pool(_ptr(xc), _ptr(m), _ptr(out), out.stride(0), B, L, H, _bf(x),
                                            current_stream_ptr()))
    return out


def attention(q, q_col0, k, k_col0, v, v_col0, B, H, Lq, Lk, add_mask=None, bias_delta=None, scale=1.0,
              causal_value=0.0, out=None, return_lse=False, dropout=None, block_live=None):
    """Fused attention reading Q/K/V in place from [B*L, ld] projection buffers (head h at col0 + 64h).
    return_lse: also return the row log-sum-exp [B, H, Lq] fp32 (saved for the backward pass).
    block_live = key_block_live(add_mask): fully masked 64-key blocks are skipped by the encoder kernel (identical results).
    dropout = (p, seed, offset): dropout on the probabilities (training), mask re-derived by attention_bwd."""
    require_cuda(q, "q")
    if out is None:
        out = torch.empty((B * Lq, H * 64), dtype=q.dtype, device=q.device)
    am = add_mask.float().contiguous() if add_mask is not None else None
    bd = bias_delta.float().contiguous() if bias_delta is not None else None
    lse = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device) if return_lse else None
    dp, dseed, doff = dropout if dropout is not None else (0.0, 0, 0)
    check(lib().atlas_b200_attention_train(_ptr(q), q.stride(0), q_col0, _ptr(k), k.stride(0), k_col0, _ptr(v), v.stride(0),
                                           v_col0, _ptr(out), out.stride(0), _ptr(am) if am is not None else None,
                                           _ptr(bd) if bd is not None else None, B, H, Lq, Lk, float(scale),
                                           float(causal_value), 1, None, None, _ptr(lse) if lse is not None else None,
                                           float(dp), int(dseed), int(doff),
                                           _ptr(block_live) if block_live is not None else None, _bf(q),
                                           current_stream_ptr()))
    return (out, lse) if return_lse else out


ATTENTION_MAX_LK = 576          # keys per segment of `attention` (its K and V stay resident in shared memory)
ATTENTION_LONG_MAX_LK = 4096    # ... of `attention_long`; Lq + Lk - 1 <= 8192 as well (the bias table of attention_bwd)


def attention_long(q, q_col0, k, k_col0, v, v_col0, B, H, Lq, Lk, add_mask=None, bias_delta=None, scale=1.0,
                   causal_value=0.0, out=None, return_lse=False, dropout=None, block_live=None):
    """`attention` for key ranges up to ATTENTION_LONG_MAX_LK: K and V stream through shared memory (atlas_b200_attention_long).
    Same arguments and results; its lse and dropout masks are those `attention_bwd` expects."""
    require_cuda(q, "q")
    if out is None:
        out = torch.empty((B * Lq, H * 64), dtype=q.dtype, device=q.device)
    am = add_mask.float().contiguous() if add_mask is not None else None
    bd = bias_delta.float().contiguous() if bias_delta is not None else None
    lse = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device) if return_lse else None
    dp, dseed, doff = dropout if dropout is not None else (0.0, 0, 0)
    check(lib().atlas_b200_attention_long(_ptr(q), q.stride(0), q_col0, _ptr(k), k.stride(0), k_col0, _ptr(v), v.stride(0),
                                          v_col0, _ptr(out), out.stride(0), _ptr(am) if am is not None else None,
                                          _ptr(bd) if bd is not None else None, B, H, Lq, Lk, float(scale),
                                          float(causal_value), _ptr(lse) if lse is not None else None, float(dp),
                                          int(dseed), int(doff), _ptr(block_live) if block_live is not None else None,
                                          _bf(q), current_stream_ptr()))
    return (out, lse) if return_lse else out


def encoder_attention(L):
    """The self-attention forward for segments of L tokens: `attention` up to ATTENTION_MAX_LK, `attention_long` above."""
    return attention if L <= ATTENTION_MAX_LK else attention_long


_SKIP_MASKED = os.environ.get("ATLAS_B200_ATTN_SKIP_MASKED", "1") != "0"    # A/B switch of the masked-key-block skipping


def key_block_live(add_mask, block=64):
    """uint8 [B, ceil(Lk / block)]: 1 where a block of `block` consecutive keys holds at least one key whose additive mask is
    > -5000 (a live key).  The reference masks with -10000 (`get_extended_attention_mask`, transformers 4.18) or -1e4 / -1e9
    (`invert_attention_mask`): the softmax weight of such a key is exp(-10000 + s - max) = 0.0 exactly in fp32, so a block
    without a live key contributes nothing and the attention kernels skip its loads, MMAs and exponentials - bit-identical
    results.  (Assumes |score| < ~4000, like the reference's own fp32 softmax needs to stay finite.)  A batch element without
    any live key keeps every block live: its uniform-over-masked-keys softmax is computed like the reference's.  Returns None
    when skipping is switched off (ATLAS_B200_ATTN_SKIP_MASKED=0) or there is no mask."""
    if add_mask is None or not _SKIP_MASKED:
        return None
    B, Lk = add_mask.shape
    nb = (Lk + block - 1) // block
    m = add_mask
    if nb * block != Lk:
        m = torch.nn.functional.pad(m, (0, nb * block - Lk), value=float("-inf"))
    live = (m.view(B, nb, block) > -5000.0).any(-1)
    live = live | ~live.any(-1, keepdim=True)
    return live.to(torch.uint8).contiguous()


_XKV_COMPACT = os.environ.get("ATLAS_B200_XKV_COMPACT", "1") != "0"        # A/B switch of the compacted cross K | V


def compact_live_tiles(x, tile_live):
    """x [n_tiles * 64, d] 16-bit, tile_live uint8 [n_tiles] (flattened key_block_live) -> (x_live: the rows of the live 64-row
    tiles packed to the front of a buffer of the same shape, tile_off int32 [n_tiles]: position of every live tile in it (-1 =
    dead), count_rows int32 [1] on the device = 64 x #live).  Static shapes, no host synchronisation."""
    require_cuda(x, "x")
    x2 = _rows2d(x)
    flags = tile_live.reshape(-1)
    n_tiles = flags.numel()
    if x2.shape[0] != n_tiles * 64:
        raise AtlasB200Error(f"compact_live_tiles: {x2.shape[0]} rows for {n_tiles} tiles of 64")
    dst = torch.empty_like(x2)
    tile_off = torch.empty(n_tiles, dtype=torch.int32, device=x.device)
    count = torch.empty(1, dtype=torch.int32, device=x.device)
    check(lib().atlas_b200_compact_live_tiles(_ptr(x2), x2.stride(0), _ptr(flags), n_tiles, x2.shape[1], _ptr(dst),
                                              dst.stride(0), _ptr(tile_off), _ptr(count), current_stream_ptr()))
    return dst, tile_off, count


_ENC_PACKED = os.environ.get("ATLAS_B200_ENC_PACKED", "1") != "0"          # A/B switch of the padding-compacted FiD encoder
_BERT_PACKED = os.environ.get("ATLAS_B200_BERT_PACKED", "1") != "0"        # ... of the Contriever encoder (needs _ENC_PACKED too)


PACKED_MAX_L = ATTENTION_MAX_LK     # segment length limit of the padding-compacted encoder (attention_packed)


def encoder_packs(live, L):
    """Whether the padding-compacted encoder (no-grad and training) takes segments of L tokens with the live 64-key blocks
    `live` (key_block_live): there is a mask, the segments are whole 64-row tiles, and at most PACKED_MAX_L tokens long.
    Longer segments run padded, on attention_long."""
    return live is not None and L % 64 == 0 and 64 <= L <= PACKED_MAX_L


def segment_tile_scan(live):
    """live uint8 [S, nb] (key_block_live) -> (keep uint8 [S, nb], tile_off int32 [S * nb], tile_src int32 [S * nb], count_rows
    int32 [1]): the packed layout of the padding-compacted encoder (include/atlas_b200.h).  No host synchronisation."""
    require_cuda(live, "live")
    S, nb = live.shape
    live = live.contiguous()
    keep = torch.empty_like(live)
    tile_off = torch.empty(S * nb, dtype=torch.int32, device=live.device)
    tile_src = torch.empty(S * nb, dtype=torch.int32, device=live.device)
    count = torch.empty(1, dtype=torch.int32, device=live.device)
    check(lib().atlas_b200_segment_tile_scan(_ptr(live), S, nb, _ptr(keep), _ptr(tile_off), _ptr(tile_src), _ptr(count),
                                             current_stream_ptr()))
    return keep, tile_off, tile_src, count


def embed_packed_tiles(ids, table, tile_src):
    """Embedding rows of the token ids (int64 [n_tiles * 64]) of the kept tiles, in packed order; zeros past the end."""
    require_cuda(table, "table")
    ids = ids.reshape(-1)
    if ids.dtype != torch.int64:                   # torch's own embedding lookup takes int32 ids too
        if ids.dtype not in (torch.int32, torch.int16, torch.uint8):
            raise AtlasB200Error(f"embed_packed_tiles: integer token ids expected (got {ids.dtype})")
        ids = ids.to(torch.int64)
    ids = ids.contiguous()
    n_tiles = tile_src.numel()
    if ids.numel() != n_tiles * 64:
        raise AtlasB200Error(f"embed_packed_tiles: need {n_tiles * 64} token ids (got {ids.numel()})")
    out = torch.empty((n_tiles * 64, table.shape[1]), dtype=table.dtype, device=table.device)
    check(lib().atlas_b200_embed_packed_tiles(_ptr(ids), _ptr(table), table.stride(0), table.shape[0], _ptr(tile_src), n_tiles,
                                              _ptr(out), out.stride(0), table.shape[1], current_stream_ptr()))
    return out


def attention_packed(qkv, keep, tile_off, S, H, L, add_mask, bias_delta, scale=1.0, out=None, lse=False, dropout=None):
    """Encoder self-attention on the packed rows (segment s = its kept tiles, back to back): atlas_b200_attention_packed.
    lse: also return the row log-sum-exp [S, H, L] fp32 in the padded layout (kept rows written), for attention_packed_bwd.
    dropout = (p, seed, offset): dropout on the probabilities with the padded layout's masks."""
    require_cuda(qkv, "qkv")
    if out is None:
        out = torch.empty((qkv.shape[0], H * 64), dtype=qkv.dtype, device=qkv.device)
    am = add_mask.float().contiguous()
    bd = bias_delta.float().contiguous() if bias_delta is not None else None
    lse_t = torch.empty((S, H, L), dtype=torch.float32, device=qkv.device) if lse else None
    dp, dseed, doff = dropout if dropout is not None else (0.0, 0, 0)
    check(lib().atlas_b200_attention_packed(_ptr(qkv), qkv.stride(0), 0, H * 64, 2 * H * 64, _ptr(out), out.stride(0), _ptr(am),
                                            _ptr(bd) if bd is not None else None, _ptr(keep), _ptr(tile_off), S, H, L,
                                            float(scale), _ptr(lse_t) if lse else None, float(dp), int(dseed), int(doff),
                                            _bf(qkv), current_stream_ptr()))
    return (out, lse_t) if lse else out


def attention_packed_bwd(qkv, out, dout, keep, tile_off, S, H, L, add_mask, bias_delta, lse, scale=1.0, need_dbias=False,
                         dropout=None):
    """Backward of `attention_packed(..., lse=True)` (atlas_b200_attention_packed_bwd) -> (dqkv like qkv: dq | dk | dv at the
    columns of q | k | v, dbias_delta fp32 [H, 2L - 1] or None)."""
    require_cuda(qkv, "qkv")
    if lse is None:
        raise AtlasB200Error("attention_packed_bwd: needs the forward's log-sum-exp (lse, from lse=True)")
    am = add_mask.float().contiguous()
    bd = bias_delta.float().contiguous() if bias_delta is not None else None
    dbias = torch.zeros((H, 2 * L - 1), dtype=torch.float32, device=qkv.device) if (need_dbias and bd is not None) else None
    dsum = torch.empty((S, H, L), dtype=torch.float32, device=qkv.device)
    dqkv = torch.empty_like(qkv)
    o2, do2 = _rows2d(out), _rows2d(dout)
    dp, dseed, doff = dropout if dropout is not None else (0.0, 0, 0)
    check(lib().atlas_b200_attention_packed_bwd(_ptr(qkv), qkv.stride(0), _ptr(o2), o2.stride(0), _ptr(do2), do2.stride(0),
                                                _ptr(dqkv), dqkv.stride(0), _ptr(am), _ptr(bd) if bd is not None else None,
                                                _ptr(dbias) if dbias is not None else None, _ptr(lse.contiguous()), _ptr(dsum),
                                                _ptr(keep), _ptr(tile_off), S, H, L, float(scale), float(dp), int(dseed),
                                                int(doff), _bf(qkv), current_stream_ptr()))
    return dqkv, dbias


def expand_packed_tiles(x, tile_off):
    """Packed rows -> the padded layout [n_tiles * 64, d]; dropped tiles are zero."""
    require_cuda(x, "x")
    n_tiles = tile_off.numel()
    out = torch.empty((n_tiles * 64, x.shape[1]), dtype=x.dtype, device=x.device)
    check(lib().atlas_b200_expand_packed_tiles(_ptr(x), x.stride(0), _ptr(tile_off), n_tiles, _ptr(out), out.stride(0),
                                               x.shape[1], current_stream_ptr()))
    return out


def _combine(o_part, ml, B, splits, Lq, H, dtype, out=None, return_lse=False):
    """Merge the split-KV partials o_part [B*splits*Lq, H*64] / ml [B*splits*Lq, H, 2] (atlas_b200_attention_combine_ex)
    -> out [B*Lq, H*64] in `dtype` (and the row log-sum-exp [B, H, Lq] fp32 over all splits with return_lse)."""
    if out is None:
        out = torch.empty((B * Lq, H * 64), dtype=dtype, device=o_part.device)
    lse = torch.empty((B, H, Lq), dtype=torch.float32, device=o_part.device) if return_lse else None
    check(lib().atlas_b200_attention_combine_ex(_ptr(o_part), _ptr(ml), B, splits, Lq, H, _ptr(out), out.stride(0),
                                                _ptr(lse) if lse is not None else None, 1 if dtype == torch.bfloat16 else 0,
                                                current_stream_ptr()))
    return (out, lse) if return_lse else out


def cross_attention_stream_compact(q, kv_live, tile_live, tile_off, B, H, Lq, Lk_total, add_mask, scale=1.0, return_lse=False):
    """`cross_attention_split` on the stream kernel with K | V given as the compacted live tiles (`compact_live_tiles` of the
    encoder output, projected by `linear(..., rows=count)`)."""
    require_cuda(q, "q")
    am = add_mask.float().contiguous()
    chunk = _XATTN_CHUNK
    chunks = (Lk_total + chunk - 1) // chunk
    o_part = torch.empty((B * chunks * Lq, H * 64), dtype=torch.float32, device=q.device)
    ml = torch.empty((B * chunks * Lq, H, 2), dtype=torch.float32, device=q.device)
    check(lib().atlas_b200_cross_attention_stream_compact(_ptr(q), q.stride(0), 0, _ptr(kv_live), kv_live.stride(0), 0, H * 64,
                                                          _ptr(am), _ptr(tile_live), _ptr(tile_off), B, H, Lq, Lk_total,
                                                          chunk, float(scale), _ptr(o_part), _ptr(ml), _bf(q),
                                                          current_stream_ptr()))
    return _combine(o_part, ml, B, chunks, Lq, H, q.dtype, return_lse=return_lse)


_XATTN_STREAM = os.environ.get("ATLAS_B200_XATTN_STREAM", "1") != "0"      # A/B switch of the stream kernel
_XATTN_CHUNK = int(os.environ.get("ATLAS_B200_XATTN_CHUNK", "1024"))        # keys per CTA (multiple of 64)


def cross_attention_streams(Lq, Lk_total, dropout=None):
    """Whether `cross_attention_split` runs the K / V stream kernel, which takes any Lk_total, instead of `split`-key
    segments."""
    return Lq <= 64 and dropout is None and Lk_total >= 1024 and _XATTN_STREAM


def cross_attention_split(q, q_col0, kv, k_col0, v_col0, B, H, Lq, Lk_total, add_mask=None, scale=1.0, split=512,
                          return_lse=False, dropout=None, tile_live=None):
    """Attention of Lq (<= 128) queries per batch element over Lk_total keys (FiD decoder cross-attention,
    Lk_total = n_ctx * L): split-KV over segments of `split` keys + combine.  q [B*Lq, ld], kv [B*Lk_total, ld]."""
    require_cuda(q, "q")
    am = add_mask.float().contiguous() if add_mask is not None else None
    if cross_attention_streams(Lq, Lk_total, dropout):
        # few target tokens against the concatenated encoder keys: the K / V stream kernel (csrc/attention_stream.cu)
        chunk = _XATTN_CHUNK
        chunks = (Lk_total + chunk - 1) // chunk
        o_part = torch.empty((B * chunks * Lq, H * 64), dtype=torch.float32, device=q.device)
        ml = torch.empty((B * chunks * Lq, H, 2), dtype=torch.float32, device=q.device)
        if tile_live is None:
            tile_live = key_block_live(am)          # callers with many layers compute it once (fid.py)
        check(lib().atlas_b200_cross_attention_stream(_ptr(q), q.stride(0), q_col0, _ptr(kv), kv.stride(0), k_col0, v_col0,
                                                      _ptr(am) if am is not None else None,
                                                      _ptr(tile_live) if tile_live is not None else None, B, H, Lq, Lk_total,
                                                      chunk, float(scale), _ptr(o_part), _ptr(ml), _bf(q),
                                                      current_stream_ptr()))
        return _combine(o_part, ml, B, chunks, Lq, H, q.dtype, return_lse=return_lse)
    if Lk_total % split != 0:
        raise AtlasB200Error(f"cross_attention_split: Lk_total={Lk_total} must be a multiple of {split}")
    splits = Lk_total // split
    o_part = torch.empty((B * splits * Lq, H * 64), dtype=torch.float32, device=q.device)
    ml = torch.empty((B * splits * Lq, H, 2), dtype=torch.float32, device=q.device)
    dummy = torch.empty((8,), dtype=q.dtype, device=q.device)
    dp, dseed, doff = dropout if dropout is not None else (0.0, 0, 0)
    check(lib().atlas_b200_attention_train(_ptr(q), q.stride(0), q_col0, _ptr(kv), kv.stride(0), k_col0, _ptr(kv),
                                           kv.stride(0), v_col0, _ptr(dummy), 8, _ptr(am) if am is not None else None, None,
                                           B * splits, H, Lq, split, float(scale), 0.0, splits, _ptr(o_part), _ptr(ml),
                                           None, float(dp), int(dseed), int(doff), None, _bf(q), current_stream_ptr()))
    return _combine(o_part, ml, B, splits, Lq, H, q.dtype, return_lse=return_lse)


# ---------------------------------------------------------------------------------------------
# backward pass (csrc/backward.cu, csrc/attention_bwd.cu): raw kernel wrappers; the autograd wiring is grad_ops.py
# ---------------------------------------------------------------------------------------------
def _rows2d(t):
    t2 = t.reshape(-1, t.shape[-1])
    return t2 if t2.stride(-1) == 1 else t2.contiguous()


def transpose(x, pad_to=8):
    """[R, C] 16-bit -> [C, Rpad] with Rpad = R rounded up to `pad_to` and the pad columns zero."""
    require_cuda(x, "x")
    x2 = _rows2d(x)
    R, C = x2.shape
    Rpad = (R + pad_to - 1) // pad_to * pad_to
    out = torch.empty((C, Rpad), dtype=x.dtype, device=x.device)
    check(lib().atlas_b200_transpose(_ptr(x2), x2.stride(0), _ptr(out), out.stride(0), R, C, Rpad, current_stream_ptr()))
    return out


def colsum(x):
    """fp32 [N] column sums of a 16-bit [M, N] matrix (bias gradient)."""
    require_cuda(x, "x")
    x2 = _rows2d(x)
    out = torch.zeros(x2.shape[1], dtype=torch.float32, device=x.device)
    check(lib().atlas_b200_colsum(_ptr(x2), x2.stride(0), _ptr(out), x2.shape[0], x2.shape[1], _bf(x), current_stream_ptr()))
    return out


def linear_dgrad(dy, weight):
    """dX [M, K] = dY [M, N] . W [N, K]: the same wgmma GEMM on W^T (a weight-sized transpose per call)."""
    return linear(dy, transpose(weight))


def linear_wgrad(dy, x):
    """dW [N, K] = dY^T [N, M] . X [M, K] (contraction over the M tokens, fp32 accumulation, 16-bit result): the wgmma
    GEMM with both operands MN-major (no transposes)."""
    require_cuda(dy, "dy")
    dy2, x2 = _rows2d(dy), _rows2d(x)
    if dy2.shape[0] != x2.shape[0] or dy2.dtype != x2.dtype:
        raise AtlasB200Error(f"linear_wgrad: dy {tuple(dy2.shape)} and x {tuple(x2.shape)} do not match")
    M, N = dy2.shape
    K = x2.shape[1]
    dw = torch.empty((N, K), dtype=dy.dtype, device=dy.device)
    nbytes = lib().atlas_b200_linear_wgrad_workspace_bytes(M, N, K)        # split-K partial tiles (0 = un-split)
    ws = _wgrad_ws.get(nbytes, dy.device) if nbytes else None
    check(lib().atlas_b200_linear_wgrad(_ptr(dy2), dy2.stride(0), _ptr(x2), x2.stride(0), _ptr(dw), dw.stride(0), M, N, K,
                                        _bf(dy), _ptr(ws) if ws is not None else None, ws.numel() if ws is not None else 0,
                                        current_stream_ptr()))
    return dw


def layernorm_bwd(x, dy, weight, eps, kind, dres=None, need_bias=False):
    """-> (dx like x, dweight fp32 [H], dbias fp32 [H] or None)."""
    require_cuda(x, "x")
    H = x.shape[-1]
    x2, dy2 = _rows2d(x), _rows2d(dy)
    r2 = _rows2d(dres) if dres is not None else None
    dx = torch.empty_like(x2)
    dw = torch.zeros(H, dtype=torch.float32, device=x.device)
    db = torch.zeros(H, dtype=torch.float32, device=x.device) if (need_bias or kind == 0) else None
    check(lib().atlas_b200_layernorm_bwd(_ptr(x2), x2.stride(0), _ptr(dy2), dy2.stride(0), _ptr(weight),
                                         _ptr(r2) if r2 is not None else None, r2.stride(0) if r2 is not None else 0,
                                         _ptr(dx), dx.stride(0), _ptr(dw), _ptr(db) if db is not None else None,
                                         x2.shape[0], H, float(eps), kind, _bf(x), current_stream_ptr()))
    return dx.reshape(x.shape), dw, db


def gated_gelu(u, dg=None):
    """u [M, 2F] interleaved (wi_0 | wi_1) pre-activations -> g [M, F]; with dg [M, F] -> du [M, 2F]."""
    require_cuda(u, "u")
    u2 = _rows2d(u)
    M, F2 = u2.shape
    F = F2 // 2
    if dg is None:
        out = torch.empty((M, F), dtype=u.dtype, device=u.device)
        check(lib().atlas_b200_gated_gelu(_ptr(u2), u2.stride(0), None, 0, _ptr(out), out.stride(0), M, F, _bf(u),
                                          current_stream_ptr()))
        return out.reshape(*u.shape[:-1], F)
    d2 = _rows2d(dg)
    out = torch.empty((M, F2), dtype=u.dtype, device=u.device)
    check(lib().atlas_b200_gated_gelu(_ptr(u2), u2.stride(0), _ptr(d2), d2.stride(0), _ptr(out), out.stride(0), M, F,
                                      _bf(u), current_stream_ptr()))
    return out.reshape(u.shape)


def relu_bwd(g, dg):
    """du = dg * [g > 0] from the ReLU's saved output g (T5 v1.0 feed-forward, linear(..., epilogue=EPI_RELU))."""
    require_cuda(g, "g")
    if g.shape != dg.shape or g.dtype != dg.dtype or g.dtype not in (torch.float16, torch.bfloat16):
        raise AtlasB200Error(f"relu_bwd: g {tuple(g.shape)} {g.dtype} and dg {tuple(dg.shape)} {dg.dtype} must match, 16-bit")
    g2, d2 = _rows2d(g).contiguous(), _rows2d(dg).contiguous()
    out = torch.empty_like(g2)
    check(lib().atlas_b200_relu_bwd(_ptr(g2), g2.stride(0), _ptr(d2), d2.stride(0), _ptr(out), out.stride(0), g2.shape[0],
                                    g2.shape[1], _bf(g), current_stream_ptr()))
    return out.reshape(g.shape)


def gelu_erf(z, dy=None):
    """erf GELU of z (dy None) or its backward dy * gelu'(z)."""
    require_cuda(z, "z")
    z2 = _rows2d(z)
    d2 = _rows2d(dy) if dy is not None else None
    out = torch.empty_like(z2)
    check(lib().atlas_b200_gelu_erf(_ptr(z2), z2.stride(0), _ptr(d2) if d2 is not None else None,
                                    d2.stride(0) if d2 is not None else 0, _ptr(out), out.stride(0), z2.shape[0],
                                    z2.shape[1], _bf(z), current_stream_ptr()))
    return out.reshape(z.shape)


def dropout(x, p, seed, offset, residual=None, row_tiles=None):
    """out = (residual +) dropout(x): keep decisions are a pure function of (seed, offset, position), so calling this on
    dy with the same (seed, offset) is the backward of the forward call (csrc/dropout.cu).  row_tiles (int32, one entry per
    64 rows): x holds the packed rows of the padding-compacted encoder, row r takes the mask of padded row
    64 row_tiles[r // 64] + r % 64 (segment_tile_scan's tile_src)."""
    require_cuda(x, "x")
    x2 = _rows2d(x)
    r2 = _rows2d(residual) if residual is not None else None
    if row_tiles is not None and (row_tiles.dtype != torch.int32 or row_tiles.device != x.device
                                  or x2.shape[0] % 64 or row_tiles.numel() < x2.shape[0] // 64):
        raise AtlasB200Error(f"dropout: row_tiles must be int32 on {x.device} with one entry per 64 of the {x2.shape[0]} rows")
    rt = row_tiles.contiguous() if row_tiles is not None else None
    out = torch.empty_like(x2)
    check(lib().atlas_b200_dropout(_ptr(x2), x2.stride(0), _ptr(r2) if r2 is not None else None,
                                   r2.stride(0) if r2 is not None else 0, _ptr(out), out.stride(0), x2.shape[0],
                                   x2.shape[1], float(p), int(seed), int(offset), _ptr(rt) if rt is not None else None,
                                   _bf(x), current_stream_ptr()))
    return out.reshape(x.shape)


def dropout_mask(M, N, p, seed, offset, device):
    """The keep mask (uint8 [M, N]) `dropout` applies to an [M, N] tensor with this (seed, offset)."""
    out = torch.empty((M, N), dtype=torch.uint8, device=device)
    check(lib().atlas_b200_dropout_mask(_ptr(out), M, N, float(p), int(seed), int(offset), current_stream_ptr()))
    return out


def attention_dropout_mask(B, H, Lq, Lk, p, seed, offset, device):
    """The keep mask (uint8 [B, H, Lq, Lk]) the attention kernels apply to the probabilities with this (seed, offset)."""
    out = torch.empty((B, H, Lq, Lk), dtype=torch.uint8, device=device)
    check(lib().atlas_b200_attention_dropout_mask(_ptr(out), B * H * Lq, Lk, float(p), int(seed), int(offset),
                                                  current_stream_ptr()))
    return out


_inf_flags = {}


def clamp_inf_(x, row_ss=None, rows=None):
    """The reference's per-sub-layer fp16 overflow clamp (src/modeling_t5.py:657-708), in place, decided on the device
    (no host synchronisation).  A no-op for any other dtype, like the reference's `dtype == torch.float16` test.
    rows: int32 [1] device row count (as `linear(..., rows=)`): only the first min(max(rows, 0), M) rows are looked at,
    the rest (never computed) is neither read nor written."""
    if x.dtype != torch.float16:
        return x
    require_cuda(x, "x")
    x2 = _rows2d(x)
    if rows is not None and (rows.dtype != torch.int32 or rows.numel() != 1 or rows.device != x.device):
        raise AtlasB200Error(f"clamp_inf_: rows must be an int32 tensor of one element on {x.device}")
    flag = _inf_flags.get(x.device)
    if flag is None:
        flag = _inf_flags[x.device] = torch.zeros(1, dtype=torch.int32, device=x.device)
    check(lib().atlas_b200_clamp_inf_fp16(_ptr(x2), x2.stride(0), x2.shape[0], x2.shape[1],
                                          _ptr(rows) if rows is not None else None, _ptr(flag),
                                          _ptr(row_ss) if row_ss is not None else None, current_stream_ptr()))
    return x


def bert_embed_sum(input_ids, token_type_ids, word_emb, type_emb, pos_emb):
    require_cuda(input_ids, "input_ids")
    B, L = input_ids.shape
    H = word_emb.shape[1]
    y = torch.empty((B, L, H), dtype=word_emb.dtype, device=word_emb.device)
    ids = input_ids.contiguous()
    tt = token_type_ids.contiguous() if token_type_ids is not None else None
    check(lib().atlas_b200_bert_embed_sum(_ptr(ids), _ptr(tt) if tt is not None else None, _ptr(word_emb), _ptr(type_emb),
                                          _ptr(pos_emb), _ptr(y), B, L, H, _bf(word_emb), current_stream_ptr()))
    return y


def scatter_add_rows(src, table_rows, index=None, modulo=0, skip_index=-1):
    """fp32 [table_rows, H] with dst[index[r]] += src[r] (index None: r % modulo)."""
    require_cuda(src, "src")
    s2 = _rows2d(src)
    H = s2.shape[1]
    dst = torch.zeros((table_rows, H), dtype=torch.float32, device=src.device)
    idx = index.reshape(-1).contiguous() if index is not None else None
    check(lib().atlas_b200_scatter_add_rows(_ptr(idx) if idx is not None else None, int(modulo), _ptr(s2), s2.stride(0),
                                            _ptr(dst), s2.shape[0], H, int(skip_index), int(table_rows), _bf(src),
                                            current_stream_ptr()))
    return dst


def masked_mean_pool_bwd(demb, mask, L, H):
    require_cuda(demb, "demb")
    d2 = demb if demb.stride(-1) == 1 else demb.contiguous()
    B = d2.shape[0]
    m = mask.to(torch.int64).contiguous()
    dx = torch.empty((B, L, H), dtype=demb.dtype, device=demb.device)
    if B > 1 and d2.stride(0) % 2:
        d2 = d2.clone(memory_format=torch.contiguous_format)
    ld = d2.stride(0) if B > 1 else H          # a single row: its (arbitrary) stride is never used
    check(lib().atlas_b200_masked_mean_pool_bwd(_ptr(d2), ld, _ptr(m), _ptr(dx), B, L, H, _bf(demb),
                                                current_stream_ptr()))
    return dx


def cross_entropy_fwd(logits, labels):
    """-> (lse fp32 [rows], per-row loss fp32 [rows], 0 where label == -100)."""
    require_cuda(logits, "logits")
    l2 = _rows2d(logits)
    rows, V = l2.shape
    y = labels.reshape(-1).to(torch.int64).contiguous()
    lse = torch.empty(rows, dtype=torch.float32, device=logits.device)
    loss = torch.empty(rows, dtype=torch.float32, device=logits.device)
    check(lib().atlas_b200_cross_entropy_fwd(_ptr(l2), l2.stride(0), _ptr(y), _ptr(lse), _ptr(loss), rows, V, _bf(logits),
                                             current_stream_ptr()))
    return lse, loss


def cross_entropy_bwd(logits, labels, lse, gscale):
    """dlogits = (softmax - onehot) * gscale[0] for the valid rows (gscale: fp32 device scalar)."""
    l2 = _rows2d(logits)
    rows, V = l2.shape
    y = labels.reshape(-1).to(torch.int64).contiguous()
    out = torch.empty_like(l2)
    gs = gscale.reshape(1).to(torch.float32).contiguous()
    check(lib().atlas_b200_cross_entropy_bwd(_ptr(l2), l2.stride(0), _ptr(y), _ptr(lse), _ptr(gs), _ptr(out),
                                             out.stride(0), rows, V, _bf(logits), current_stream_ptr()))
    return out.reshape(logits.shape)


def attention_bwd(q, q_col0, k, k_col0, v, v_col0, out, dout, dq, dq_col0, dk, dk_col0, dv, dv_col0, B, H, Lq, Lk,
                  add_mask=None, bias_delta=None, need_dbias=False, scale=1.0, causal_value=0.0, lse=None,
                  split_keys=False, dropout=None, block_live=None):
    """Backward of `attention` / `cross_attention_split` (un-split key range).  dq / dk / dv are written in place at
    their column offsets; returns dbias_delta fp32 [H, Lq+Lk-1] (or None).  `lse` = the forward's log-sum-exp
    (return_lse=True), required; split_keys (no dbias; dq must be a whole contiguous [B*Lq, H*64] tensor) spreads a long
    key range over many CTAs (FiD cross-attention)."""
    if lse is None:
        raise AtlasB200Error("attention_bwd: needs the forward's log-sum-exp (lse, from return_lse=True)")
    require_cuda(q, "q")
    am = add_mask.float().contiguous() if add_mask is not None else None
    bd = bias_delta.float().contiguous() if bias_delta is not None else None
    dbias = torch.zeros((H, Lq + Lk - 1), dtype=torch.float32, device=q.device) if (need_dbias and bd is not None) else None
    dsum = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device)
    lse = lse.contiguous()
    o2 = out if out.stride(-1) == 1 else out.contiguous()
    do2 = _rows2d(dout)
    accum = None
    if split_keys:
        if dbias is not None or dq_col0 != 0 or not dq.is_contiguous() or dq.shape[1] != H * 64:
            raise AtlasB200Error("attention_bwd: split_keys needs no dbias and a contiguous dq")
        accum = torch.zeros((B * Lq, H * 64), dtype=torch.float32, device=q.device)
    dp, dseed, doff = dropout if dropout is not None else (0.0, 0, 0)
    check(lib().atlas_b200_attention_bwd_train(
        _ptr(q), q.stride(0), q_col0, _ptr(k), k.stride(0), k_col0, _ptr(v), v.stride(0), v_col0, _ptr(o2), o2.stride(0),
        _ptr(do2), do2.stride(0), _ptr(dq), dq.stride(0), dq_col0, _ptr(dk), dk.stride(0), dk_col0, _ptr(dv),
        dv.stride(0), dv_col0, _ptr(am) if am is not None else None, _ptr(bd) if bd is not None else None,
        _ptr(dbias) if dbias is not None else None, _ptr(lse), _ptr(dsum),
        _ptr(accum) if accum is not None else None, B, H, Lq, Lk, float(scale), float(causal_value), float(dp),
        int(dseed), int(doff), _ptr(block_live) if block_live is not None else None, _bf(q), current_stream_ptr()))
    if accum is not None:
        check(lib().atlas_b200_cast_f32(_ptr(accum), _ptr(dq), accum.numel(), _bf(q), current_stream_ptr()))
    return dbias


def cross_attention_stats(q, q_col0, kv, k_col0, v_col0, B, H, T, Lk, lse, add_mask=None, scale=1.0):
    """Means over heads of the cross-attention logits, probabilities and ||V||-weighted probabilities -> three fp32
    [B, T, Lk] tensors (`score_storage`, `prob_storage`, `normalized_score_storage` of src/fid.py:333-343)."""
    require_cuda(q, "q")
    am = add_mask.float().contiguous() if add_mask is not None else None
    out = torch.empty((3, B, T, Lk), dtype=torch.float32, device=q.device)
    l2 = lse.contiguous()
    check(lib().atlas_b200_cross_attention_stats(_ptr(q), q.stride(0), q_col0, _ptr(kv), kv.stride(0), k_col0, v_col0,
                                                 _ptr(am) if am is not None else None, _ptr(l2), _ptr(out[0]), _ptr(out[1]),
                                                 _ptr(out[2]), B, H, T, Lk, float(scale), _bf(q), current_stream_ptr()))
    return out[0], out[1], out[2]


# ---------------------------------------------------------------------------------------------
# single-token decode (csrc/decode.cu): KV-cached greedy generation
# ---------------------------------------------------------------------------------------------
def decode_self_attention(qkv, cache, t_dev, H, bias_delta=None, scale=1.0, out=None):
    """qkv [B, 3*H*64] of the new token; cache [B, Tmax, 2*H*64] (k | v) updated in place at row t_dev[0]; -> ctx [B, H*64]."""
    require_cuda(qkv, "qkv")
    B, Tmax = cache.shape[0], cache.shape[1]
    if out is None:
        out = torch.empty((B, H * 64), dtype=qkv.dtype, device=qkv.device)
    bd = bias_delta.float().contiguous() if bias_delta is not None else None
    check(lib().atlas_b200_decode_self_attention(_ptr(qkv), qkv.stride(0), _ptr(cache), Tmax, _ptr(t_dev),
                                                 _ptr(bd) if bd is not None else None, float(scale), _ptr(out),
                                                 out.stride(0), B, H, _bf(qkv), current_stream_ptr()))
    return out


def decode_cross_attention(q, kv, B, H, Lk, add_mask=None, scale=1.0, chunk=256, out=None, tile_live=None):
    """q [B, H*64] against kv [B*Lk, 2*H*64] (k | v): chunked partials + the split-KV combine -> ctx [B, H*64].
    tile_live = key_block_live(add_mask): 64-key tiles of masked keys only are not read (identical result)."""
    require_cuda(q, "q")
    chunks = (Lk + chunk - 1) // chunk
    o_part = torch.empty((B * chunks, H * 64), dtype=torch.float32, device=q.device)
    ml = torch.empty((B * chunks, H, 2), dtype=torch.float32, device=q.device)
    am = add_mask.float().contiguous() if add_mask is not None else None
    check(lib().atlas_b200_decode_cross_attention_live(_ptr(q), q.stride(0), _ptr(kv), kv.stride(0), 0, H * 64,
                                                       _ptr(am) if am is not None else None,
                                                       _ptr(tile_live) if tile_live is not None else None, B, H, Lk, chunk,
                                                       float(scale), _ptr(o_part), _ptr(ml), _bf(q), current_stream_ptr()))
    return _combine(o_part, ml, B, chunks, 1, H, q.dtype, out=out)


def decode_argmax(logits, seq, tok_in, done, t_dev, eos_id, pad_id, min_length):
    """Greedy pick on the device (see include/atlas_b200.h); advances t_dev."""
    require_cuda(logits, "logits")
    B, V = logits.shape
    check(lib().atlas_b200_decode_argmax(_ptr(logits), logits.stride(0), V, _ptr(seq), seq.stride(0), _ptr(tok_in),
                                         _ptr(done), _ptr(t_dev), int(eos_id), int(pad_id), int(min_length), B, _bf(logits),
                                         current_stream_ptr()))


# ---------------------------------------------------------------------------------------------
# beam search (csrc/beam.cu, the ancestry-gathered self-attention of csrc/decode.cu)
# ---------------------------------------------------------------------------------------------
MAX_BEAMS = 16      # ATLAS_B200_MAX_BEAMS


def decode_self_attention_beam(qkv, cache, t_dev, anc, H, bias_delta=None, scale=1.0, out=None):
    """decode_self_attention over R = B * nb beam rows whose history is gathered through anc int32 [2, R, Tmax] (buffer
    t_dev[0] & 1): the new K | V lands in cache row (r, t), keys / values j come from (anc[r, j], j)."""
    require_cuda(qkv, "qkv")
    R, Tmax = cache.shape[0], cache.shape[1]
    if anc.shape != (2, R, Tmax) or anc.dtype != torch.int32 or not anc.is_contiguous():
        raise AtlasB200Error(f"decode_self_attention_beam: anc must be contiguous int32 [2, {R}, {Tmax}]")
    if out is None:
        out = torch.empty((R, H * 64), dtype=qkv.dtype, device=qkv.device)
    bd = bias_delta.float().contiguous() if bias_delta is not None else None
    check(lib().atlas_b200_decode_self_attention_beam(_ptr(qkv), qkv.stride(0), _ptr(cache), Tmax, _ptr(t_dev), _ptr(anc),
                                                      _ptr(bd) if bd is not None else None, float(scale), _ptr(out),
                                                      out.stride(0), R, H, _bf(qkv), current_stream_ptr()))
    return out


def decode_cross_attention_beams(q, kv, B, nb, H, Lk, add_mask, chunk, tile_live=None):
    """The nb beams of a batch element (consecutive rows of q [B * nb, H*64]) against its ONE cross K | V kv [B * Lk, 2*H*64]:
    the Lq = nb shape of the cross-attention stream kernel (live-tile skipping) + the split combine -> ctx [B * nb, H*64].
    The K | V bytes read per step do not grow with nb."""
    require_cuda(q, "q")
    if chunk % 64 != 0:
        raise AtlasB200Error(f"decode_cross_attention_beams: chunk {chunk} must be a multiple of 64")
    chunks = (Lk + chunk - 1) // chunk
    o_part = torch.empty((B * chunks * nb, H * 64), dtype=torch.float32, device=q.device)
    ml = torch.empty((B * chunks * nb, H, 2), dtype=torch.float32, device=q.device)
    am = add_mask.float().contiguous() if add_mask is not None else None
    check(lib().atlas_b200_cross_attention_stream(_ptr(q), q.stride(0), 0, _ptr(kv), kv.stride(0), 0, H * 64,
                                                  _ptr(am) if am is not None else None,
                                                  _ptr(tile_live) if tile_live is not None else None, B, H, nb, Lk, chunk,
                                                  1.0, _ptr(o_part), _ptr(ml), _bf(q), current_stream_ptr()))
    return _combine(o_part, ml, B, chunks, nb, H, q.dtype)


# ---------------------------------------------------------------------------------------------
# opt-in FP8 (e4m3) cross K|V cache of KV-cached generation (csrc/kv_fp8.cu): lossy, off by default
# ---------------------------------------------------------------------------------------------
def _check_2d(t, name, dtype, shape, ld_mult=1):
    require_cuda(t, name)
    if t.dtype != dtype or t.dim() != 2 or tuple(t.shape) != tuple(shape) or t.stride(1) != 1 or \
            t.stride(0) % ld_mult != 0 or (shape[0] > 1 and t.stride(0) < shape[1]):
        raise AtlasB200Error(f"{name} must be {dtype} {list(shape)} with unit inner stride and a row stride that is a multiple of "
                             f"{ld_mult}, got {t.dtype} {list(t.shape)} strides {t.stride()}")


def _check_e4m3_cache(q, kv8, kv_scale, Bq, B, H, Lk, add_mask, tile_live, what):
    if q.dtype not in (torch.float16, torch.bfloat16):
        raise AtlasB200Error(f"{what}: q must be fp16 or bf16 (got {q.dtype})")
    _check_2d(q, "q", q.dtype, (Bq, H * 64), 8)
    _check_2d(kv8, "kv8", torch.uint8, (B * Lk, 2 * H * 64), 16)
    _check_2d(kv_scale, "kv_scale", torch.float32, (B * Lk, 2 * H))
    if any(t is not None and t.device != q.device for t in (kv8, kv_scale, add_mask, tile_live)):
        raise AtlasB200Error(f"{what}: q, kv8, kv_scale, add_mask and tile_live must be on one device")
    if q.data_ptr() % 16 != 0 or kv8.data_ptr() % 16 != 0:
        raise AtlasB200Error(f"{what}: q and kv8 must start 16-byte aligned (16-byte loads)")
    if add_mask is not None and tuple(add_mask.shape) != (B, Lk):
        raise AtlasB200Error(f"{what}: add_mask must be [{B}, {Lk}] (got {list(add_mask.shape)})")
    if tile_live is not None and (tile_live.dtype != torch.uint8 or tuple(tile_live.shape) != (B, (Lk + 63) // 64)
                                  or not tile_live.is_contiguous()):
        raise AtlasB200Error(f"{what}: tile_live must be contiguous uint8 [{B}, {(Lk + 63) // 64}]")


def quantize_kv_e4m3(x, out=None, scale_out=None):
    """x [rows, C*64] fp16 / bf16 (unit inner stride) -> (codes uint8 [rows, C*64] e4m3fn, scales fp32 [rows, C]): one scale
    per 64-value block, amax / 448 (see include/atlas_b200.h).  `out` / `scale_out`: pre-allocated (possibly strided) buffers."""
    require_cuda(x, "x")
    if x.dtype not in (torch.float16, torch.bfloat16) or x.dim() != 2 or x.shape[1] % 64 != 0 or x.shape[1] == 0:
        raise AtlasB200Error(f"quantize_kv_e4m3: x must be fp16 / bf16 [rows, C*64] (got {x.dtype} {list(x.shape)})")
    rows, C = x.shape[0], x.shape[1] // 64
    _check_2d(x, "x", x.dtype, (rows, C * 64), 8)
    if out is None:
        out = torch.empty((rows, C * 64), dtype=torch.uint8, device=x.device)
    if scale_out is None:
        scale_out = torch.empty((rows, C), dtype=torch.float32, device=x.device)
    _check_2d(out, "out", torch.uint8, (rows, C * 64), 8)
    _check_2d(scale_out, "scale_out", torch.float32, (rows, C))
    if out.device != x.device or scale_out.device != x.device:
        raise AtlasB200Error("quantize_kv_e4m3: x, out and scale_out must be on one device")
    if x.data_ptr() % 16 != 0 or out.data_ptr() % 8 != 0:
        raise AtlasB200Error("quantize_kv_e4m3: x must start 16-byte aligned (16-byte loads), out 8-byte aligned")
    check(lib().atlas_b200_quantize_kv_e4m3(_ptr(x), max(x.stride(0), C * 64), rows, C, _ptr(out), max(out.stride(0), C * 64),
                                            _ptr(scale_out), max(scale_out.stride(0), C), _bf(x), current_stream_ptr()))
    return out, scale_out


def decode_cross_attention_e4m3(q, kv8, kv_scale, B, H, Lk, add_mask=None, scale=1.0, chunk=256, out=None, tile_live=None):
    """decode_cross_attention over the e4m3 cache: q [B, H*64] against codes kv8 uint8 [B*Lk, 2*H*64] (k | v) and their scales
    kv_scale fp32 [B*Lk, 2*H] (quantize_kv_e4m3) -> ctx [B, H*64] in q's dtype."""
    _check_e4m3_cache(q, kv8, kv_scale, B, B, H, Lk, add_mask, tile_live, "decode_cross_attention_e4m3")
    if chunk <= 0 or chunk % 16 != 0:
        raise AtlasB200Error(f"decode_cross_attention_e4m3: chunk {chunk} must be a positive multiple of 16")
    chunks = (Lk + chunk - 1) // chunk
    o_part = torch.empty((B * chunks, H * 64), dtype=torch.float32, device=q.device)
    ml = torch.empty((B * chunks, H, 2), dtype=torch.float32, device=q.device)
    am = add_mask.float().contiguous() if add_mask is not None else None
    check(lib().atlas_b200_decode_cross_attention_e4m3(_ptr(q), q.stride(0), _ptr(kv8), max(kv8.stride(0), 2 * H * 64),
                                                       _ptr(kv_scale), max(kv_scale.stride(0), 2 * H), 0, H * 64,
                                                       _ptr(am) if am is not None else None,
                                                       _ptr(tile_live) if tile_live is not None else None, B, H, Lk, chunk,
                                                       float(scale), _ptr(o_part), _ptr(ml), _bf(q), current_stream_ptr()))
    return _combine(o_part, ml, B, chunks, 1, H, q.dtype, out=out)


def decode_cross_attention_beams_e4m3(q, kv8, kv_scale, B, nb, H, Lk, add_mask, chunk, tile_live=None, scale=1.0):
    """decode_cross_attention_beams over the e4m3 cache (the stream kernel's e4m3 path, Lq = nb <= 64): q [B * nb, H*64], codes
    kv8 uint8 [B*Lk, 2*H*64], scales kv_scale fp32 [B*Lk, 2*H] -> ctx [B * nb, H*64]."""
    _check_e4m3_cache(q, kv8, kv_scale, B * nb, B, H, Lk, add_mask, tile_live, "decode_cross_attention_beams_e4m3")
    if chunk <= 0 or chunk % 64 != 0:
        raise AtlasB200Error(f"decode_cross_attention_beams_e4m3: chunk {chunk} must be a positive multiple of 64")
    chunks = (Lk + chunk - 1) // chunk
    o_part = torch.empty((B * chunks * nb, H * 64), dtype=torch.float32, device=q.device)
    ml = torch.empty((B * chunks * nb, H, 2), dtype=torch.float32, device=q.device)
    am = add_mask.float().contiguous() if add_mask is not None else None
    check(lib().atlas_b200_cross_attention_stream_e4m3(_ptr(q), q.stride(0), 0, _ptr(kv8), max(kv8.stride(0), 2 * H * 64),
                                                       _ptr(kv_scale), max(kv_scale.stride(0), 2 * H), 0, H * 64,
                                                       _ptr(am) if am is not None else None,
                                                       _ptr(tile_live) if tile_live is not None else None, B, H, nb, Lk, chunk,
                                                       float(scale), _ptr(o_part), _ptr(ml), _bf(q), current_stream_ptr()))
    return _combine(o_part, ml, B, chunks, nb, H, q.dtype)


def beam_topk(logits, beam_scores, t_dev, k, eos_id, min_length, round_lp, add_mask=None, cand_score=None, cand_tok=None,
              lp_out=None):
    """Per-row log-softmax + EOS ban + mask + beam score -> the row's top-k (cand_score fp32, cand_tok int32 [R, k])."""
    require_cuda(logits, "logits")
    R, V = logits.shape
    if cand_score is None:
        cand_score = torch.empty((R, k), dtype=torch.float32, device=logits.device)
        cand_tok = torch.empty((R, k), dtype=torch.int32, device=logits.device)
    if add_mask is not None and (add_mask.dtype != torch.float32 or add_mask.shape != (R, V) or add_mask.stride(1) != 1):
        raise AtlasB200Error(f"beam_topk: add_mask must be fp32 [{R}, {V}] with unit inner stride")
    if lp_out is not None and (lp_out.dtype != torch.float32 or lp_out.shape != (R, V) or not lp_out.is_contiguous()):
        raise AtlasB200Error(f"beam_topk: lp_out must be contiguous fp32 [{R}, {V}]")
    check(lib().atlas_b200_beam_topk(_ptr(logits), logits.stride(0), V,
                                     _ptr(add_mask) if add_mask is not None else None,
                                     add_mask.stride(0) if add_mask is not None else 0, _ptr(beam_scores), _ptr(t_dev),
                                     int(eos_id), int(min_length), int(bool(round_lp)), int(k), _ptr(cand_score),
                                     _ptr(cand_tok), _ptr(lp_out) if lp_out is not None else None, R, _bf(logits),
                                     current_stream_ptr()))
    return cand_score, cand_tok


def beam_select(cand_score, cand_tok, nb, V, beam_scores, tok_in, parent, done, anc, tok, t_dev, hyp_score, hyp_len, hyp_ins,
                hyp_tok, hyp_state, hyp_worst, eos_id, pad_id, length_penalty):
    """Scorer step on the device over the candidates of beam_topk (k = 2 * nb), for B = done.numel() batch elements and
    R = B * nb rows: beam_scores fp32 [R], tok_in int64 [R], parent int32 [R], done uint8 [B], anc int32 [2, R, Tmax],
    tok int32 [R, Tmax], t_dev int32 [1], hyp_score fp64 [B, nb], hyp_len / hyp_ins int32 [B, nb], hyp_tok int32
    [B, nb, Tmax], hyp_state int32 [B, 2], hyp_worst fp64 [B] (include/atlas_b200.h).  Advances t_dev."""
    require_cuda(cand_score, "cand_score")
    B = done.numel()
    R, Tmax = tok.shape
    want = {"cand_score": (cand_score, torch.float32, (R, 2 * nb)), "cand_tok": (cand_tok, torch.int32, (R, 2 * nb)),
            "beam_scores": (beam_scores, torch.float32, (R,)), "tok_in": (tok_in, torch.int64, (R,)),
            "parent": (parent, torch.int32, (R,)), "done": (done, torch.uint8, (B,)), "anc": (anc, torch.int32, (2, R, Tmax)),
            "tok": (tok, torch.int32, (R, Tmax)), "t_dev": (t_dev, torch.int32, (1,)),
            "hyp_score": (hyp_score, torch.float64, (B, nb)), "hyp_len": (hyp_len, torch.int32, (B, nb)),
            "hyp_ins": (hyp_ins, torch.int32, (B, nb)), "hyp_tok": (hyp_tok, torch.int32, (B, nb, Tmax)),
            "hyp_state": (hyp_state, torch.int32, (B, 2)), "hyp_worst": (hyp_worst, torch.float64, (B,))}
    for name, (t, dtype, shape) in want.items():
        if t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous():
            raise AtlasB200Error(f"beam_select: {name} must be contiguous {dtype} {list(shape)} (B={B}, nb={nb}), got "
                                 f"{t.dtype} {list(t.shape)}")
    if R != B * nb:
        raise AtlasB200Error(f"beam_select: {R} rows for B={B} x nb={nb}")
    check(lib().atlas_b200_beam_select(_ptr(cand_score), _ptr(cand_tok), B, nb, V, _ptr(beam_scores), _ptr(tok_in),
                                       _ptr(parent), _ptr(done), _ptr(anc), _ptr(tok), Tmax, _ptr(t_dev), _ptr(hyp_score),
                                       _ptr(hyp_len), _ptr(hyp_ins), _ptr(hyp_tok), _ptr(hyp_state), _ptr(hyp_worst),
                                       int(eos_id), int(pad_id), float(length_penalty), current_stream_ptr()))
