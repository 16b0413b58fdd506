"""Drop-in for `src.index.DistributedIndex` (reference src/index.py:43-160) on B200.

Same public surface: `embeddings` ([768, N] fp16 CUDA, slice-assignable on dim 1),
`doc_map`, `is_in_gpu`, `init_embeddings`, `search_knn`, `save_index`, `load_index`,
`is_index_trained`, `train_index`.  What changes underneath:

  * the bank is stored passage-major, `[N, 768]` row-major (1536 contiguous bytes per passage, what
    TMA / wgmma want); `embeddings` is the transposed VIEW, so `index.embeddings[:, a:b] = emb.T`
    (src/atlas.py:79) and `embeddings[:, s:e]` (src/index.py:85) keep working and write through;
  * `_compute_scores_and_indices` is ONE fused scan (csrc/mips.cu) instead of matmul + topk: the
    [nq, N] score matrix is never materialised;
  * `search_knn` exchanges (fp16 score, int64 global id) pairs - one fixed-shape all-gather - instead
    of pickled passage dicts through 4*W var-size gathers; passage text is resolved from a node-shared
    store (atlas_b200/passage_store.py);
  * ties are ordered canonically: score descending, then global passage id ascending.

There is no CPU path: `is_in_gpu = False` raises here.  `DistributedFAISSIndex` (below) is the reference's
`--index_mode faiss` with host-resident rows and a product-quantized (csrc/pq.cu), 4-bit scalar-quantized
(csrc/ivfsq.cu) or full-precision inverted-list (csrc/ivfflat.cu) device index.
"""
import ctypes
import logging
import math
import os
import pickle
from typing import Optional

import numpy as np
import torch

from . import dist_utils, ops
from ._lib import MAX_TOPK, AtlasB200Error, check, lib
from .passage_store import make_store

logger = logging.getLogger(__name__)

EMBEDDINGS_DIM: int = 768  # src/retrievers.py:13


class DistributedIndex(object):
    def __init__(self):
        self._bank = None  # [N_local, 768] fp16, CUDA
        self.doc_map = dict()
        self.is_in_gpu = True
        self._store = None
        self._workspace = ops.Workspace()
        # global id of local row l is _id_base + _id_stride * l
        self._id_base, self._id_stride = 0, 1
        self._offsets = None  # contiguous layout (after load_index): first global id of every rank
        # Upper bound of the queries ANY rank passes to one search (e.g. --per_gpu_batch_size, identical on all ranks).
        # When set, a distributed search pads every rank's block to this many rows: no size exchange, no host
        # synchronisation in front of the query all-gather (src/index.py:127-129 does a var-size gather + a size gather).
        self.max_queries_per_rank = None

    # ------------------------------------------------------------------ bank / reference view
    @property
    def embeddings(self):
        """The reference's `[768, N]` tensor (src/index.py:51), as a view of the passage-major bank."""
        return None if self._bank is None else self._bank.t()

    @embeddings.setter
    def embeddings(self, value):
        if value is None:
            self._bank = None
            return
        if value.dim() != 2 or value.shape[0] != EMBEDDINGS_DIM:
            raise ValueError(f"embeddings must be [{EMBEDDINGS_DIM}, N], got {tuple(value.shape)}")
        self._bank = value.t().contiguous().to(device=self._device(), dtype=torch.float16)

    @staticmethod
    def _device():
        if not torch.cuda.is_available():
            raise AtlasB200Error("atlas_b200.DistributedIndex needs a CUDA device (no CPU fallback)")
        return torch.device("cuda", torch.cuda.current_device())

    def init_embeddings(self, passages, dim: Optional[int] = EMBEDDINGS_DIM):
        """src/index.py:49-53.  Local row l holds global passage line l*W + rank (src/index_io.py:41)."""
        if dim != EMBEDDINGS_DIM:
            raise ValueError(f"only dim={EMBEDDINGS_DIM} is supported (src/retrievers.py:13)")
        if not self.is_in_gpu:
            raise AtlasB200Error("is_in_gpu=False (CPU-resident bank) is a FAISS-only mode and is not supported")
        self.doc_map = {i: doc for i, doc in enumerate(passages)}
        self._bank = torch.zeros(len(passages), dim, dtype=torch.float16, device=self._device())
        self._id_base, self._id_stride = dist_utils.get_rank(), dist_utils.get_world_size()
        self._offsets = None
        self._reset_store()

    def _reset_store(self):
        if self._store is not None:
            self._store.close()
        self._store = None

    def _get_store(self):
        if self._store is None:
            self._store = make_store(self.doc_map, dist_utils.get_rank(), dist_utils.get_world_size())
        return self._store

    # ------------------------------------------------------------------ persistence (reference format)
    def _get_saved_embedding_path(self, save_dir: str, shard: int) -> str:
        return os.path.join(save_dir, f"embeddings.{shard}.pt")

    def _get_saved_passages_path(self, save_dir: str, shard: int) -> str:
        return os.path.join(save_dir, f"passages.{shard}.pt")

    def save_index(self, path: str, total_saved_shards: int, overwrite_saved_passages: bool = False) -> None:
        """Same files as src/index.py:61-87: `embeddings.{s}.pt` = [768, n_s] fp16, `passages.{s}.pt`."""
        assert self._bank is not None
        rank = dist_utils.get_rank()
        ws = dist_utils.get_world_size()
        assert total_saved_shards % ws == 0, f"N workers must be a multiple of shards to save"
        shards_per_worker = total_saved_shards // ws
        n_embeddings = self._bank.shape[0]
        embeddings_per_shard = math.ceil(n_embeddings / shards_per_worker)
        assert n_embeddings == len(self.doc_map), len(self.doc_map)
        for shard_ind, shard_start in enumerate(range(0, n_embeddings, embeddings_per_shard)):
            shard_end = min(shard_start + embeddings_per_shard, n_embeddings)
            shard_id = shard_ind + rank * shards_per_worker
            passage_shard_path = self._get_saved_passages_path(path, shard_id)
            if not os.path.exists(passage_shard_path) or overwrite_saved_passages:
                passage_shard = [self.doc_map[i] for i in range(shard_start, shard_end)]
                with open(passage_shard_path, "wb") as fobj:
                    pickle.dump(passage_shard, fobj, protocol=pickle.HIGHEST_PROTOCOL)
            embeddings_shard = self._bank[shard_start:shard_end].t().contiguous()  # [768, n_s]
            torch.save(embeddings_shard, self._get_saved_embedding_path(path, shard_id))

    def load_index(self, path: str, total_saved_shards: int):
        """src/index.py:89-111.  Rank r holds shard files r*S/W .. (r+1)*S/W-1 concatenated; global ids
        are then contiguous per rank (offsets exchanged once here)."""
        rank = dist_utils.get_rank()
        ws = dist_utils.get_world_size()
        assert total_saved_shards % ws == 0, f"N workers must be a multiple of shards to save"
        shards_per_worker = total_saved_shards // ws
        passages = []
        shard_ids = list(range(rank * shards_per_worker, (rank + 1) * shards_per_worker))
        for shard_id in shard_ids:
            with open(self._get_saved_passages_path(path, shard_id), "rb") as fobj:
                passages.append(pickle.load(fobj))
        self.doc_map = {}
        n_passages = 0
        for chunk in passages:
            for p in chunk:
                self.doc_map[n_passages] = p
                n_passages += 1
        device = self._device()
        files = [self._get_saved_embedding_path(path, s) for s in shard_ids]
        self._bank = self._load_rows(files, device)
        sizes = dist_utils.get_varsize(torch.empty((self._bank.shape[0], 0), device=self._query_device()))
        self._offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        self._id_base, self._id_stride = int(self._offsets[rank]), 1
        self._reset_store()

    def _load_rows(self, files, device):
        if device.type == "cuda":
            return self._load_bank_streamed(files, device)
        # CPU test doubles of this class (tests/test_index_gloo.py)
        rows = [torch.load(f, map_location="cpu").t().to(torch.float16) for f in files]
        return torch.cat(rows, dim=0).contiguous().to(device)

    def _query_device(self):
        """Where the query rows of a search live (the bank's device)."""
        return self._bank.device

    @staticmethod
    def _load_bank_streamed(files, device, chunk_cols=262144, host=False):
        """The shard files (`embeddings.{s}.pt` = [768, n_s] fp16, src/index.py:75-87) straight into the device bank
        [sum n_s, 768]: every file is memory-mapped (`torch.load(mmap=True)`: no host copy of the whole tensor), column
        chunks are staged through two pinned buffers, copied H2D asynchronously and transposed into their bank rows by
        `atlas_b200_transpose` on the GPU.  The reference (and round 1 here) reads every shard into host memory,
        transposes it on ONE CPU core (`.t()` + `cat` -> a strided 2-byte copy, ~1 GB/s) and only then uploads it.
        host=True: the rows go to a pinned HOST tensor instead (DistributedFAISSIndex): every chunk is transposed into a
        device staging buffer and copied back asynchronously."""
        shards = []
        for f in files:
            try:
                t = torch.load(f, map_location="cpu", mmap=True)
            except (RuntimeError, ValueError, TypeError):     # legacy (non-zip) checkpoint: no mmap
                t = torch.load(f, map_location="cpu")
            if t.dim() != 2 or t.shape[0] != EMBEDDINGS_DIM:
                raise AtlasB200Error(f"{f}: expected a [{EMBEDDINGS_DIM}, n] embedding shard, got {tuple(t.shape)}")
            shards.append(t)
        total = sum(int(t.shape[1]) for t in shards)
        width = max(8, min(chunk_cols, max((int(t.shape[1]) for t in shards), default=8)))
        width = (width + 7) // 8 * 8
        if host:
            bank = torch.empty((total, EMBEDDINGS_DIM), dtype=torch.float16).pin_memory()
            tstage = [torch.empty((width, EMBEDDINGS_DIM), dtype=torch.float16, device=device) for _ in range(2)]
        else:
            bank = torch.empty((total, EMBEDDINGS_DIM), dtype=torch.float16, device=device)
        stage = [torch.empty((EMBEDDINGS_DIM, width), dtype=torch.float16).pin_memory() for _ in range(2)]
        dstage = [torch.empty((EMBEDDINGS_DIM, width), dtype=torch.float16, device=device) for _ in range(2)]
        done = [torch.cuda.Event(), torch.cuda.Event()]
        used = [False, False]
        stream = torch.cuda.current_stream(device)
        row0, it = 0, 0
        for t in shards:
            n = int(t.shape[1])
            for a in range(0, n, width):
                w = min(width, n - a)
                k = it & 1
                if used[k]:
                    done[k].synchronize()                      # the pinned buffer is free again
                src = t[:, a:a + w]
                stage[k][:, :w].copy_(src if src.dtype == torch.float16 else src.to(torch.float16))   # the disk read
                dstage[k][:, :w].copy_(stage[k][:, :w], non_blocking=True)
                done[k].record(stream)
                used[k] = True
                view = dstage[k][:, :w]
                target = tstage[k][:w] if host else bank[row0 + a:row0 + a + w]
                if w % 2 == 0:
                    check(lib().atlas_b200_transpose(view.data_ptr(), view.stride(0), target.data_ptr(), target.stride(0),
                                                     EMBEDDINGS_DIM, w, EMBEDDINGS_DIM, ctypes.c_void_p(stream.cuda_stream)))
                else:   # odd tail width: the transpose kernel moves 2-column words
                    target.copy_(view.t())
                if host:
                    bank[row0 + a:row0 + a + w].copy_(target, non_blocking=True)
                it += 1
            row0 += n
        torch.cuda.current_stream(device).synchronize()
        return bank

    # ------------------------------------------------------------------ search
    def _compute_scores_and_indices(self, allqueries: torch.Tensor, topk: int):
        """src/index.py:113-120 semantics (fp16 scores of `allqueries.half() @ embeddings`, row top-k),
        fused.  Returns (scores [nq, k] fp16 desc, indices [nq, k] int64 LOCAL row numbers)."""
        return ops.search_shard(self._bank, allqueries, topk, 0, 1, self._workspace)

    def _merge(self, blob_all, ids_off, world, nq_total, topk, q_begin, nq_out):
        return ops.topk_merge_blob(blob_all, ids_off, world, nq_total, topk, q_begin, nq_out, torch.float16)

    def _owner_local(self, gid, world):
        if self._offsets is None:
            return gid % world, gid // world
        r = int(np.searchsorted(self._offsets, gid, side="right")) - 1
        return r, gid - int(self._offsets[r])

    def _local_search(self, allqueries, topk, exhaustive=False):
        """Local shard scan returning GLOBAL ids + the device status word (no host synchronisation)."""
        return ops.mips_topk(self._bank, allqueries, topk, self._id_base, self._id_stride, self._workspace,
                             exhaustive=exhaustive)

    @torch.no_grad()
    def search_device(self, queries, topk, return_status=False, exhaustive=False):
        """Device half of `search_knn`: (scores [nq_local, k] fp16, global ids [nq_local, k] int64) as CUDA tensors.

        Collective when world_size > 1: ONE all-gather of the query rows + ONE all-gather of the packed per-shard
        (scores | ids | status) blobs (the reference: 3 + 4*W collectives with pickled passages, src/index.py:127-143).
        With `max_queries_per_rank` set there is no host synchronisation at all; otherwise one scalar size exchange.

        return_status=False: the overflow flag of the fast path is read here (one host sync) and the exhaustive path is
        re-run if needed, so the result is final.  return_status=True: nothing synchronises; the third return value is a
        device int64 scalar (max over shards) that the caller checks at its own synchronisation point
        (`search_knn` folds it into the D2H copy it needs anyway) and, if non-zero, calls again with exhaustive=True."""
        if self._bank is None:
            raise AtlasB200Error("search_knn before init_embeddings/load_index")
        if topk > MAX_TOPK:
            raise AtlasB200Error(f"topk={topk} > {MAX_TOPK}")
        if topk > self._bank.shape[0]:
            # torch.topk in the reference raises the same way (src/index.py:118)
            raise RuntimeError(f"selected index k out of range: topk={topk} > local bank size {self._bank.shape[0]}")
        world = dist_utils.get_world_size()
        rank = dist_utils.get_rank()
        queries = queries.reshape(-1, EMBEDDINGS_DIM)
        nq_local = queries.shape[0]
        if world == 1:
            s, i, status = self._local_search(queries, topk, exhaustive)
            status = status.to(torch.int64).reshape(())
        else:
            q16 = queries.to(self._query_device()).to(torch.float16)                  # `.half()`, src/index.py:117
            cap = self.max_queries_per_rank
            if cap:
                if nq_local > cap:
                    raise AtlasB200Error(f"search_knn: {nq_local} queries on this rank but max_queries_per_rank={cap} "
                                         "(set it to the per-GPU batch size, identical on every rank, or to None)")
                if nq_local < cap:
                    q16 = torch.cat([q16, q16.new_zeros((cap - nq_local, EMBEDDINGS_DIM))], dim=0)
                allq = dist_utils.all_gather_fixed(q16).reshape(world * cap, EMBEDDINGS_DIM)     # all_gather #1, no sync
                nq_total, q_begin = world * cap, rank * cap
            else:
                sizes = dist_utils.get_varsize(queries)                            # tiny all_gather (+ host sync)
                allq = dist_utils.varsize_all_gather(q16, sizes)                   # all_gather #1
                nq_total, q_begin = int(sum(sizes)), int(sum(sizes[:rank]))
            s_loc, i_loc, st_loc = self._local_search(allq, topk, exhaustive)
            blob, ids_off, st_off = ops.pack_results(s_loc, i_loc, st_loc.to(torch.int64))
            blob_all = dist_utils.all_gather_fixed(blob)                           # all_gather #2
            s, i = self._merge(blob_all, ids_off, world, nq_total, topk, q_begin, nq_local)
            status = blob_all[:, st_off:].contiguous().view(torch.int64).max()
        if return_status:
            return s, i, status
        if not exhaustive and int(status.item()) != 0:      # identical on every rank (max over shards): collective retry
            return self.search_device(queries, topk, exhaustive=True)
        return s, i

    @torch.no_grad()
    def search_knn(self, queries, topk):
        """Exhaustive k-nearest-neighbour search by inner product (src/index.py:122-157).

        Collective: every rank must call it, also with 0 queries (src/atlas.py:103-106).
        Returns (docs: List[nq][k] passage dicts, scores: List[nq][k] floats, descending)."""
        world = dist_utils.get_world_size()
        nq_local = queries.reshape(-1, EMBEDDINGS_DIM).shape[0]
        scores, ids, status = self.search_device(queries, topk, return_status=True)
        # the overflow flag (max over shards, identical on every rank) is read at the host sync the results need anyway
        scores_host = scores.float().cpu()
        ids_host = ids.cpu()
        if int(status.item()) != 0:                         # massive ties (e.g. an all-zero bank): exact chunked path
            scores, ids, _ = self.search_device(queries, topk, return_status=True, exhaustive=True)
            scores_host, ids_host = scores.float().cpu(), ids.cpu()
        ids_host = ids_host.tolist()
        flat = [self._owner_local(g, world) for row in ids_host for g in row]
        docs_flat = self._get_store().lookup(flat)
        docs = [docs_flat[r * topk:(r + 1) * topk] for r in range(nq_local)]
        return docs, scores_host.tolist()

    def is_index_trained(self) -> bool:  # src/index.py:159-160
        return True

    def train_index(self):
        return None


def _check_nprobe(index_type, nprobe):
    """nprobe: None (every list) or an int >= 1 (not a bool), and None for types pq and flat, which have no lists."""
    if nprobe is not None and (isinstance(nprobe, bool) or not isinstance(nprobe, int) or nprobe < 1):
        raise AtlasB200Error(f"DistributedFAISSIndex: nprobe={nprobe!r} must be None (every list) or an integer >= 1")
    if nprobe is not None and index_type in ("pq", "flat"):
        raise AtlasB200Error(f"DistributedFAISSIndex({index_type!r}): nprobe={nprobe!r} needs inverted lists; index type "
                             f"{index_type} has none (use ivfpq, ivfsq or ivfflat, or nprobe=None)")
    return nprobe


class DistributedFAISSIndex(DistributedIndex):
    """`--index_mode faiss` (src/index.py:163-381) with a product-quantized index on the device (csrc/pq.cu).

    index_type "pq": `code_size` one-byte sub-quantizer codes per passage; "ivfpq": floor(sqrt(N_local)) coarse centroids
    (inner-product assignment) and PQ codes of the residuals.  The reference probes every inverted list
    (nprobe = n_list, src/index.py:212,269), so a search scores every row: sum_m LUT[m][code_m] (+ <q, c_list>), fp32,
    rounded once to fp16 - the same scores faiss's IndexPQ / IVFPQ produce, up to the fp32 summation order.

    Memory: the full-precision rows stay in pinned HOST memory as [N, 768] fp16 (`embeddings` is the reference's
    [768, N] view of them, `is_in_gpu = False`).  The device holds M bytes of codes (plus 2 bytes of list id for ivfpq)
    per passage, the codebooks and the coarse centroids; training and encoding stage host chunks through a transient
    device buffer.

    Training: `train_index()` retrains both quantizers (k-means, faiss's defaults, deterministic) on the current rows and
    re-encodes every row.  After writing rows by hand (`index.embeddings[:, a:b] = ...`) call `train_index()` again;
    `Atlas.build_index` does this itself (it marks the index stale, as the reference's inverted `is_index_trained`
    makes it do after every refresh, src/atlas.py:86-88).  Searching an untrained index raises.

    Persistence: `save_index` writes the reference's `embeddings.{s}.pt` / `passages.{s}.pt` shards and, per rank,
    `index{type}_{code_size}_rank_{r}.atlas_b200.pt` (format version, type, M, n_list, row count, codebooks, coarse
    centroids, codes, list ids).  `load_index` uses that file when type, M and row count match and retrains otherwise;
    a reference `.faiss` file is not read (faiss's format is not reproduced here).

    Refinement (faiss IndexRefineFlat / `k_factor`, opt-in): with `refine_factor` R > 1 (a constructor keyword and a plain
    attribute that may be set at any time; Atlas sets it from `--faiss_refine_factor`) each rank takes its top
    k' = min(k * R, N_local) rows by PQ score, re-scores them against their full-precision host rows (read zero-copy over
    the host link, csrc/pq_refine.cu) and keeps its top k by that exact score; the ranks' lists are then merged as
    before, which gives the exact top k of the union of the candidates.  The scores returned are then the exact inner
    products rounded once to fp16 (the flat index's scores up to the fp32 summation order), not PQ scores.  k' must
    not exceed MAX_TOPK.  No per-passage device memory is added; nothing is added to the index files.  `status` and the
    exhaustive retry refer to the candidate search; the retry refines too.  R = 1 (default) runs the PQ search alone.

    index_type "ivfsq" (faiss IndexIVFScalarQuantizer, QT_4bit, residual encoding): the ivfpq coarse quantizer, then each
    residual dim in 4 bits between the per-dim min and max of the training residuals, scored by faiss's decode rule and
    rounded once to fp16 (csrc/ivfsq.cu, include/atlas_b200.h).  `code_size` is bits per dimension (faiss's SQ4 naming):
    None or 4.  The device holds 384 bytes of codes and a 4-byte row id per slot, in inverted-list order with every list
    padded to a multiple of 64 slots; the index file holds the codes in row order and faiss's packing, with the list
    ids, and `load_index` rebuilds the slot layout from them.  Training needs one row.

    index_type "ivfflat" (faiss IndexIVFFlat, inner product): the ivfpq coarse quantizer and the full-precision rows on
    the device in ivfsq's inverted-list slot layout (fp16 rows in place of codes, csrc/ivfflat.cu): 1536 bytes of row and
    a 4-byte row id per slot, every list padded to a multiple of 64 slots.  Its scores are the flat index's, bit for bit:
    the inner product of the fp16 query and row, accumulated in fp32 and rounded once to fp16, with no coarse term; with
    `nprobe` it scores only the rows of each query's best lists, so it loses recall on the lists it skips and no precision
    on the lists it scans.  An IVF-Flat index has no code: `code_size` must be None.  `refine_factor` is accepted and
    ignored (the scores are already exact), as the flat index ignores `--faiss_refine_factor`.  The index file holds the
    coarse centroids and the row-order list ids, and `load_index` rebuilds the slot layout from the shards' rows.
    Training needs one row.
    index_type "flat" (faiss IndexFlatIP, the reference's default `--faiss_index_type`): ivfflat with one list and no
    k-means - the rows in row order, padded to a multiple of 64 - always fully scanned; a non-None `nprobe` raises.  Its
    results are `DistributedIndex.search_knn`'s, with the rows kept in host memory between trainings.

    Probing (faiss's `nprobe`, opt-in, ivfpq, ivfsq and ivfflat): with `nprobe` an int >= 1 (a constructor keyword and a
    plain attribute that may be set at any time; Atlas sets it from `--faiss_nprobe`) each query is scored only against the
    rows of its best lists: the shortest prefix of the lists ordered by the coarse term <q, c_l> (descending, then list
    id) that has at least `nprobe` lists and holds at least k rows (faiss would return id -1 when the probed lists hold
    fewer than k rows instead; see include/atlas_b200.h).  The result is the exact top-k over those rows, and the sweep
    reads only the codes of lists some query of the block probes.  None (default) or nprobe >= n_list scans every row,
    as before.  Types pq and flat have no lists: a non-None value raises.  Refinement composes (the probed search supplies
    the k' candidates).  ivfpq keeps its codes in row order and reads them through a list-order permutation built on the first
    probed search: +4 bytes per row of device memory from then on, dropped with the index on retraining or
    `mark_stale()`.  `nprobe` is not written to the index file."""

    SUPPORTED_TYPES = ("pq", "ivfpq", "ivfsq", "ivfflat", "flat")
    FILE_FORMAT = 1
    TRAIN_SEED = 1234
    STAGE_ROWS = 65536

    def __init__(self, index_type: str = "flat", code_size: Optional[int] = None, refine_factor: int = 1,
                 nprobe: Optional[int] = None):
        if index_type not in self.SUPPORTED_TYPES:
            raise AtlasB200Error(
                f"DistributedFAISSIndex: index_type={index_type!r} is not provided by atlas_b200; supported types are "
                f"{', '.join(self.SUPPORTED_TYPES)}.  For exact search use --index_mode flat "
                "(atlas_b200.index.DistributedIndex)")
        if index_type in ("ivfflat", "flat"):
            # checked before the device, so that the error does not depend on the machine
            if code_size is not None:
                raise AtlasB200Error(f"DistributedFAISSIndex({index_type!r}): code_size={code_size!r}, but an {index_type} "
                                     "index stores full-precision rows and has no code: pass None (--faiss_code_size "
                                     "unset).  For the exact search with the rows on the device use --index_mode flat "
                                     "(atlas_b200.index.DistributedIndex)")
        elif index_type == "ivfsq":
            # faiss's SQ4 naming: code_size is bits per dimension; the reference builds QT_4bit whatever its value
            if code_size is not None and (isinstance(code_size, bool) or code_size != ops.SQ_BITS):
                raise AtlasB200Error(f"DistributedFAISSIndex('ivfsq'): code_size={code_size!r} is bits per dimension and "
                                     f"the scalar quantizer is {ops.SQ_BITS}-bit: pass None or {ops.SQ_BITS}.  For exact "
                                     "search use --index_mode flat (atlas_b200.index.DistributedIndex)")
        elif code_size is None:
            raise AtlasB200Error(f"DistributedFAISSIndex({index_type!r}) needs a code_size (--faiss_code_size)")
        else:
            ops.pq_check_code_size(code_size)
        _check_nprobe(index_type, nprobe)
        super().__init__()
        self._device()                 # no CUDA device: raise here, like the flat index (no CPU path)
        self.index_type = index_type
        self.code_size = None if code_size is None else int(code_size)
        self.is_in_gpu = False
        # the trained index: dict(codebooks, coarse, codes, list_ids, n_list) for pq / ivfpq;
        # dict(coarse, vmin, vdiff, codes, slot_rows, tile_lists, n_list) in the device slot layout for ivfsq;
        # dict(coarse (None for flat), rows, slot_rows, tile_lists, n_list) in the same layout for ivfflat / flat
        self._pq = None
        self.refine_factor = refine_factor
        self._refine_factor()
        self.nprobe = nprobe
        self._nprobe()

    # ------------------------------------------------------------------ host rows
    @property
    def embeddings(self):
        return None if self._bank is None else self._bank.t()

    @embeddings.setter
    def embeddings(self, value):
        if value is None:
            self._bank = None
        else:
            if value.dim() != 2 or value.shape[0] != EMBEDDINGS_DIM:
                raise ValueError(f"embeddings must be [{EMBEDDINGS_DIM}, N], got {tuple(value.shape)}")
            self._bank = self._host_rows(value.shape[1])
            self._bank.copy_(value.t())
        self._pq = None

    def _host_rows(self, n):
        rows = torch.zeros((n, EMBEDDINGS_DIM), dtype=torch.float16)
        return rows.pin_memory() if torch.cuda.is_available() else rows

    def _query_device(self):
        return self._device()

    def init_embeddings(self, passages, dim: Optional[int] = EMBEDDINGS_DIM):
        if dim != EMBEDDINGS_DIM:
            raise ValueError(f"only dim={EMBEDDINGS_DIM} is supported (src/retrievers.py:13)")
        self.doc_map = {i: doc for i, doc in enumerate(passages)}
        self._bank = self._host_rows(len(passages))
        self._id_base, self._id_stride = dist_utils.get_rank(), dist_utils.get_world_size()
        self._offsets = None
        self._pq = None
        self._reset_store()

    def _load_rows(self, files, device):
        if device.type == "cuda":
            return self._load_bank_streamed(files, device, host=True)
        rows = [torch.load(f, map_location="cpu").t().to(torch.float16) for f in files]
        return torch.cat(rows, dim=0).contiguous()

    # ------------------------------------------------------------------ training
    def is_index_trained(self) -> bool:
        return self._pq is not None

    def mark_stale(self):
        """The rows changed: the next `is_index_trained()` is False and searching raises until `train_index()`."""
        self._pq = None

    def n_list(self, n_rows=None):
        n = self._bank.shape[0] if n_rows is None else n_rows
        if self.index_type == "flat":
            return 1
        return int(math.floor(math.sqrt(n))) if self.index_type in ("ivfpq", "ivfsq", "ivfflat") else 0

    def _min_train_rows(self):
        """faiss's k-means needs 256 points per PQ centroid; IVF-SQ and IVF-Flat need one row per list, i.e. one row."""
        return ops.PQ_KSUB if self.index_type in ("pq", "ivfpq") else 1

    def train_index(self):
        """Train the quantizers on the current rows and encode every row (src/index.py:352-381 trains + adds)."""
        if self._bank is None:
            raise AtlasB200Error("train_index before init_embeddings/load_index")
        n = self._bank.shape[0]
        if n < self._min_train_rows():
            raise AtlasB200Error(f"train_index: {n} rows on this rank; index type {self.index_type} needs at least "
                                 f"{self._min_train_rows()} training points (faiss raises the same way)")
        self._pq = None
        if self.index_type == "ivfsq":
            self._pq = self._train_and_encode_sq(self._bank, n)
        elif self.index_type in ("ivfflat", "flat"):
            self._pq = self._train_flat(self._bank, n)
        else:
            self._pq = self._train_and_encode(self._bank, n)

    def _sample(self, rows, n, n_sample, device):
        """The first n_sample rows of the seeded permutation, on the device."""
        perm = np.random.default_rng(self.TRAIN_SEED).permutation(n)[:n_sample]
        return rows[torch.from_numpy(perm)].to(device)

    def _stream_rows(self, rows, n, device, fn):
        """fn(chunk, a, b) for the pinned host rows [a, b), staged through two device buffers of STAGE_ROWS rows."""
        width = min(self.STAGE_ROWS, n)
        stage = [torch.empty((width, EMBEDDINGS_DIM), dtype=torch.float16, device=device) for _ in range(2)]
        for it, a in enumerate(range(0, n, width)):
            b = min(n, a + width)
            st = stage[it & 1][: b - a]
            st.copy_(rows[a:b], non_blocking=True)       # pinned source; the stream orders the reuse of `st`
            fn(st, a, b)
        torch.cuda.current_stream(device).synchronize()

    def _train_and_encode(self, rows, n):
        device = self._device()
        n_list = self.n_list(n)
        sample = self._sample(rows, n, min(n, max(ops.PQ_KSUB * ops.PQ_KSUB, ops.PQ_KSUB * n_list)), device)
        codebooks, coarse = ops.pq_train(sample, self.code_size, n_list)
        del sample
        codes = torch.empty((n, self.code_size), dtype=torch.uint8, device=device)
        list_ids = torch.empty(n, dtype=ops.pq_list_dtype(n_list), device=device) if n_list else None
        ws = ops.Workspace()
        self._stream_rows(rows, n, device, lambda st, a, b: ops.pq_encode(st, codebooks, coarse, codes[a:b],
                                                                          list_ids[a:b] if n_list else None, ws))
        return dict(codebooks=codebooks, coarse=coarse, codes=codes, list_ids=list_ids, n_list=n_list)

    def _train_and_encode_sq(self, rows, n):
        """IVF-SQ: coarse k-means and ranges on the seeded sample, then two passes over the rows: their lists (which
        fix the slot layout), then their codes straight into their slots."""
        device = self._device()
        n_list = self.n_list(n)
        sample = self._sample(rows, n, min(n, max(ops.SQ_RANGE_MAX, ops.PQ_KSUB * n_list)), device)
        coarse, vmin, vdiff = ops.ivfsq_train(sample, n_list)
        del sample
        ws = ops.Workspace()
        lists = torch.empty(n, dtype=torch.int32, device=device)
        self._stream_rows(rows, n, device,
                          lambda st, a, b: ops.ivfsq_encode(st, coarse, vmin, vdiff, list_ids=lists[a:b], workspace=ws))
        slot_rows, tile_lists, row_slot = ops.ivfsq_layout(lists, n_list)
        del lists
        codes = torch.zeros((slot_rows.numel(), ops.SQ_CODE_BYTES), dtype=torch.uint8, device=device)
        self._stream_rows(rows, n, device, lambda st, a, b: ops.ivfsq_encode(st, coarse, vmin, vdiff, row_slot=row_slot[a:b],
                                                                             codes=codes, workspace=ws))
        return dict(coarse=coarse, vmin=vmin, vdiff=vdiff, codes=codes, slot_rows=slot_rows, tile_lists=tile_lists,
                    n_list=n_list)

    def _train_flat(self, rows, n):
        """IVF-Flat: the coarse k-means of ivfpq / ivfsq on the same seeded sample rows, the rows' lists; type flat puts
        every row in list 0 without k-means."""
        device = self._device()
        n_list = self.n_list(n)
        lists = torch.zeros(n, dtype=torch.int32, device=device)
        coarse = None
        if self.index_type == "ivfflat":
            sample = self._sample(rows, n, min(n, ops.PQ_KSUB * n_list), device)
            coarse = ops.ivfflat_train(sample, n_list)
            del sample
            ws = ops.Workspace()
            self._stream_rows(rows, n, device, lambda st, a, b: ops.ivf_list_ids(st, coarse, lists[a:b], ws))
        return self._flat_layout(rows, n, coarse, lists, n_list)

    def _flat_layout(self, rows, n, coarse, lists, n_list):
        """The slot layout of the list ids `lists` (ivfsq's), then the pinned host rows scattered into their slots."""
        device = self._device()
        slot_rows, tile_lists, row_slot = ops.ivfsq_layout(lists, n_list)
        del lists
        dev_rows = torch.zeros((slot_rows.numel(), EMBEDDINGS_DIM), dtype=torch.float16, device=device)
        self._stream_rows(rows, n, device,
                          lambda st, a, b: dev_rows.index_copy_(0, row_slot[a:b].to(torch.int64), st))
        return dict(coarse=coarse, rows=dev_rows, slot_rows=slot_rows, tile_lists=tile_lists, n_list=n_list)

    def _flat_list_ids(self, p, n):
        """Row-order list ids of the IVF-Flat layout."""
        slots = torch.nonzero(p["slot_rows"] >= 0).flatten()
        lists = torch.empty(n, dtype=torch.int32, device=slots.device)
        lists[p["slot_rows"][slots].to(torch.int64)] = p["tile_lists"][slots // ops.SQ_TILE]
        return lists

    # ------------------------------------------------------------------ search
    def _trained(self):
        if self._pq is None:
            raise AtlasB200Error("search_knn on an untrained DistributedFAISSIndex: call train_index() after writing rows")
        return self._pq

    def _refine_factor(self):
        r = self.refine_factor
        if isinstance(r, bool) or not isinstance(r, int) or r < 1:
            raise AtlasB200Error(f"DistributedFAISSIndex: refine_factor={r!r} must be an integer >= 1 (1 = no refinement)")
        return r

    def _nprobe(self):
        return _check_nprobe(self.index_type, self.nprobe)

    def _probe_tables(self, p, nprobe):
        """The list tables of a probed search, built on the first one and kept in the trained index (dropped with it)."""
        if nprobe is None or nprobe >= p["n_list"]:
            return {}
        if self.index_type in ("ivfsq", "ivfflat"):
            if "list_tile_off" not in p:
                p["list_tile_off"], p["list_rows"] = ops.ivfsq_list_tables(p["slot_rows"], p["tile_lists"], p["n_list"])
            return dict(list_tile_off=p["list_tile_off"], list_rows=p["list_rows"])
        if "list_order" not in p:
            p["list_order"], p["list_offsets"] = ops.ivfpq_list_tables(p["list_ids"], p["n_list"])
        return dict(list_order=p["list_order"], list_offsets=p["list_offsets"])

    def _local_search(self, allqueries, topk, exhaustive=False):
        self._nprobe()
        r = self._refine_factor()
        if r == 1 or self.index_type in ("ivfflat", "flat"):     # the scores are exact already: nothing to refine
            return self._candidate_search(allqueries, topk, self._id_base, self._id_stride, exhaustive)
        k_cand = min(topk * r, int(self._bank.shape[0]))
        if k_cand > MAX_TOPK:
            raise AtlasB200Error(f"DistributedFAISSIndex: refine_factor={r} x topk={topk} = {topk * r} candidates per "
                                 f"query exceed MAX_TOPK={MAX_TOPK}; lower refine_factor or topk")
        _, cand, status = self._candidate_search(allqueries, k_cand, 0, 1, exhaustive)
        s, i = self._refine(allqueries, cand, topk)
        return s, i, status

    def _candidate_search(self, allqueries, k, id_base, id_stride, exhaustive):
        """Top k by the index's score: (scores, ids = id_base + id_stride * row, device status word)."""
        p = self._trained()
        nprobe = self._nprobe()
        tables = self._probe_tables(p, nprobe)
        if self.index_type in ("ivfflat", "flat"):
            return ops.ivfflat_topk(p["rows"], p["slot_rows"], p["tile_lists"], int(self._bank.shape[0]), p["coarse"],
                                    allqueries, k, id_base, id_stride, self._workspace, exhaustive=exhaustive, nprobe=nprobe,
                                    **tables)
        if self.index_type == "ivfsq":
            return ops.ivfsq_topk(p["codes"], p["slot_rows"], p["tile_lists"], int(self._bank.shape[0]), p["coarse"],
                                  p["vmin"], p["vdiff"], allqueries, k, id_base, id_stride, self._workspace,
                                  exhaustive=exhaustive, nprobe=nprobe, **tables)
        return ops.pq_topk(p["codes"], p["list_ids"], p["codebooks"], p["coarse"], allqueries, k, id_base, id_stride,
                           self._workspace, exhaustive=exhaustive, nprobe=nprobe, **tables)

    def _refine(self, allqueries, cand_local, topk):
        """Top `topk` of the candidate rows `cand_local` [nq, k'] by exact score: (scores, global ids)."""
        return ops.pq_refine_topk(self._bank, allqueries, cand_local, topk, self._id_base, self._id_stride,
                                  self._workspace)

    # ------------------------------------------------------------------ persistence
    def _index_file_stem(self) -> str:
        """src/index.py:175-182: `index{type}_{code_size}_rank_{r}`, without the code size when it is None."""
        size = f"_{self.code_size}" if self.code_size else ""
        return f"index{self.index_type}{size}_rank_{dist_utils.get_rank()}"

    def _get_index_filename(self, path: str) -> str:
        """The reference's `.faiss` name with this format's own suffix."""
        return os.path.join(path, f"{self._index_file_stem()}.atlas_b200.pt")

    def _get_faiss_index_filename(self, path: str) -> str:
        return os.path.join(path, f"{self._index_file_stem()}.faiss")

    def save_index(self, path: str, total_saved_shards: int, overwrite_saved_passages: bool = False) -> None:
        super().save_index(path, total_saved_shards, overwrite_saved_passages)
        if self._pq is None:
            return
        p = self._pq
        cpu = lambda t: None if t is None else t.cpu()
        if self.index_type in ("ivfflat", "flat"):
            n = int(self._bank.shape[0])
            torch.save(dict(format=self.FILE_FORMAT, index_type=self.index_type, code_size=self.code_size,
                            n_list=p["n_list"], n_rows=n, coarse=cpu(p["coarse"]), list_ids=cpu(self._flat_list_ids(p, n))),
                       self._get_index_filename(path))
            return
        if self.index_type == "ivfsq":
            codes, lists = ops.ivfsq_export(p["codes"], p["slot_rows"], p["tile_lists"], int(self._bank.shape[0]))
            torch.save(dict(format=self.FILE_FORMAT, index_type=self.index_type, code_size=self.code_size,
                            n_list=p["n_list"], n_rows=int(self._bank.shape[0]), coarse=cpu(p["coarse"]),
                            vmin=cpu(p["vmin"]), vdiff=cpu(p["vdiff"]), codes=cpu(codes), list_ids=cpu(lists)),
                       self._get_index_filename(path))
            return
        torch.save(dict(format=self.FILE_FORMAT, index_type=self.index_type, code_size=self.code_size, n_list=p["n_list"],
                        n_rows=int(self._bank.shape[0]), codebooks=cpu(p["codebooks"]), coarse=cpu(p["coarse"]),
                        codes=cpu(p["codes"]), list_ids=cpu(p["list_ids"])),
                   self._get_index_filename(path))

    def load_index(self, path: str, total_saved_shards: int):
        """Loads the shards into the host rows, then the index file if it matches (type, M, row count); else retrains."""
        super().load_index(path, total_saved_shards)
        self._pq = None
        f = self._get_index_filename(path)
        n = int(self._bank.shape[0])
        if os.path.exists(f):
            d = torch.load(f, map_location="cpu")
            if (d.get("format") == self.FILE_FORMAT and d.get("index_type") == self.index_type
                    and d.get("code_size") == self.code_size and d.get("n_rows") == n
                    and d.get("n_list") == self.n_list(n)):
                dev = self._device()
                to = lambda t: None if t is None else t.to(dev)
                if self.index_type in ("ivfflat", "flat"):
                    lists = to(d["list_ids"]).to(torch.int32).contiguous()
                    if tuple(lists.shape) != (n,):
                        raise AtlasB200Error(f"{f}: list_ids must hold {n} entries, got {tuple(lists.shape)}")
                    self._pq = self._flat_layout(self._bank, n, to(d["coarse"]), lists, int(d["n_list"]))
                    return
                if self.index_type == "ivfsq":
                    codes, slot_rows, tile_lists = ops.ivfsq_import(to(d["codes"]), to(d["list_ids"]), int(d["n_list"]))
                    self._pq = dict(coarse=to(d["coarse"]), vmin=to(d["vmin"]), vdiff=to(d["vdiff"]), codes=codes,
                                    slot_rows=slot_rows, tile_lists=tile_lists, n_list=int(d["n_list"]))
                    return
                self._pq = dict(codebooks=to(d["codebooks"]), coarse=to(d["coarse"]), codes=to(d["codes"]),
                                list_ids=to(d["list_ids"]), n_list=int(d["n_list"]))
                return
            logger.info(f"{f} does not match this index (type {self.index_type}, code_size {self.code_size}, {n} rows): "
                        "retraining")
        elif os.path.exists(self._get_faiss_index_filename(path)):
            logger.info(f"{self._get_faiss_index_filename(path)} is a faiss file, which atlas_b200 does not read: retraining")
        if n >= self._min_train_rows():
            self.train_index()
