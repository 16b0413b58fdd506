/* atlas_b200 — C ABI of the H100-native (sm_90a) retrieve-then-read hot path.
 *
 * The reference (facebookresearch/atlas) is pure Python and has no FFI; its boundary for this path
 * is the Python module surface.  This header is the C-ABI layer underneath our
 * drop-in Python modules (`atlas_b200/index.py` etc.): plain pointers and sizes, no torch types.
 * Every entry point cites the reference code it replaces.
 *
 * Conventions
 *   - return value: 0 = ATLAS_B200_OK, otherwise an ATLAS_B200_E* code; `atlas_b200_last_error()`
 *     returns a thread-local human-readable message.  Entry points never exit() or throw.
 *   - all device pointers must belong to the current CUDA device; work is enqueued on `stream`
 *     (a cudaStream_t passed as void*; NULL = legacy default stream) and is asynchronous unless
 *     stated otherwise.
 *   - memory is owned by the caller; kernels borrow pointers for the duration of the launch.
 */
#ifndef ATLAS_B200_H
#define ATLAS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ATLAS_B200_OK 0
#define ATLAS_B200_EINVAL 1      /* bad argument (k > n, misaligned pointer, ...)            */
#define ATLAS_B200_ECUDA 2       /* a CUDA runtime / driver call failed                      */
#define ATLAS_B200_EWORKSPACE 3  /* workspace too small                                      */
#define ATLAS_B200_EUNSUPPORTED 4

#define ATLAS_B200_EMBEDDINGS_DIM 768 /* src/retrievers.py:13 */
#define ATLAS_B200_MAX_TOPK 1024

const char* atlas_b200_last_error(void);
const char* atlas_b200_version(void);

/* Number of kernel launches issued by this library since load (bench.py's `gpu_launches`). */
uint64_t atlas_b200_launch_count(void);

/* --------------------------------------------------------------------------------------------
 * Exact max-inner-product search over one shard of the passage bank.
 *
 * Replaces `DistributedIndex._compute_scores_and_indices` (src/index.py:113-120):
 *     scores = torch.matmul(allqueries.half(), self.embeddings); torch.topk(scores, topk, dim=1)
 * Semantics kept: fp16 operands, fp32 accumulation, ONE rounding of each score to fp16, selection on
 * the fp16-rounded scores.  Tie order (unspecified in the reference) is pinned: score descending,
 * then id ascending.  The [nq, n] score matrix is never materialised.
 *
 *   bank        device, [n, 768] row-major (row = passage = one column of the reference's
 *               `embeddings[768, n]`), fp16 (is_bf16 = 0) or bf16 (1); 16-byte aligned.
 *   ld          row stride of `bank` in elements (>= 768, multiple of 8).
 *   queries     device, [nq, 768] row-major, same dtype as the bank, 16-byte aligned.
 *   out_scores  device, [nq, k] in the bank dtype, descending.
 *   out_ids     device, [nq, k] int64 = id_base + id_stride * row   (global line number of the
 *               passage under the round-robin sharding of src/index_io.py:41 when
 *               id_base = rank, id_stride = world_size).
 *   status      device int32[1]: 0 on success; 1 if the candidate buffers overflowed (pathological
 *               tie/ordering patterns) — results are then INVALID and the caller must call
 *               atlas_b200_mips_topk_exhaustive().  Written on `stream`.
 *   workspace   device scratch of at least atlas_b200_mips_workspace_bytes(n, nq, k) bytes.
 * nq == 0 is allowed (no-op): every rank must call search every step (src/atlas.py:103-106).
 * -------------------------------------------------------------------------------------------- */
size_t atlas_b200_mips_workspace_bytes(int64_t n, int32_t nq, int32_t k);

int atlas_b200_mips_topk(const void* bank, int64_t n, int64_t ld, int32_t is_bf16,
                         const void* queries, int32_t nq, int32_t k,
                         void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride,
                         int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* Same contract, exact for ANY input (chunked scan, no thresholds); slower.  Used as the fallback
 * when `status` reports overflow.  Synchronous with respect to nothing: enqueued on `stream`. */
int atlas_b200_mips_topk_exhaustive(const void* bank, int64_t n, int64_t ld, int32_t is_bf16,
                                    const void* queries, int32_t nq, int32_t k,
                                    void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride,
                                    void* workspace, size_t workspace_bytes, void* stream);

/* Merge of W per-shard top-k lists (replaces the second `torch.topk` over the concatenated
 * [nq, W*k] candidates, src/index.py:144-156).  Shard w's lists are scores_in + w*shard_stride_scores
 * ([nq_total, k] 16-bit) and ids_in + w*shard_stride_ids ([nq_total, k] int64) — strides in elements,
 * so the blob produced by ONE NCCL all-gather of each rank's (scores | ids) buffer can be used in
 * place.  Rows [q_begin, q_begin+nq_out) of every shard list are merged with the canonical order
 * (score desc, id asc) into out_scores / out_ids [nq_out, k]. */
int atlas_b200_topk_merge(const void* scores_in, const int64_t* ids_in,
                          int64_t shard_stride_scores, int64_t shard_stride_ids, int32_t is_bf16,
                          int32_t world, int32_t nq_total, int32_t k,
                          int32_t q_begin, int32_t nq_out,
                          void* out_scores, int64_t* out_ids, void* stream);

/* End-to-end search of one shard with HOST buffers (the call bench.py times as `e2e`):
 * queries_host [nq, 768] fp32 (what the reference's live retriever emits) are converted with
 * round-to-nearest-even (`.half()`, src/index.py:117), copied to the device, searched, and the
 * results copied back.  Synchronous.  out_scores_host is fp32 holding the fp16/bf16 values
 * (`scores.tolist()`, src/index.py:152). */
int atlas_b200_search_host(const void* bank, int64_t n, int64_t ld, int32_t is_bf16,
                           const float* queries_host, int32_t nq, int32_t k,
                           float* out_scores_host, int64_t* out_ids_host,
                           int64_t id_base, int64_t id_stride,
                           void* workspace, size_t workspace_bytes, void* stream);

/* --------------------------------------------------------------------------------------------
 * Product-quantized passage index (csrc/pq.cu): `DistributedFAISSIndex` with index_type pq / ivfpq
 * (src/index.py:163-381; faiss IndexPQ / GpuIndexIVFPQ with 8-bit codes and nprobe = n_list).
 *
 *   M          code_size: sub-quantizers of 256 centroids each; M divides 768 and dsub = 768 / M >= 8.
 *   n_list     coarse centroids (ivfpq), 0 = pq.  The reference probes every list, so a search scans all rows.
 *   codebooks  device fp32 [M][256][dsub];  coarse: device fp32 [n_list][768] (NULL for pq).
 *   codes      device uint8 [n, M] (4-byte aligned when M % 4 == 0);  list_ids: device [n] uint16 when
 *              n_list <= 65535, else int32 (NULL for pq).
 *   scores     fp32 LUTs <q_m, cb_m[j]> and coarse terms <q, c_l> from the fp16 queries; each row's score is
 *              sum_m LUT[m][code_m] (m ascending, fp32) + <q, c_list>, rounded ONCE to fp16.
 *
 * atlas_b200_pq_train: k-means with faiss's defaults on the device.  `sample` [n_sample, 768] fp16 holds the
 *   training rows in a seeded random order: the coarse quantizer (inner-product assignment, plain means) is trained
 *   on the first min(n_sample, 256 n_list) rows, the product quantizer (L2 per sub-space) on the residuals of the
 *   first min(n_sample, 65536); the first rows are the initial centroids; empty clusters are split off the largest
 *   one.  Bitwise deterministic.  n_sample >= max(256, n_list).
 * atlas_b200_pq_encode: codes (and list ids) of n fp16 rows [n, 768] - call it chunk by chunk.
 * atlas_b200_pq_topk / _exhaustive: atlas_b200_mips_topk's contract (fp16 scores desc, ids = id_base +
 *   id_stride * row, canonical tie order, `status` overflow flag and the exhaustive retry) over these scores.
 * Workspace: atlas_b200_pq_workspace_bytes(op, n, M, n_list, k) with n = n_sample (train), unused (encode) or the
 *   row count (search); 0 for an unsupported M.
 * -------------------------------------------------------------------------------------------- */
#define ATLAS_B200_PQ_OP_TRAIN 0
#define ATLAS_B200_PQ_OP_ENCODE 1
#define ATLAS_B200_PQ_OP_SEARCH 2
#define ATLAS_B200_PQ_OP_SEARCH_PROBED 3
size_t atlas_b200_pq_workspace_bytes(int32_t op, int64_t n, int32_t M, int32_t n_list, int32_t k);
int atlas_b200_pq_train(const void* sample, int64_t n_sample, int32_t M, int32_t n_list, int32_t iters,
                        float* codebooks, float* coarse, void* workspace, size_t workspace_bytes, void* stream);
int atlas_b200_pq_encode(const void* rows, int64_t n, int32_t M, const float* codebooks, const float* coarse,
                         int32_t n_list, uint8_t* codes, void* list_ids, void* workspace, size_t workspace_bytes,
                         void* stream);
int atlas_b200_pq_topk(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M, const float* codebooks,
                       const float* coarse, int32_t n_list, const void* queries, int32_t nq, int32_t k,
                       void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride, int32_t* status,
                       void* workspace, size_t workspace_bytes, void* stream);
int atlas_b200_pq_topk_exhaustive(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M,
                                  const float* codebooks, const float* coarse, int32_t n_list, const void* queries,
                                  int32_t nq, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                                  int64_t id_stride, void* workspace, size_t workspace_bytes, void* stream);

/* --------------------------------------------------------------------------------------------
 * Probed IVF search (`nprobe`, csrc/ivf_probe.cu) for ivfpq and ivfsq (the ivfsq tables are below).
 *
 *   T[q][l]    the fp32 coarse term the scan adds to every row of list l: <q, c_l> from the fp16-rounded query.
 *   order(q)   the lists sorted by T[q][l] descending, then by list id ascending.
 *   P(q)       the shortest prefix of order(q) with at least nprobe lists (empty lists count) that holds at least k
 *              real rows.  Unlike faiss, which returns id -1 when the probed lists hold fewer than k rows, the prefix
 *              is extended; as k <= n, it always exists.
 *   result     the exact top-k of the full search's contract (scores, canonical tie order) over the rows whose list
 *              is in P(q).  It does not depend on the other queries of the call.  Probe sets grow by prefix with
 *              nprobe, so each position of a query's sorted top-k scores is non-decreasing in nprobe.
 *   nprobe     >= 1; nprobe >= n_list runs the full search (atlas_b200_pq_topk / atlas_b200_ivfsq_topk) unchanged.
 *
 * Per block of <= 256 queries: one CTA per query selects P(q) (a radix select on (T, list id), then the extension),
 * the lists some query probes are compacted into the sweep's work items, and their count stays in device memory: the
 * scan and select grids are sized from an upper bound, so nothing synchronises with the host (graph-capturable).
 * The candidate bound of the sampled path comes from each query's own best probed lists (their first max(512, k)
 * positions, until they hold max(k, 4 k |P(q)| / capq) of its rows), so large probe sets do not overflow it.
 * The list tables are trusted: they must describe the same layout as the codes (offsets non-decreasing from 0 to n,
 * or to n_tiles for ivfsq; list_order a permutation of the rows).  Other tables can make the compaction write past
 * its workspace.
 *
 * atlas_b200_pq_topk_probed / _exhaustive: the arguments of atlas_b200_pq_topk plus
 *   list_order    device int32 [n]: the rows sorted by list id, stable (rows of a list ascending);
 *   list_offsets  device int32 [n_list + 1]: list l holds list_order[list_offsets[l] .. list_offsets[l + 1]);
 *   nprobe.       n_list must be >= 1.  A work item is 512 consecutive positions of one list.
 * Workspace: atlas_b200_pq_workspace_bytes(ATLAS_B200_PQ_OP_SEARCH_PROBED, n, M, n_list, k) (0 when n_list < 1).
 * -------------------------------------------------------------------------------------------- */
int atlas_b200_pq_topk_probed(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M, const float* codebooks,
                              const float* coarse, int32_t n_list, const int32_t* list_order, const int32_t* list_offsets,
                              int32_t nprobe, const void* queries, int32_t nq, int32_t k, void* out_scores,
                              int64_t* out_ids, int64_t id_base, int64_t id_stride, int32_t* status, void* workspace,
                              size_t workspace_bytes, void* stream);
int atlas_b200_pq_topk_probed_exhaustive(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M,
                                         const float* codebooks, const float* coarse, int32_t n_list,
                                         const int32_t* list_order, const int32_t* list_offsets, int32_t nprobe,
                                         const void* queries, int32_t nq, int32_t k, void* out_scores, int64_t* out_ids,
                                         int64_t id_base, int64_t id_stride, void* workspace, size_t workspace_bytes,
                                         void* stream);

/* --------------------------------------------------------------------------------------------
 * IVF-SQ passage index (csrc/pq.cu, csrc/ivfsq.cu): `DistributedFAISSIndex` with index_type ivfsq (faiss
 * IndexIVFScalarQuantizer with QT_4bit, residual encoding, inner product, nprobe = n_list).
 *
 *   n_list      coarse centroids (>= 1), coarse: device fp32 [n_list][768], trained as for ivfpq.
 *   vmin/vdiff  device fp32 [768]: per-dim min and max - min of the residuals r = fp32(x) - coarse[list(x)].
 *   layout      rows in inverted-list order: stable-sorted by list, every list padded to a multiple of 64 slots, so
 *               each 64-slot tile belongs to one list.  codes: device uint8 [n_tiles * 64][384], 16-byte aligned,
 *               nibbles permuted inside a slot (csrc/ivfsq.cuh); slot_rows: device int32 [n_tiles * 64], the local
 *               row of each slot or -1 for padding; tile_lists: device int32 [n_tiles].
 *   code        xi = (r_d - vmin_d) / vdiff_d (0 when vdiff_d == 0) clamped to [0, 1]; code_d = (int)(xi * 15.0) in
 *               double, as faiss does.
 *   score       w^[q][d] = fp16(2^e_q * q_d * (vdiff_d / 15)) with e_q putting max_d |w^| in [2^14, 2^15);
 *               C[q] = sum_d q_d (vmin_d + 0.5 vdiff_d / 15) + 2^-e_q * 8 sum_d w^[q][d] and T[q][l] = <q, c_l>
 *               in fp32;  s = fp16(T[q][list] + C[q] + 2^-e_q * sum_d w^[q][d] (code_d - 8)), the last sum accumulated
 *               in fp32 on the tensor cores.
 *               This is faiss's decode rule sum_d q_d (vmin_d + (code_d + 0.5) / 15 vdiff_d) + <q, c_l> to about one
 *               fp16 ulp of the largest score.
 *
 * atlas_b200_ivfsq_train: `sample` [n_sample, 768] fp16 in a seeded random order, n_sample >= n_list: the coarse
 *   k-means of atlas_b200_pq_train on the first min(n_sample, 256 n_list) rows, then vmin / vdiff over the residuals
 *   of the first min(n_sample, 100000).  Bitwise deterministic.  vmin = vdiff = NULL: the coarse k-means alone (the
 *   IVF-Flat index below).
 * atlas_b200_ivfsq_encode: for n fp16 rows [n, 768] (call it chunk by chunk), the coarse assignment (inner product,
 *   lowest list on ties) into list_ids (int32 [n], may be NULL) and, when `codes` is not NULL, each row's 384 code
 *   bytes into slot row_slot[i] of `codes` (row_slot: int32 [n]).
 * atlas_b200_ivfsq_topk / _exhaustive: atlas_b200_mips_topk's contract (fp16 scores desc, ids = id_base + id_stride *
 *   row, canonical tie order, `status` overflow flag and the exhaustive retry) over the n_rows real rows; padding
 *   slots are never returned.  k <= n_rows.
 * Workspace: atlas_b200_ivfsq_workspace_bytes(op, n, n_list, k) with op ATLAS_B200_PQ_OP_TRAIN (n = n_sample),
 *   _ENCODE (n unused) or _SEARCH (n = n_tiles * 64); 0 when n_list < 1.
 * -------------------------------------------------------------------------------------------- */
size_t atlas_b200_ivfsq_workspace_bytes(int32_t op, int64_t n, int32_t n_list, int32_t k);
int atlas_b200_ivfsq_train(const void* sample, int64_t n_sample, int32_t n_list, int32_t iters, float* coarse, float* vmin,
                           float* vdiff, void* workspace, size_t workspace_bytes, void* stream);
int atlas_b200_ivfsq_encode(const void* rows, int64_t n, const float* coarse, int32_t n_list, const float* vmin,
                            const float* vdiff, int32_t* list_ids, const int32_t* row_slot, uint8_t* codes, void* workspace,
                            size_t workspace_bytes, void* stream);
int atlas_b200_ivfsq_topk(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists, int64_t n_tiles,
                          int64_t n_rows, const float* coarse, int32_t n_list, const float* vmin, const float* vdiff,
                          const void* queries, int32_t nq, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                          int64_t id_stride, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);
int atlas_b200_ivfsq_topk_exhaustive(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists,
                                     int64_t n_tiles, int64_t n_rows, const float* coarse, int32_t n_list, const float* vmin,
                                     const float* vdiff, const void* queries, int32_t nq, int32_t k, void* out_scores,
                                     int64_t* out_ids, int64_t id_base, int64_t id_stride, void* workspace,
                                     size_t workspace_bytes, void* stream);
/* atlas_b200_ivfsq_topk_probed / _exhaustive: the probed IVF search above over the ivfsq layout; the arguments of
 * atlas_b200_ivfsq_topk plus
 *   list_tile_off  device int32 [n_list + 1]: list l owns tiles list_tile_off[l] .. list_tile_off[l + 1];
 *   list_rows      device int32 [n_list]: the real rows of list l;
 *   nprobe.        A work item is one 64-slot tile; a 128-query group of the scan skips tiles none of its queries probes.
 * Workspace: atlas_b200_ivfsq_workspace_bytes(ATLAS_B200_PQ_OP_SEARCH_PROBED, n_tiles * 64, n_list, k). */
int atlas_b200_ivfsq_topk_probed(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists, int64_t n_tiles,
                                 int64_t n_rows, const int32_t* list_tile_off, const int32_t* list_rows, const float* coarse,
                                 int32_t n_list, const float* vmin, const float* vdiff, int32_t nprobe, const void* queries,
                                 int32_t nq, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                                 int64_t id_stride, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);
int atlas_b200_ivfsq_topk_probed_exhaustive(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists,
                                            int64_t n_tiles, int64_t n_rows, const int32_t* list_tile_off,
                                            const int32_t* list_rows, const float* coarse, int32_t n_list, const float* vmin,
                                            const float* vdiff, int32_t nprobe, const void* queries, int32_t nq, int32_t k,
                                            void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride,
                                            void* workspace, size_t workspace_bytes, void* stream);

/* --------------------------------------------------------------------------------------------
 * IVF-Flat passage index (csrc/pq.cu, csrc/ivfflat.cu): `DistributedFAISSIndex` with index_type ivfflat (faiss
 * IndexIVFFlat, inner product) and flat (faiss IndexFlatIP: the same layout with one list, always fully scanned).
 *
 *   n_list      coarse centroids (>= 1), coarse: device fp32 [n_list][768], trained by atlas_b200_ivfsq_train with
 *               vmin = vdiff = NULL (the coarse quantizer of ivfpq / ivfsq); list ids by atlas_b200_ivfsq_encode with
 *               codes = NULL.
 *   layout      ivfsq's with fp16 rows in place of codes: rows stable-sorted by list, every list padded to a multiple of
 *               64 slots, so each 64-slot tile belongs to one list.  rows: device fp16 [n_tiles * 64][768], 16-byte
 *               aligned, padding slots zero; slot_rows: device int32 [n_tiles * 64], the local row of each slot or -1
 *               for padding.  (tile_lists, int32 [n_tiles], is not an argument of the search: the probed search takes
 *               its lists from list_tile_off.)
 *   score       s = fp16(<q, x>) of the fp16 query and the fp16 row, accumulated in fp32 on the tensor cores: the flat
 *               index's score (atlas_b200_mips_topk), bit for bit with the same operands.  No coarse term is added.
 *   probe       the probed IVF search above, with T[q][l] = <q, c_l> in fp32 from the fp16-rounded query - ivfsq's T,
 *               which here only chooses P(q): for the same coarse quantizer and lists, ivfflat and ivfsq probe the same
 *               lists.  The result is the exact top-k by s over the rows whose list is in P(q).
 *
 * atlas_b200_ivfflat_topk / _exhaustive: atlas_b200_mips_topk's contract (fp16 scores desc, ids = id_base + id_stride *
 *   row, canonical tie order, `status` overflow flag and the exhaustive retry) over the n_rows real rows; padding slots
 *   are never returned.  k <= n_rows.
 *   nprobe         0 or >= n_list: every row (the full scan; coarse, list_tile_off and list_rows are unused and may be
 *                  NULL); 1 <= nprobe < n_list: the probed search, with
 *   list_tile_off  device int32 [n_list + 1]: list l owns tiles list_tile_off[l] .. list_tile_off[l + 1];
 *   list_rows      device int32 [n_list]: the real rows of list l.  A work item is one 64-slot tile.
 * Workspace: atlas_b200_ivfflat_workspace_bytes(op, n_tiles * 64, n_list, k) with op ATLAS_B200_PQ_OP_SEARCH (full
 *   scan) or ATLAS_B200_PQ_OP_SEARCH_PROBED; 0 when n_list < 1.
 * -------------------------------------------------------------------------------------------- */
size_t atlas_b200_ivfflat_workspace_bytes(int32_t op, int64_t n_slots, int32_t n_list, int32_t k);
int atlas_b200_ivfflat_topk(const void* rows, const int32_t* slot_rows, int64_t n_tiles, int64_t n_rows,
                            const int32_t* list_tile_off, const int32_t* list_rows, const float* coarse, int32_t n_list,
                            int32_t nprobe, const void* queries, int32_t nq, int32_t k, void* out_scores, int64_t* out_ids,
                            int64_t id_base, int64_t id_stride, int32_t* status, void* workspace, size_t workspace_bytes,
                            void* stream);
int atlas_b200_ivfflat_topk_exhaustive(const void* rows, const int32_t* slot_rows, int64_t n_tiles, int64_t n_rows,
                                       const int32_t* list_tile_off, const int32_t* list_rows, const float* coarse,
                                       int32_t n_list, int32_t nprobe, const void* queries, int32_t nq, int32_t k,
                                       void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride, void* workspace,
                                       size_t workspace_bytes, void* stream);

/* Exact re-ranking of PQ search candidates (csrc/pq_refine.cu; faiss IndexRefineFlat, `k_factor`): for every query,
 * the k_cand candidate rows are re-scored against their full-precision rows and the top k are returned.
 *   rows_host   PINNED host memory, [n, 768] fp16 row-major, 16-byte aligned.  Read zero-copy by the kernel through
 *               cudaHostGetDevicePointer (ATLAS_B200_ECUDA if that fails); each candidate row is read once.
 *   queries     device fp16 [nq, 768], 16-byte aligned.
 *   cand_local  device int64 [nq, k_cand]: local row numbers (atlas_b200_pq_topk with id_base = 0, id_stride = 1),
 *               distinct within a query; entries outside [0, n) are skipped.  1 <= k <= k_cand <= ATLAS_B200_MAX_TOPK.
 *   scores      fp16( sum_d fp32(q_d) fp32(x_d) ): fp32 accumulation in a fixed order, rounded ONCE to fp16, i.e. the
 *               flat index's score up to the fp32 summation order; bitwise reproducible.
 *   out_scores  device fp16 [nq, k], descending;  out_ids: device int64 [nq, k] = id_base + id_stride * row, canonical
 *               tie order (score desc, id asc; id_stride >= 1).  Fewer than k valid candidates: -inf / -1 tail.
 *   workspace   device scratch of atlas_b200_pq_refine_workspace_bytes(nq, k_cand) bytes (at most 256 queries' worth).
 * nq == 0 is a no-op.  Reads of rows_host are ordered on `stream` after earlier work on it (e.g. copies into the rows). */
size_t atlas_b200_pq_refine_workspace_bytes(int32_t nq, int32_t k_cand);
int atlas_b200_pq_refine_topk(const void* rows_host, int64_t n, const void* queries, int32_t nq, const int64_t* cand_local,
                              int32_t k_cand, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                              int64_t id_stride, void* workspace, size_t workspace_bytes, void* stream);

/* --------------------------------------------------------------------------------------------
 * Dense linear layer with a fused epilogue on wgmma (csrc/gemm.cu):
 *     C[M, N] = epilogue( A[M, K] . W[N, K]^T )     A, W, C, bias, residual: fp16 (is_bf16 = 0) or bf16
 * W is the nn.Linear weight as stored by torch ([out_features, in_features]).  fp32 accumulation.
 * Replaces cuBLAS GEMM + ATen elementwise kernels behind the Linear layers of the Contriever encoder
 * (src/modeling_bert.py:280-466) and of FiD's T5 blocks (src/modeling_t5.py:272-289,418-531,1642-1647).
 *   epilogue  0 none | 1 +bias | 2 gelu_erf(+bias) (modeling_bert.py:444)
 *             | 3 +bias +residual[M, ldr] (dense + residual before LayerNorm)
 *             | 4 gated: C[m, j] = gelu_new(acc[m, 2j]) * acc[m, 2j+1], C has N/2 columns; W rows are
 *               wi_0 / wi_1 interleaved (modeling_t5.py:281-285; GELU evaluated in fp32 as at :283)
 *             | 5 relu: C = max(acc +bias, 0) (T5 v1.0 T5DenseReluDense wi, modeling_t5.py:256-270; with
 *               row_ss the row scale is applied first, then the bias and the ReLU)
 * lda / ldw / ldc / ldr are row strides in elements (multiples of 8); N and K multiples of 8.
 * bias may be NULL (no bias added) for epilogues 1-3 and 5.  The epilogues read the bias and the residual in pairs of
 * 16-bit values: a bias (epilogues 1-3, 5) or residual (epilogue 3) that is not 4-byte aligned is refused; C must be
 * 16-byte aligned.  A 4-byte but not 16-byte aligned residual runs a cooperative schedule (see below).
 * T5's RMSNorm (src/modeling_t5.py:244-253) fused around the GEMM, so the normalised activations never exist in memory:
 *   row_ss  device fp32 [M] = sum of squares of every A row, or NULL.  The accumulator row m is multiplied by
 *           rsqrt(row_ss[m] / K + rs_eps) before the epilogue: A holds the UN-normalised hidden states and the caller
 *           folds the norm weight into W (W'[n, k] = W[n, k] * ln_weight[k]).
 *   out_ss  device fp32 [M] or NULL (not with the gated epilogue): incremented by the sum of squares of the 16-bit values
 *           this launch stores in each row (zero it first) - the statistic of the NEXT norm, produced by the residual GEMM.
 * m_dev     device int32 [1] or NULL (= M): only the first min(M, *m_dev) rows are computed; row blocks past it are not, rows
 *           of the last computed block past *m_dev hold unspecified values.  The row count lives in device memory so that a
 *           captured CUDA graph keeps one launch shape for a data-dependent number of rows (the compacted encoders below). */
int atlas_b200_linear_rows(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, const void* residual,
                           int64_t ldr, void* C, int64_t ldc, int32_t M, int32_t N, int32_t K, int32_t epilogue,
                           int32_t is_bf16, const float* row_ss, float* out_ss, float rs_eps, const int32_t* m_dev, void* stream);

/* Which kernel schedule atlas_b200_linear_rows runs for an (M, N, K, epilogue) launch, with a 16-byte aligned
 * residual (an unaligned one falls back to a cooperative schedule):
 *   0  cooperative, 128 x 128 tiles       1  cooperative, 128 x 256 tiles      (decoder-sized launches)
 *   2  ping-pong, 128 x 128 tiles         3  wide, 128 x 256 tiles, TMA-store  (encoder-sized launches)
 * The environment variable ATLAS_B200_GEMM_SCHEDULE=pingpong|wide (read once per process) forces one of the two
 * encoder-sized schedules wherever either may run, to time them against each other. */
#define ATLAS_B200_GEMM_COOPERATIVE_128 0
#define ATLAS_B200_GEMM_COOPERATIVE_256 1
#define ATLAS_B200_GEMM_PINGPONG 2
#define ATLAS_B200_GEMM_WIDE 3
int atlas_b200_linear_schedule(int32_t M, int32_t N, int32_t K, int32_t epilogue);

/* Row-wise normalisation of 16-bit activations (csrc/elementwise.cu), one rounding point per torch op:
 *   kind 0  BertLayerNorm (src/modeling_bert.py:104-114): y = w * r16((x - mean) * rsqrt(mean(x^2) + eps)) + b
 *           — note the UNCENTRED second moment; callers pass the residual sum already rounded to 16 bits.
 *   kind 1  T5LayerNorm / RMSNorm (src/modeling_t5.py:244-253): y = w * r16(x * rsqrt(mean(x^2) + eps))
 * H a multiple of 8 up to 2048, ldx / ldy multiples of 8; x, weight, bias and y 16-byte aligned (16-byte vector accesses),
 * else ATLAS_B200_EINVAL before any launch. */
int atlas_b200_layernorm(const void* x, int64_t ldx, const void* weight, const void* bias, void* y, int64_t ldy,
                         int32_t rows, int32_t H, float eps, int32_t kind, int32_t is_bf16, void* stream);

/* BertEmbeddings.forward (src/modeling_bert.py:213-247): word + token_type + position embeddings
 * (16-bit adds in that order), BertLayerNorm.  input_ids / token_type_ids [batch, L] int64
 * (token_type_ids may be NULL = zeros); y [batch*L, H].  H a multiple of 8 up to 2048; the three tables, ln_weight, ln_bias
 * and y 16-byte aligned, else ATLAS_B200_EINVAL. */
int atlas_b200_bert_embed_ln(const int64_t* input_ids, const int64_t* token_type_ids, const void* word_emb,
                             const void* type_emb, const void* pos_emb, const void* ln_weight, const void* ln_bias,
                             void* y, int32_t batch, int32_t L, int32_t H, float eps, int32_t is_bf16, void* stream);

/* Contriever average pooling (src/retrievers.py:50-53): out[b] = sum_l mask[b,l]*x[b,l] / sum_l mask[b,l].
 * `out` rows may be strided (ld_out) so the result can be written straight into the passage bank. */
int atlas_b200_masked_mean_pool(const void* x, const int64_t* mask, void* out, int64_t ld_out, int32_t batch,
                                int32_t L, int32_t H, int32_t is_bf16, void* stream);

/* Single-token decode attention of FiD.generate (csrc/decode.cu; reference: transformers 4.18 `generate` with use_cache
 * through src/atlas.py:592-619, T5Attention.forward with past_key_value src/modeling_t5.py:418-531):
 *  decode_cross_attention_live  q [B, H*64] (one new token per sequence) against the cross K | V rows kv [B*Lk, ldkv]
 *      projected once per generation; grid = (ceil(Lk / chunk), H, B), chunk a multiple of 16; writes un-normalised fp32
 *      partials o_partial [B*chunks, H*64] and (max, sum) ml_partial [B*chunks, H, 2] for atlas_b200_attention_combine_ex with
 *      Lq = 1, splits = chunks.  HBM-bound: every K / V byte is read once per step (Lk * 2 * H*64 * 2 B per query and layer).
 *      tile_live: the live-tile flags of atlas_b200_cross_attention_stream (uint8 [B, ceil(Lk / 64)], NULL = all live); 64-key
 *      tiles of masked keys only are not read (a warp's 16-key group never straddles a tile).
 *  decode_self_attention   appends the new token's K | V (columns H*64.. of qkv [B, 3*H*64]) to cache [B, Tmax, 2*H*64] at
 *      row *t_dev and attends over keys 0..*t_dev with bias_delta [H, 2*Tmax-1] (T5 relative bias by offset, NULL = none).
 *      The step index lives in DEVICE memory so that one captured CUDA graph serves every step.
 *  decode_argmax           greedy pick as torch.argmax (a NaN beats every number; among equal values or among NaNs the lowest
 *      index wins; EOS banned while *t_dev + 1 < min_length, finished rows emit pad_id):
 *      seq[b, *t_dev + 1] = tok_in[b] = next; done[b] |= next == eos; then *t_dev += 1. */
int atlas_b200_decode_cross_attention_live(const void* q, int64_t ldq, const void* kv, int64_t ldkv, int32_t k_col0,
                                      int32_t v_col0, const float* add_mask, const uint8_t* tile_live, int32_t B, int32_t H, int32_t Lk,
                                      int32_t chunk, float scale, float* o_partial, float* ml_partial, int32_t is_bf16,
                                      void* stream);
int atlas_b200_decode_self_attention(const void* qkv, int64_t ldqkv, void* cache, int32_t Tmax, const int32_t* t_dev,
                                     const float* bias_delta, float scale, void* out, int64_t ldo, int32_t B, int32_t H,
                                     int32_t is_bf16, void* stream);

/* Opt-in FP8 (e4m3) cross K | V cache of KV-cached generation (csrc/kv_fp8.cu; FiD.generate(cross_kv_dtype="fp8")).  LOSSY:
 * the decoder attends over dequantized keys and values.  Format: codes kv8 uint8 [rows, ldkv8] holding e4m3fn (OCP, no inf,
 * max 448) in the columns of the 16-bit layout, and kv_scale fp32 [rows, ld_scale], one scale per (row, 64-column block):
 * block c = columns [64 c, 64 c + 64) (K of head h = block h, V of head h = block H + h in the 2*H*64-wide cross K | V).
 *  quantize_kv_e4m3  x [rows, ldx] 16-bit, n_blocks blocks of 64 values per row.  Per block, in fp32 with IEEE rounding:
 *      amax = max |x|, inv = 448 / amax, code = e4m3(x * inv) (round to nearest even, saturating), scale = amax / 448;
 *      amax == 0 -> scale 0 and codes 0; a NaN or inf in the block -> scale NaN and codes 0.  Dequantized value =
 *      float(e4m3(code)) * scale.  ldx and ldkv8 multiples of 8 elements.
 *  decode_cross_attention_e4m3  atlas_b200_decode_cross_attention_live over the codes: score_j = kscale_j * (q . k8_j) * scale
 *      + mask, value weight p_j * vscale_j (fp32).  k_col0 / v_col0 (multiples of 64) index kv8's columns; the scales of key
 *      row j are kv_scale[j * ld_scale + k_col0 / 64 + h] and [.. + v_col0 / 64 + h].  ldkv a multiple of 16 bytes.  Same
 *      partials and chunk rules.  Reads Lk * 2 * H * (64 + 4) bytes per query and layer (0.53x the 16-bit cache).
 *  cross_attention_stream_e4m3  atlas_b200_cross_attention_stream (Lq <= 64; the nb beams of a batch element in beam search)
 *      over the codes, same scale columns and alignment as above: the codes are converted exactly to the 16-bit type of q,
 *      kscale scales each column of S, vscale is folded into P before P is rounded to 16 bits (fp16: vscale <= 65504 / 448,
 *      as quantize_kv_e4m3 of an fp16 K | V yields). */
int atlas_b200_quantize_kv_e4m3(const void* x, int64_t ldx, int64_t rows, int32_t n_blocks, uint8_t* kv8, int64_t ldkv8,
                                float* kv_scale, int64_t ld_scale, int32_t is_bf16, void* stream);
int atlas_b200_decode_cross_attention_e4m3(const void* q, int64_t ldq, const uint8_t* kv8, int64_t ldkv, const float* kv_scale,
                                           int64_t ld_scale, int32_t k_col0, int32_t v_col0, const float* add_mask,
                                           const uint8_t* tile_live, int32_t B, int32_t H, int32_t Lk, int32_t chunk, float scale,
                                           float* o_partial, float* ml_partial, int32_t is_bf16, void* stream);
int atlas_b200_cross_attention_stream_e4m3(const void* q, int64_t ldq, int32_t q_col0, const uint8_t* kv8, int64_t ldkv,
                                           const float* kv_scale, int64_t ld_scale, int32_t k_col0, int32_t v_col0,
                                           const float* add_mask, const uint8_t* tile_live, int32_t B, int32_t H, int32_t Lq,
                                           int32_t Lk, int32_t chunk, float scale, float* o_partial, float* ml_partial,
                                           int32_t is_bf16, void* stream);
int atlas_b200_decode_argmax(const void* logits, int64_t ld, int32_t V, int64_t* seq, int64_t ld_seq, int64_t* tok_in,
                             uint8_t* done, int32_t* t_dev, int32_t eos_id, int32_t pad_id, int32_t min_length, int32_t B,
                             int32_t is_bf16, void* stream);

/* Beam-search decoding of FiD.generate(num_beams = nb > 1) (csrc/beam.cu; reference: transformers 4.18 `beam_search`,
 * `BeamSearchScorer`, `BeamHypotheses` with early_stopping = False).  R = B * nb rows, row r = b * nb + beam; the step index
 * t = *t_dev (cur_len = t + 1) lives in device memory so one captured CUDA graph serves every step.
 * Ancestry table anc int32 [2, R, Tmax], buffer (t & 1) current at step t: entry (r, j) is the cache slot row holding row r's
 * position j - its self K | V is cache[anc[r, j], j] and its token tok[anc[r, j], j] (tok int32 [R, Tmax]).  Beams are
 * reordered by rewriting this table, never by copying the K | V cache.
 *  decode_self_attention_beam  decode_self_attention over R rows with the history gathered through the ancestry: writes the new
 *      K | V at cache row (r, t), reads keys / values (anc[r, j], j) for j <= t.  Same arithmetic as decode_self_attention on the
 *      explicitly gathered cache (bit-identical).
 *  beam_topk    per row: log-prob = log_softmax(logits) in fp32 (rounded to the logits' 16-bit type when round_lp != 0),
 *      EOS -> -inf while t + 1 < min_length, + add_mask [R, ld_mask] fp32 (NULL = none; the prefix constraint, 0 / -inf),
 *      + beam_scores[r] in fp32 -> the row's top k candidates, cand_score fp32 / cand_tok int32 [R, k] (k <= 32).  Order: the
 *      larger score first, NaN above every number, among equal scores (or NaNs) the lower index; a token is always in [0, V)
 *      for V >= k.  lp_out (fp32 [R, V], NULL = not written) receives the processed log-probs before the beam score.
 *  beam_select  per batch element: merges its nb rows' candidates (k = 2 * nb, flat index beam * V + token, the same order)
 *      into the top 2 * nb and applies BeamSearchScorer.process: an EOS candidate at rank < nb becomes a hypothesis of length
 *      cur_len and score sum_logprob / cur_len ** length_penalty (fp64), one at rank >= nb is skipped, the others fill the nb
 *      beams -> beam_scores, tok_in int64 [R], parent int32 [R] (global row), tok[r, t + 1], anc buffer ((t + 1) & 1).
 *      Hypotheses (at most nb per batch element, list order = insertion number): hyp_score fp64 [B, nb], hyp_len, hyp_ins
 *      int32 [B, nb], hyp_tok int32 [B, nb, Tmax], hyp_state int32 [B, 2] = (count, next insertion number), hyp_worst fp64 [B]
 *      (initially 0, 0 and 1e9).  On overflow the lowest score goes (ties: the earliest inserted).  done[b] |= count == nb and
 *      worst >= best / cur_len ** length_penalty.  A finished batch element emits pad_id with score 0 and keeps its rows in
 *      place.  Then *t_dev += 1.  Requires 1 <= nb <= ATLAS_B200_MAX_BEAMS and V >= 2. */
#define ATLAS_B200_MAX_BEAMS 16
int atlas_b200_decode_self_attention_beam(const void* qkv, int64_t ldqkv, void* cache, int32_t Tmax, const int32_t* t_dev,
                                          const int32_t* anc, const float* bias_delta, float scale, void* out, int64_t ldo,
                                          int32_t R, int32_t H, int32_t is_bf16, void* stream);
int atlas_b200_beam_topk(const void* logits, int64_t ld, int32_t V, const float* add_mask, int64_t ld_mask,
                         const float* beam_scores, const int32_t* t_dev, int32_t eos_id, int32_t min_length, int32_t round_lp,
                         int32_t k, float* cand_score, int32_t* cand_tok, float* lp_out, int32_t R, int32_t is_bf16,
                         void* stream);
int atlas_b200_beam_select(const float* cand_score, const int32_t* cand_tok, int32_t B, int32_t nb, int32_t V,
                           float* beam_scores, int64_t* tok_in, int32_t* parent, uint8_t* done, int32_t* anc, int32_t* tok,
                           int32_t Tmax, int32_t* t_dev, double* hyp_score, int32_t* hyp_len, int32_t* hyp_ins,
                           int32_t* hyp_tok, int32_t* hyp_state, double* hyp_worst, int32_t eos_id, int32_t pad_id,
                           double length_penalty, void* stream);

/* Reader-input assembly from a device-resident passage token bank.  Replaces the per-step host work of
 * Atlas.tokenize_passages (src/atlas.py:261-280: bsz * n_context string formats + tokenizer calls, then H2D of
 * [bsz, n, L] int64 ids + mask):
 *   out_ids[b, j, :]  = (query_ids[b, :query_lens[b]] ++ bank_ids[rows[b*n + j], :bank_lens[..]])[: L-1] ++ [eos_id],
 *                       padded with pad_id;  out_mask[b, j, t] = 1 on the token positions (bool bytes).
 * rows[.] < 0 is the "" padding passage of encode_passages (src/atlas.py:26-39): EOS only.  bank_ids int32
 * [bank_rows, bank_ld], bank_lens int32 [bank_rows]; query_ids int64 [batch, ldq] (NULL = no query part). */
int atlas_b200_splice_tokens(const int32_t* bank_ids, const int32_t* bank_lens, int64_t bank_ld, int64_t bank_rows,
                             const int64_t* rows, const int64_t* query_ids, const int32_t* query_lens, int64_t ldq,
                             int32_t batch, int32_t n_ctx, int32_t L, int32_t eos_id, int32_t pad_id, int64_t* out_ids,
                             uint8_t* out_mask, void* stream);

/* Fused multi-head attention, head_dim 64, 0 < Lk <= 576 keys per segment (K and V stay resident in shared memory;
 * csrc/attention.cu):
 *   O[b,i,h,:] = softmax_j( scale*Q[b,i,h].K[b,j,h] + bias_delta[h, j-i+Lq-1] + add_mask[b,j] (+causal) ) V[b,j,h,:]
 * q / k / v point at row-major [B*L, ld] 16-bit buffers (e.g. the fused QKV projection output); head h
 * occupies columns [col0 + 64h, col0 + 64h + 64); strides and column offsets are multiples of 8 elements.
 * add_mask [B, Lk] fp32 additive (NULL = none), bias_delta [H, Lq+Lk-1] fp32 (NULL = none; T5 relative-position bias by
 * offset; Lq + Lk - 1 <= 1152), causal_value 0 = off, otherwise added where j > i (the reference adds -10000,
 * transformers 4.18 get_extended_attention_mask).
 *   lse_out         [B, H, Lq] fp32, the row log-sum-exp of the scores (natural log; NULL = not needed): all the backward
 *                   pass needs besides the output itself.  Not with split-KV partials (atlas_b200_attention_combine_ex
 *                   writes it then).
 *   split KV        the FiD decoder's cross-attention over n_ctx*L (= 15 360) keys (fid.py:298-349 /
 *                   src/modeling_t5.py:478-524): B = batch*splits key segments, q_div = splits (segment s reads the queries
 *                   of batch s / splits), and o_partial [B*Lq, H*64] / ml_partial [B*Lq, H, 2] fp32 (un-normalised output,
 *                   row max, row sum) are written instead of `out`; atlas_b200_attention_combine_ex merges them.  Otherwise
 *                   q_div = 1 and both partials NULL.
 *   dropout_p       dropout on the probabilities (training: src/modeling_t5.py:515-516, src/modeling_bert.py:354):
 *                   O = (keep o softmax(S)) V / (1 - p), lse_out is that of the un-dropped softmax.  keep[b, h, i, j] is a
 *                   function of (seed, offset, (b * H + h) * Lq + i, j) (csrc/dropout.cuh; j = key index over the whole key
 *                   range when the keys are split: segment s of `q_div` covers j = s * Lk ..., Lk % 32 == 0 required then);
 *                   atlas_b200_attention_bwd_train re-derives the same mask.  0 <= dropout_p < 1; 0 = no dropout.
 *   key_block_live  optional, uint8 [B, ceil(Lk / 64)]: 0 marks a 64-key block whose keys are ALL masked out (additive mask
 *                   <= -5000, softmax weight exactly 0 in fp32): it is neither loaded nor computed - identical results; every
 *                   row keeps at least one live block (see atlas_b200_cross_attention_stream).
 * Replaces BertSelfAttention.forward (src/modeling_bert.py:328-366, scale 1/8) and T5Attention.forward
 * (src/modeling_t5.py:478-524, scale 1) incl. the materialised scores / probabilities. */
int atlas_b200_attention_train(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                               const void* v, int64_t ldv, int32_t v_col0, void* out, int64_t ldo, const float* add_mask,
                               const float* bias_delta, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                               float causal_value, int32_t q_div, float* o_partial, float* ml_partial, float* lse_out,
                               float dropout_p, uint64_t seed, uint64_t offset, const uint8_t* key_block_live,
                               int32_t is_bf16, void* stream);
/* atlas_b200_attention_train for long key ranges: 0 < Lk <= 4096 keys per segment and Lq + Lk - 1 <= 8192 (the bias table
 * of atlas_b200_attention_bwd_train), same arguments and results except that there are no split-KV partials (q_div = 1).
 * K and V stream through shared memory in 64-key blocks instead of staying resident (csrc/attention.cu,
 * attention_long_kernel), so the key count is not bounded by shared memory.  The FiD encoder takes it for passages longer
 * than the 576 keys of atlas_b200_attention_train.  Strides and column offsets must be multiples of 8 elements; any violated
 * limit returns ATLAS_B200_EINVAL before a launch. */
int atlas_b200_attention_long(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                              const void* v, int64_t ldv, int32_t v_col0, void* out, int64_t ldo, const float* add_mask,
                              const float* bias_delta, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                              float causal_value, float* lse_out, float dropout_p, uint64_t seed, uint64_t offset,
                              const uint8_t* key_block_live, int32_t is_bf16, void* stream);

/* Merge of the split-KV partials (atlas_b200_attention_train with q_div = splits, atlas_b200_cross_attention_stream and the
 * decode cross-attention kernels): o_partial [B*splits*Lq, H*64] and ml_partial [B*splits*Lq, H, 2] fp32, row
 * (b * splits + s) * Lq + i for split s:  out[b,i,h,:] = sum_s e^(m_s-M) O_s / sum_s e^(m_s-M) l_s  (16-bit, row stride ldo),
 * and lse_out [B, H, Lq] fp32 = M + log(sum_s e^(m_s-M) l_s), the log-sum-exp over ALL splits (NULL = not needed). */
int atlas_b200_attention_combine_ex(const float* o_partial, const float* ml_partial, int32_t B, int32_t splits,
                                    int32_t Lq, int32_t H, void* out, int64_t ldo, float* lse_out, int32_t is_bf16,
                                    void* stream);

/* --------------------------------------------------------------------------------------------
 * Backward pass (training): what autograd derives in the reference's train.py step
 * (`Atlas.forward` -> `loss.backward()`, src/atlas.py:399-550) for the kernels above.  Weight and
 * input gradients of the linear layers are wgmma GEMMs (dX = dY . W: atlas_b200_linear_rows on W^T;
 * dW = dY^T . X: atlas_b200_linear_wgrad); the entry points below are the rest.
 * -------------------------------------------------------------------------------------------- */

/* Backward of atlas_b200_attention_train / atlas_b200_attention_long (any Lq / Lk, head_dim 64; csrc/attention_bwd.cu).
 * q / k / v / out as in the forward (out = the forward's result [B*Lq, H*64]); dout [B*Lq, H*64]; dq / dk / dv are written at
 * column offsets d?_col0 + 64h of [B*L, ld] buffers (so one [tokens, 3*H*64] buffer can receive dQ | dK | dV for a fused
 * projection).  dbias_delta [H, Lq+Lk-1] fp32 is INCREMENTED (zero it first; NULL = not needed; Lq + Lk - 1 <= 8192 with a
 * bias); lse / dsum are [B, H, Lq] fp32, both required: `lse` holds the forward's log-sum-exp (lse_out of the forward or of
 * atlas_b200_attention_combine_ex) and is only read - there is no path that recomputes it; `dsum` is scratch.  dropout_p /
 * seed / offset / key_block_live as in the forward: the same keep mask is re-derived, dead blocks are skipped.  For FiD's
 * cross-attention (src/fid.py:298-349) pass the un-split key range: B = batch, Lk = n_ctx * L; with dq_accum [B*Lq, H*64]
 * fp32 (zeroed, no dbias) the keys are split over several CTAs that add their partial dQ into dq_accum instead of writing
 * `dq` - the caller converts it to 16 bits (atlas_b200_cast_f32).
 * Replaces autograd through BertSelfAttention.forward (src/modeling_bert.py:328-366) and T5Attention.forward
 * (src/modeling_t5.py:478-524). */
int atlas_b200_attention_bwd_train(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                                   const void* v, int64_t ldv, int32_t v_col0, const void* out, int64_t ldo,
                                   const void* dout, int64_t lddo, void* dq, int64_t lddq, int32_t dq_col0, void* dk,
                                   int64_t lddk, int32_t dk_col0, void* dv, int64_t lddv, int32_t dv_col0,
                                   const float* add_mask, const float* bias_delta, float* dbias_delta, float* lse,
                                   float* dsum, float* dq_accum, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                                   float causal_value, float dropout_p, uint64_t seed, uint64_t offset,
                                   const uint8_t* key_block_live, int32_t is_bf16, void* stream);

/* Cross-attention statistics for retriever distillation (`cross_attention_forward`, src/fid.py:333-343): with
 * S = scale * Q K^T + add_mask and P = softmax over the Lk = n_ctx * L keys (lse = the forward's log-sum-exp [B, H, T],
 * atlas_b200_attention_combine_ex), the means over heads of S, P and ||V[b, j, h, :]|| * P -> three [B, T, Lk] fp32 maps
 * (`score_storage`, `prob_storage`, `normalized_score_storage`).  q [B*T, ldq], kv [B*Lk, ldkv] with K / V of head h at
 * columns k_col0 + 64h / v_col0 + 64h.  T <= 128.  (csrc/xattn_stats.cu) */
int atlas_b200_cross_attention_stats(const void* q, int64_t ldq, int32_t q_col0, const void* kv, int64_t ldkv,
                                     int32_t k_col0, int32_t v_col0, const float* add_mask, const float* lse,
                                     float* out_scores, float* out_probs, float* out_norms, int32_t B, int32_t H, int32_t T,
                                     int32_t Lk, float scale, int32_t is_bf16, void* stream);

/* Weight gradient of a Linear layer on wgmma (csrc/gemm.cu, MN-major operand descriptors):
 *     dW[N, K] = dY[tokens, N]^T . X[tokens, K]        16-bit operands, fp32 accumulation over the tokens
 * Both activations are read as they lie in memory (no transposes); dW is written in 16 bits like the reference's
 * bf16 gradients (`--precision bf16`, src/model_io.py:94-98).
 * Split-K: output tiles are few (N x K weights) and the contraction long (all tokens), so with `workspace` of at least
 * atlas_b200_linear_wgrad_workspace_bytes(tokens, N, K) bytes (device, 16-byte aligned) the token range is split over
 * several CTA groups whose fp32 partial tiles are summed and rounded once by a second kernel; workspace == NULL (or too
 * small) runs the un-split kernel. */
size_t atlas_b200_linear_wgrad_workspace_bytes(int32_t tokens, int32_t N, int32_t K);
int atlas_b200_linear_wgrad(const void* dY, int64_t lddy, const void* X, int64_t ldx, void* dW, int64_t lddw,
                            int32_t tokens, int32_t N, int32_t K, int32_t is_bf16, void* workspace,
                            size_t workspace_bytes, void* stream);

/* dst[c, r] = src[r, c] (16-bit elements) for r < R and 0 for R <= r < Rpad: the K-major operands of the weight-gradient
 * GEMM dW[N, K] = dY^T[N, M] . X[M, K] (contraction over the M tokens, padded to a multiple of 8). */
int atlas_b200_transpose(const void* src, int64_t lds, void* dst, int64_t ldd, int32_t R, int32_t C, int32_t Rpad,
                         void* stream);

/* out[n] += sum_m x[m, n]  (fp32; bias gradients of the Linear layers). */
int atlas_b200_colsum(const void* x, int64_t ld, float* out, int32_t M, int32_t N, int32_t is_bf16, void* stream);

/* Backward of atlas_b200_layernorm (same `kind`): dx = d(norm)/dx . (dy * w) (+ dres when given: the residual
 * branch's gradient, fused), dweight / dbias fp32 [H] INCREMENTED (dbias only for kind 0). */
int atlas_b200_layernorm_bwd(const void* x, int64_t ldx, const void* dy, int64_t lddy, const void* weight,
                             const void* dres, int64_t lddres, void* dx, int64_t lddx, float* dweight, float* dbias,
                             int32_t rows, int32_t H, float eps, int32_t kind, int32_t is_bf16, void* stream);

/* T5DenseGatedGeluDense (src/modeling_t5.py:281-285) on u [M, 2F] whose columns (2j, 2j+1) hold (x.wi_0[j], x.wi_1[j]):
 *   dg == NULL: out [M, F]  = r16(gelu_new(u0)) * u1        (training forward: the pre-activations are kept)
 *   dg != NULL: out [M, 2F] = (dg * u1 * gelu_new'(u0), dg * gelu_new(u0)) interleaved like u. */
int atlas_b200_gated_gelu(const void* u, int64_t ldu, const void* dg, int64_t lddg, void* out, int64_t ldo, int64_t M,
                          int32_t F, int32_t is_bf16, void* stream);

/* erf GELU (src/modeling_bert.py:444) on z [M, N]: dy == NULL: out = gelu(z); else out = dy * gelu'(z). */
int atlas_b200_gelu_erf(const void* z, int64_t ldz, const void* dy, int64_t lddy, void* out, int64_t ldo, int64_t M,
                        int32_t N, int32_t is_bf16, void* stream);

/* Backward of the T5 v1.0 ReLU (src/modeling_t5.py:264) from its saved OUTPUT g [M, N] (what linear's epilogue 5 wrote):
 * du = g > 0 ? dg : 0, a pure select (bit-exact).  N and the strides multiples of 8, pointers 16-byte aligned. */
int atlas_b200_relu_bwd(const void* g, int64_t ldg, const void* dg, int64_t lddg, void* du, int64_t lddu, int64_t M, int32_t N,
                        int32_t is_bf16, void* stream);

/* word + token_type + position embeddings WITHOUT the LayerNorm (src/modeling_bert.py:236-243): the training forward
 * keeps the sum for the LayerNorm backward.  H even; the three tables and y 4-byte aligned, else ATLAS_B200_EINVAL. */
int atlas_b200_bert_embed_sum(const int64_t* input_ids, const int64_t* token_type_ids, const void* word_emb,
                              const void* type_emb, const void* pos_emb, void* y, int32_t batch, int32_t L, int32_t H,
                              int32_t is_bf16, void* stream);

/* Embedding gradient: dst[index[row], :] += src[row, :] in fp32 (index == NULL: row % modulo, the position ids);
 * rows whose index equals skip_index (nn.Embedding padding_idx; -1 = none) or lies outside [0, table_rows) are dropped. */
int atlas_b200_scatter_add_rows(const int64_t* index, int32_t modulo, const void* src, int64_t lds, float* dst,
                                int64_t rows, int32_t H, int64_t skip_index, int64_t table_rows, int32_t is_bf16,
                                void* stream);

/* Backward of atlas_b200_masked_mean_pool: dx[b, l, :] = mask[b, l] ? demb[b, :] / sum_l mask[b, l] : 0. */
int atlas_b200_masked_mean_pool_bwd(const void* demb, int64_t ld_demb, const int64_t* mask, void* dx, int32_t batch,
                                    int32_t L, int32_t H, int32_t is_bf16, void* stream);

/* CrossEntropyLoss(ignore_index=-100) over 16-bit logits [rows, V] (src/modeling_t5.py:1650-1652):
 *   fwd: lse[row] = logsumexp(logits[row]), loss[row] = lse - logits[row, label] (0 for ignored rows); the caller
 *        divides the sum by the number of valid rows.
 *   bwd: dlogits[row, c] = (softmax(logits[row])[c] - [c == label]) * gscale[0] (0 for ignored rows); gscale is a
 *        device scalar (upstream gradient / number of valid rows), so no host synchronisation is needed. */
int atlas_b200_cross_entropy_fwd(const void* logits, int64_t ld, const int64_t* labels, float* lse, float* loss,
                                 int32_t rows, int32_t V, int32_t is_bf16, void* stream);
int atlas_b200_cross_entropy_bwd(const void* logits, int64_t ld, const int64_t* labels, const float* lse,
                                 const float* gscale, void* dlogits, int64_t ldd, int32_t rows, int32_t V, int32_t is_bf16,
                                 void* stream);

/* nn.Dropout on 16-bit hidden states in the TRAINING path (src/modeling_t5.py:266,286,310,561,960,1070;
 * src/modeling_bert.py:222,378,459):  out = (residual +) r16(keep ? x / (1 - p) : 0).  The keep decisions are a pure
 * function of (seed, offset, element position) - Philox4x32-7, 16-bit uniforms, realised drop rate round(p * 65536) / 65536
 * (csrc/dropout.cuh) - so the backward of y = dropout(x) is the same call on dy with the same (seed, offset).  row_tiles
 * (NULL: row r is row r): the rows are the packed rows of the padding-compacted encoder, row r is keyed as the padded row
 * 64 row_tiles[r / 64] + r % 64 (atlas_b200_segment_tile_scan's tile_src; M must be a multiple of 64).
 * atlas_b200_dropout_mask / atlas_b200_attention_dropout_mask export the keep masks (1 byte per element) of the
 * elementwise layout ([M, N]) and of the attention-probability layout ([B * H * Lq, Lk], see atlas_b200_attention_train)
 * for the parity tests. */
int atlas_b200_dropout(const void* x, int64_t ldx, const void* residual, int64_t ldr, void* out, int64_t ldo, int64_t M,
                       int32_t N, float p, uint64_t seed, uint64_t offset, const int32_t* row_tiles, int32_t is_bf16,
                       void* stream);
int atlas_b200_dropout_mask(uint8_t* out, int64_t M, int32_t N, float p, uint64_t seed, uint64_t offset, void* stream);
int atlas_b200_attention_dropout_mask(uint8_t* out, int64_t rows, int32_t Lk, float p, uint64_t seed, uint64_t offset,
                                      void* stream);

/* Multi-tensor optimiser step and gradient statistics of the training loop.  The work list is a device
 * table of (tensor index, chunk index) int32 pairs, `chunk_elems` elements per chunk (multiple of 4).
 *   atlas_b200_adamw_fp32copy: src/AdamWFP32Copy.py:79-169 for one param group - per element, on the fp32 master copy:
 *     g = grad * inv_scale; p *= decay; m = lerp(m, g, one_minus_beta1); v = beta2*v + one_minus_beta2*g*g;
 *     p -= step_size * m / (sqrt(v) / bias_correction2_sqrt + eps); param = cast(p)
 *     (torch.optim AdamW, amsgrad = False, maximize = False).  decay = 1 - lr*wd, 1 - beta and step_size = lr /
 *     bias_correction1 are passed as the caller computed them in DOUBLE precision (as torch does) and rounded once to fp32;
 *     step_size and bias_correction2_sqrt are per tensor (state["step"] may differ between parameters).
 *   atlas_b200_grad_stats: src/util.py:200-222 - stats[i] = (min |g|, max |g|, mean |g|, ||g||_2) per tensor in fp32 on the
 *     device (zeros for a tensor without gradient), instead of four `.item()` synchronisations per parameter. */
typedef struct {
    void* param;             /* the nn.Parameter's storage (param_kind: 0 fp32, 1 bf16, 2 fp16) */
    float* master;           /* state["float32copy"] */
    float* exp_avg;          /* state["exp_avg"] */
    float* exp_avg_sq;       /* state["exp_avg_sq"] */
    const void* grad;        /* p.grad (grad_kind: 0 fp32, 1 bf16, 2 fp16) */
    int64_t numel;
    int32_t param_kind, grad_kind;
    float step_size;              /* lr / (1 - beta1^step) */
    float bias_correction2_sqrt;  /* sqrt(1 - beta2^step) */
} AtlasB200AdamTensor;
typedef struct {
    const void* grad;        /* NULL: no gradient */
    int64_t numel;
    int32_t grad_kind, pad_;
} AtlasB200GradTensor;
int atlas_b200_adamw_fp32copy(const AtlasB200AdamTensor* descs_dev, const int32_t* chunks_dev, int32_t n_chunks,
                              int32_t chunk_elems, float decay, float beta2, float one_minus_beta1, float one_minus_beta2,
                              float eps, float inv_scale, void* stream);
int atlas_b200_grad_stats(const AtlasB200GradTensor* descs_dev, int32_t n_tensors, const int32_t* chunks_dev,
                          int32_t n_chunks, int32_t chunk_elems, float* stats, void* stream);

/* fp16 overflow clamp of the T5 blocks (src/modeling_t5.py:657-708: `if dtype == fp16 and isinf(h).any(): h = clamp(h,
 * +-(65504 - 1000))` after every sub-layer, three host synchronisations per block in the reference): in place on x [M, N]
 * fp16, decided on the device through `flag` (one int32 of scratch), no synchronisation.  row_ss (optional, [M] fp32) is
 * rewritten with the rows' sums of squares when (and only when) the clamp fires (fused-RMSNorm statistic).
 * m_dev (optional, device int32): only rows [0, min(max(*m_dev, 0), M)) are scanned, clamped and get a row_ss, the row count
 * atlas_b200_linear_rows computed (m_dev = NULL: all M).  It is read on the device, so a captured graph follows it.  x must be
 * 16-byte aligned. */
int atlas_b200_clamp_inf_fp16(void* x, int64_t ld, int64_t M, int32_t N, const int32_t* m_dev, int32_t* flag, float* row_ss,
                              void* stream);

/* FiD decoder cross-attention for FEW queries (Lq <= 64 target tokens) against Lk concatenated encoder keys per batch element
 * (src/fid.py:298-349 at the teacher-forced / training forward shape): an HBM-bound K / V stream.  q [B*Lq, ldq], kv [B*Lk, ldkv]
 * (k at k_col0 + 64 h, v at v_col0 + 64 h).  Every CTA covers `chunk` keys (multiple of 64) of one (batch, head) and writes
 * un-normalised fp32 partials o_partial [(b * chunks + c) * Lq + i, H*64] and ml_partial [.., H, 2] = (row max, row sum) in the
 * layout atlas_b200_attention_combine_ex merges (splits = ceil(Lk / chunk)).
 * tile_live (optional, uint8 [B, ceil(Lk / 64)]): 0 marks a 64-key tile whose keys are ALL masked out (additive mask <= -5000:
 * their probabilities are exactly 0 in fp32, the reference's `exp(-10000 + s - max)` underflows); such tiles are neither
 * loaded nor computed - same result, ~45 % fewer K / V bytes on text_maxlength-padded FiD passages.  A row of tile_live must
 * keep at least one live tile (the caller marks all tiles live for a fully masked batch element). */
int atlas_b200_cross_attention_stream(const void* q, int64_t ldq, int32_t q_col0, const void* kv, int64_t ldkv, int32_t k_col0,
                                      int32_t v_col0, const float* add_mask, const uint8_t* tile_live, int32_t B, int32_t H,
                                      int32_t Lq, int32_t Lk, int32_t chunk, float scale, float* o_partial, float* ml_partial,
                                      int32_t is_bf16, void* stream);

/* Compacted cross-attention K | V (FiD decoder, inference forward): only the encoder positions whose 64-key block holds a live
 * key are ever read by the cross-attention (atlas_b200_cross_attention_stream skips the others), so only they get a K | V
 * projection.  Everything keeps STATIC launch shapes (CUDA graphs): the live-row count lives in device memory.
 *   atlas_b200_compact_live_tiles: tile_off[t] = index of live 64-row tile t among the live tiles (-1 = dead), *count_rows =
 *     64 x #live; the rows of the live tiles of src [n_tiles * 64, d] are copied to dst rows [64 tile_off[t], +64), which
 *     atlas_b200_linear_rows with m_dev = count_rows then projects.
 *   atlas_b200_cross_attention_stream_compact: as atlas_b200_cross_attention_stream with kv holding only the live tiles:
 *     tile t of batch b starts at row 64 * tile_row[b * (Lk / 64) + t] (tile_row = the tile_off table above). */
int atlas_b200_compact_live_tiles(const void* src, int64_t lds, const uint8_t* tile_live, int32_t n_tiles, int32_t d, void* dst,
                                  int64_t ldd, int32_t* tile_off, int32_t* count_rows, void* stream);
int atlas_b200_cross_attention_stream_compact(const void* q, int64_t ldq, int32_t q_col0, const void* kv, int64_t ldkv,
                                              int32_t k_col0, int32_t v_col0, const float* add_mask, const uint8_t* tile_live,
                                              const int32_t* tile_row, int32_t B, int32_t H, int32_t Lq, int32_t Lk,
                                              int32_t chunk, float scale, float* o_partial, float* ml_partial, int32_t is_bf16,
                                              void* stream);

/* Padding-compacted FiD encoder (no-grad forward: fid.py FiD._encode_rows; training step: FiD._encode_train), for
 * text_maxlength L a multiple of 64 up to 576.  The reference encodes every passage padded to text_maxlength (src/atlas.py:261-270,
 * src/fid.py:32-78) and masks the padding keys; a padded position never influences a live one (its softmax weight is exactly 0,
 * every other encoder op is row-wise) and the decoder's cross-attention masks it too (so its gradients are exactly 0), so the
 * encoder runs on the 64-row tiles up to each segment's last live key only, packed back to back.  Static launch shapes: the
 * packed row count lives in device memory (the training step reads it to the host once per forward).
 *   atlas_b200_segment_tile_scan: live uint8 [S, nb] (key_block_live) -> keep [S, nb] (tiles 0 .. last live tile of the segment;
 *     all nb if none is live), tile_off int32 [S * nb] (packed index of a kept tile, -1 = dropped), tile_src int32 [S * nb] (source
 *     tile of packed tile o, -1 past the end), *count_rows = 64 x #kept.
 *   atlas_b200_embed_packed_tiles: dst[64 o + r, :] = table[ids[64 tile_src[o] + r], :] (zeros past the end): T5Stack's
 *     embed_tokens (src/modeling_t5.py:930-934) straight into the packed layout.
 *   The projections run on atlas_b200_linear_rows with m_dev = count_rows.
 *   atlas_b200_attention_packed: T5Attention.forward (src/modeling_t5.py:478-524) of the encoder on the packed rows: segment b =
 *     rows [64 tile_off[b * nb], + 64 popcount(keep[b, :])) of qkv / out; add_mask [B, L] and bias_delta [H, 2L - 1] as in
 *     atlas_b200_attention_train (positions are those of the padded layout: kept tiles are a prefix of the segment).  lse_out
 *     (or NULL): the row log-sum-exp [B, H, L] in the padded layout, written for the kept rows; dropout_p / seed / offset: dropout
 *     on the probabilities with the masks of atlas_b200_attention_train on the padded layout (row (b H + h) L + i, key j).
 *     L <= 384 without lse_out and dropout runs a persistent kernel; otherwise the resident kernel of atlas_b200_attention_train.
 *   atlas_b200_attention_packed_bwd: its backward, the contract of atlas_b200_attention_bwd_train for self-attention: lse
 *     (required, only read) and dsum scratch [B, H, L] in the padded layout, dbias_delta [H, 2L - 1] incremented (or NULL), the
 *     dropout masks re-derived, dropped tiles never touched.  qkv / dqkv hold q | k | v and dq | dk | dv at columns 0, 64 H and
 *     128 H; out / dout are the forward's output and its gradient.
 *   atlas_b200_expand_packed_tiles: back to the padded layout [S * nb * 64, d] (zeros at dropped tiles - the positions the
 *     reference fills with values nothing reads).
 * embed_packed_tiles, expand_packed_tiles and compact_live_tiles move 16-byte vectors: d and the row strides are multiples of 8
 * and table / src / dst 16-byte aligned, else ATLAS_B200_EINVAL. */
int atlas_b200_segment_tile_scan(const uint8_t* live, int32_t S, int32_t nb, uint8_t* keep, int32_t* tile_off, int32_t* tile_src,
                                 int32_t* count_rows, void* stream);
int atlas_b200_embed_packed_tiles(const int64_t* ids, const void* table, int64_t ldt, int32_t vocab, const int32_t* tile_src,
                                  int32_t n_tiles, void* dst, int64_t ldd, int32_t d, void* stream);
int atlas_b200_attention_packed(const void* qkv, int64_t ld, int32_t q_col0, int32_t k_col0, int32_t v_col0, void* out, int64_t ldo,
                                const float* add_mask, const float* bias_delta, const uint8_t* keep, const int32_t* tile_off,
                                int32_t B, int32_t H, int32_t L, float scale, float* lse_out, float dropout_p, uint64_t seed,
                                uint64_t offset, int32_t is_bf16, void* stream);
int atlas_b200_attention_packed_bwd(const void* qkv, int64_t ld, const void* out, int64_t ldo, const void* dout, int64_t lddo,
                                    void* dqkv, int64_t ldd, const float* add_mask, const float* bias_delta, float* dbias_delta,
                                    const float* lse, float* dsum, const uint8_t* keep, const int32_t* tile_off, int32_t B,
                                    int32_t H, int32_t L, float scale, float dropout_p, uint64_t seed, uint64_t offset,
                                    int32_t is_bf16, void* stream);
int atlas_b200_expand_packed_tiles(const void* src, int64_t lds, const int32_t* tile_off, int32_t n_tiles, void* dst, int64_t ldd,
                                   int32_t d, void* stream);

/* Measurement hook for bench.py's roofline: while enabled, every launch of ONE kind of kernel is bracketed
 * with CUDA events on its launching stream:
 *   kind 1  the bank sweep of atlas_b200_mips_topk (work = algorithmic bytes swept); also the code sweep of
 *           atlas_b200_ivfsq_topk (work = code bytes swept, once per 128 queries of a block)
 *   kind 2  the wgmma GEMM of atlas_b200_linear_rows (work = 2*M*N*K FLOPs over the computed rows)
 *   kind 3  the attention forward kernels: atlas_b200_attention_train / _long / _packed, the cross-attention stream
 *           kernels (work = 4*B*H*Lq*Lk*64 FLOPs)
 *   kind 4  the attention backward kernels           (work = 16*B*H*Lq*Lk*64 FLOPs)
 *   kind 5  the decode cross-attention kernels of atlas_b200_decode_cross_attention_live / _e4m3 (work = K | V bytes read:
 *           4*B*H*Lk*64, or 2*B*H*Lk*68 for the e4m3 codes and scales)
 *   kind 6  atlas_b200_beam_topk and atlas_b200_beam_select (work = bytes read: 2*R*V of logits, 16*B*nb*nb of candidates)
 *   kind 7  the refine kernel of atlas_b200_pq_refine_topk (work = host-row bytes read, nq * k_cand * 1536)
 *   kind 0  off (default).
 * atlas_b200_profile_work() returns the work summed over the bracketed launches so far;
 * atlas_b200_profile_collect() synchronises the events, returns the summed kernel time and the number of
 * bracketed launches, and resets the list (call profile_work first).  atlas_b200_profile_launches() (before collect) returns
 * each bracketed launch's time and work in launch order.  Not thread safe. */
void atlas_b200_profile_enable(int32_t kind);
int32_t atlas_b200_profile_launches(double* ms, double* work, int32_t cap);
double atlas_b200_profile_work(void);
int atlas_b200_profile_collect(double* total_ms, int32_t* launches);

/* fp32 -> fp16/bf16 row conversion (`allqueries.half()`), device to device. */
int atlas_b200_cast_f32(const float* src, void* dst, int64_t count, int32_t to_bf16, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ATLAS_B200_H */
