// Exact re-ranking of product-quantized search candidates against the full-precision rows (faiss IndexRefineFlat /
// `k_factor`) for `DistributedFAISSIndex(refine_factor > 1)`, sm_90a.
//
// The rows stay where the index keeps them, in pinned HOST memory ([n, 768] fp16).  The kernel reads each candidate row
// once, zero-copy over the host link, through the device alias of the host pointer (cudaHostGetDevicePointer).
//   score(q, x) = fp16( sum_d fp32(q_d) * fp32(x_d) )    fp32 accumulation, rounded ONCE to fp16: the flat index's score
//                                                        up to the fp32 summation order.
// Summation order (fixed, so a score is the same bits on every run): lane l of a warp holds the 16-byte chunks
// c = l, l + 32, l + 64 (dims [8c, 8c + 8)) of the query and of the row, accumulates them with fmaf in that order, then a
// xor butterfly over offsets 16, 8, 4, 2, 1 adds the 32 lane sums (every lane ends with the same bits).
// Selection: the refined (fp16 score, local row) pairs are written in mips.cu's candidate format and mips_select_kernel
// (SEL_EMIT) takes the canonical top-k - score descending, then id ascending - and writes id_base + id_stride * row.
//
// Latency hiding: a read of host memory takes microseconds.  Each warp owns ROWS_PER_WARP = 4 candidates, fetches their
// ids in one load and issues its row loads without branches; ptxas (62 registers, no spills) keeps two rows = 6 16-byte
// loads per lane in flight (3 KB per warp).  With 4 CTAs of 8 warps resident per SM that is 6144 loads (96 KB) in flight
// per SM, given >= 32 candidates per SM (e.g. 256 queries x 160 candidates = 1280 CTAs on 132 SMs).  A host link of
// ~64 GB/s with ~2 us of read latency needs ~128 KB in flight over the whole GPU, i.e. about 64 loads (1 KB) per SM: the
// design assumes >= 64 loads in flight per SM and provides ~100x that, so the host link, not latency, bounds it.
#include "mips_select.cuh"

namespace pq_refine {

constexpr int DIM = ATLAS_B200_EMBEDDINGS_DIM;
constexpr int QBLOCK = 256;                          // queries per select launch (workspace bound)
constexpr int WARPS = 8;
constexpr int ROWS_PER_WARP = 4;
constexpr int ROWS_PER_CTA = WARPS * ROWS_PER_WARP;
constexpr int CHUNKS = DIM / (8 * 32);               // 16-byte chunks per lane per row
static_assert(DIM % (8 * 32) == 0, "a row must split into whole 16-byte chunks per lane");

__device__ __forceinline__ float dot8(const uint4 a, const uint4 b, float acc) {
    const __half2* ha = reinterpret_cast<const __half2*>(&a);
    const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 x = __half22float2(ha[e]);
        const float2 y = __half22float2(hb[e]);
        acc = fmaf(x.x, y.x, acc);
        acc = fmaf(x.y, y.y, acc);
    }
    return acc;
}

// grid (ceil(k_cand / ROWS_PER_CTA), nq).  Candidate j of query q is row cand_local[q][j]; rows outside [0, n) are
// skipped.  Every refined candidate is appended to cand[q][0 .. count[q]) (count[q] zeroed by the caller); the order of
// the list does not matter to the select kernel, whose result depends only on the set of (score, row) keys.
__global__ void __launch_bounds__(WARPS * 32) pq_refine_kernel(const __half* __restrict__ rows, int64_t n,
                                                               const __half* __restrict__ queries,
                                                               const int64_t* __restrict__ cand_local, int k_cand,
                                                               uint32_t* __restrict__ count, uint64_t* __restrict__ cand) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q = blockIdx.y;
    const int j0 = blockIdx.x * ROWS_PER_CTA + warp * ROWS_PER_WARP;
    if (j0 >= k_cand) return;
    const int64_t* ids = cand_local + static_cast<int64_t>(q) * k_cand;

    // Straight-line code without branches, so that all 12 host loads are issued before the first product: the warp's
    // row ids arrive in one load (lane r holds id r) and are broadcast, then every row load is issued.  A skipped slot
    // loads the query row (device memory) instead of a host row.
    const __half* qrow = queries + static_cast<int64_t>(q) * DIM;
    int64_t my_id = -1;
    if (lane < ROWS_PER_WARP && j0 + lane < k_cand) my_id = ids[j0 + lane];
    if (my_id >= n) my_id = -1;
    int64_t row[ROWS_PER_WARP];
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) row[r] = __shfl_sync(0xffffffffu, my_id, r);
    uint4 x[ROWS_PER_WARP][CHUNKS];
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
        const uint4* src = reinterpret_cast<const uint4*>(row[r] >= 0 ? rows + row[r] * DIM : qrow);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) x[r][c] = __ldcs(src + lane + 32 * c);
    }
    const uint4* qv = reinterpret_cast<const uint4*>(qrow);
    uint4 qr[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) qr[c] = __ldg(qv + lane + 32 * c);

#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) acc = dot8(qr[c], x[r][c], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0 && row[r] >= 0) {
            const uint32_t pos = atomicAdd(&count[q], 1u);
            cand[static_cast<size_t>(q) * k_cand + pos] =
                mips::pack_candidate(mips::bits_to_key(mips::round_to_bits<false>(acc)), static_cast<uint32_t>(row[r]));
        }
    }
}

struct RefineWs {
    uint32_t* count;   // [QBLOCK]
    uint64_t* cand;    // [QBLOCK][k_cand]
};

static size_t refine_bytes(int nq, int k_cand, RefineWs* w, void* base) {
    const int qb = nq < QBLOCK ? (nq < 1 ? 1 : nq) : QBLOCK;
    const size_t count_bytes = abh::align_up(static_cast<size_t>(qb) * sizeof(uint32_t), 256);
    const size_t total = count_bytes + static_cast<size_t>(qb) * k_cand * sizeof(uint64_t);
    if (w) {
        uint8_t* b = static_cast<uint8_t*>(base);
        *w = RefineWs{reinterpret_cast<uint32_t*>(b), reinterpret_cast<uint64_t*>(b + count_bytes)};
    }
    return total;
}

static int refine_topk(const void* rows_host, int64_t n, const __half* queries, int nq, const int64_t* cand_local,
                       int k_cand, int k, __half* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride,
                       void* ws, size_t ws_bytes, cudaStream_t s) {
    AB_REQUIRE(nq >= 0, "nq=%d must be >= 0", nq);
    AB_REQUIRE(k >= 1 && k <= k_cand, "need 1 <= k <= k_cand (k=%d k_cand=%d)", k, k_cand);
    AB_REQUIRE(k_cand <= ATLAS_B200_MAX_TOPK, "k_cand=%d exceeds ATLAS_B200_MAX_TOPK=%d", k_cand, ATLAS_B200_MAX_TOPK);
    AB_REQUIRE(n >= 1 && n < (1ll << 31), "rows n=%lld out of range", (long long)n);
    if (nq == 0) return ATLAS_B200_OK;
    AB_REQUIRE(rows_host != nullptr && queries != nullptr && cand_local != nullptr && out_scores != nullptr &&
               out_ids != nullptr, "null pointer argument");
    AB_REQUIRE((reinterpret_cast<uintptr_t>(rows_host) & 15u) == 0 && (reinterpret_cast<uintptr_t>(queries) & 15u) == 0,
               "rows and queries must be 16-byte aligned");
    RefineWs w;
    const size_t need = refine_bytes(nq, k_cand, &w, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    void* rows_dev = nullptr;
    const cudaError_t e = cudaHostGetDevicePointer(&rows_dev, const_cast<void*>(rows_host), 0);
    if (e != cudaSuccess) {
        cudaGetLastError();   // not sticky: do not leave it for the next unrelated error check
        abh::set_error("cudaHostGetDevicePointer on the rows failed: %s (the rows must be pinned host memory mapped into "
                       "the device's address space)", cudaGetErrorString(e));
        return ATLAS_B200_ECUDA;
    }
    const __half* rows = static_cast<const __half*>(rows_dev);
    for (int q0 = 0; q0 < nq; q0 += QBLOCK) {
        const int nqb = nq - q0 < QBLOCK ? nq - q0 : QBLOCK;
        AB_CUDA_CHECK(cudaMemsetAsync(w.count, 0, static_cast<size_t>(nqb) * sizeof(uint32_t), s));
        const dim3 grid((k_cand + ROWS_PER_CTA - 1) / ROWS_PER_CTA, nqb);
        abh::prof_begin(s, abh::PROF_PQ_REFINE);
        pq_refine_kernel<<<grid, WARPS * 32, 0, s>>>(rows, n, queries + static_cast<int64_t>(q0) * DIM,
                                                     cand_local + static_cast<int64_t>(q0) * k_cand, k_cand, w.count, w.cand);
        abh::prof_end(s, abh::PROF_PQ_REFINE, static_cast<double>(nqb) * k_cand * DIM * sizeof(__half));
        AB_CUDA_CHECK(cudaGetLastError());
        mips::mips_select_kernel<false><<<nqb, mips::SEL_THREADS, 0, s>>>(
            w.cand, w.count, static_cast<uint32_t>(k_cand), k, mips::SEL_EMIT, nullptr,
            reinterpret_cast<uint16_t*>(out_scores + static_cast<size_t>(q0) * k), out_ids + static_cast<size_t>(q0) * k,
            id_base, id_stride, nullptr);
        abh::count_launch(2);
        AB_CUDA_CHECK(cudaGetLastError());
    }
    return ATLAS_B200_OK;
}

}  // namespace pq_refine

extern "C" {

size_t atlas_b200_pq_refine_workspace_bytes(int32_t nq, int32_t k_cand) {
    if (k_cand < 1) k_cand = 1;
    return pq_refine::refine_bytes(nq, k_cand, nullptr, nullptr);
}

int atlas_b200_pq_refine_topk(const void* rows_host, int64_t n, const void* queries, int32_t nq, const int64_t* cand_local,
                              int32_t k_cand, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                              int64_t id_stride, void* workspace, size_t workspace_bytes, void* stream) {
    return pq_refine::refine_topk(rows_host, n, static_cast<const __half*>(queries), nq, cand_local, k_cand, k,
                                  static_cast<__half*>(out_scores), out_ids, id_base, id_stride, workspace,
                                  workspace_bytes, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
