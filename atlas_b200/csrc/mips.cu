// Exact max-inner-product search with fused top-k candidate filtering for sm_90a.
//
// Replaces the reference's `torch.matmul(q.half(), E)` + `torch.topk` (src/index.py:113-120): the
// [nq, n] score matrix is never written.  Pipeline per block of <= 256 queries:
//
//   (1) sample scan   : the scan kernel over a strided sample of ~2*sqrt(k*n) bank rows, every
//                       score kept                                   -> candidate lists
//   (2) select (thr)  : per query, exact k-th best of the sample      -> a VALID lower bound on the
//                       final k-th best score (k real passages reach it)
//   (3) main scan     : ONE sweep of the whole bank (the HBM-bound part): wgmma GEMM tiles
//                       [<=256 queries] x [128 passages] x 768, fp32 accumulators in registers;
//                       the epilogue appends (score, id) of the few scores >= bound to the
//                       per-query candidate list
//   (4) select (final): per query, exact radix-select + sort of the candidates with the canonical
//                       order (fp16 score desc, id asc)               -> [nq, k] scores / ids
//
// Exactness: a passage whose fp16-rounded score is below a score that k other passages reach cannot be
// in the top-k, so filtering with `>= bound` never loses a winner; ties at the bound are kept and
// resolved by id in (4).  If a candidate list overflows (massive ties, adversarial order) `status`
// is raised and the caller falls back to `atlas_b200_mips_topk_exhaustive` (chunked, no thresholds).
//
// Scan kernel roles (384 threads, persistent, 1 CTA / SM):
//   warpgroup 0     TMA producer (one thread): bank tile + query tile K-blocks -> 4-stage smem ring (128B swizzle)
//   warpgroups 1-4  64 queries each (query half h = (wg - 1) / 2, rows 64 ((wg - 1) % 2) ..): one wgmma m64n128k16 per
//                   K step into 64 accumulator registers per thread, then the threshold filter + append straight from the
//                   registers
#include "common.cuh"
#include "host_common.h"
#include "mips_select.cuh"
#include "wgmma.cuh"

#include <math.h>
#include <stdlib.h>

namespace mips {

constexpr int DIM = ATLAS_B200_EMBEDDINGS_DIM;
constexpr int BLOCK_K = 64;  // 128 bytes of 16-bit elements = one swizzle row
constexpr int K_BLOCKS = DIM / BLOCK_K;
constexpr int UMMA_K = 16;   // K of one wgmma
constexpr int TILE_N = 128;   // passages per tile (wgmma N)
constexpr int HALF_M = 128;   // queries per consumer warpgroup
constexpr int QBLOCK = 256;   // queries per scan launch
constexpr int STAGES = 4;
constexpr int A_HALF_BYTES = HALF_M * BLOCK_K * 2;
constexpr int B_BYTES = TILE_N * BLOCK_K * 2;
constexpr int STAGE_BYTES = 2 * A_HALF_BYTES + B_BYTES;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
constexpr int NUM_THREADS = 640;

static_assert(DIM % BLOCK_K == 0, "");

// ---------------------------------------------------------------------------------------------
// scan kernel
// ---------------------------------------------------------------------------------------------
struct ScanParams {
    int n_rows;       // rows in this bank shard
    int tile_begin;   // tiles visited: tile_begin + i * tile_step, i in [0, num_tiles)
    int tile_step;
    int num_tiles;
    int nq;           // valid queries in this block (<= QBLOCK)
    int n_halves;     // 1 if nq <= 128 else 2
    const float* bound;   // [QBLOCK]
    uint32_t* count;      // [QBLOCK]
    uint64_t* cand;       // [QBLOCK][capq]
    uint32_t capq;
};

template <bool kBF16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
mips_scan_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_bank,
                 const ScanParams p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    // 1024-byte aligned tile ring (128B swizzle atoms are 1024 bytes)
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));

    if (threadIdx.x == 0) {
        ab::tma_prefetch_desc(&tmap_q);
        ab::tma_prefetch_desc(&tmap_bank);
        for (int s = 0; s < STAGES; ++s) {
            ab::mbar_init(&full_bar[s], 1);
            ab::mbar_init(&empty_bar[s], static_cast<uint32_t>(2 * p.n_halves));   // one arrive per active consumer warpgroup
        }
        ab::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        if (warp == 0 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            const uint32_t tx_bytes = static_cast<uint32_t>(p.n_halves) * A_HALF_BYTES + B_BYTES;
            for (int i = blockIdx.x; i < p.num_tiles; i += gridDim.x) {
                const int tile = p.tile_begin + i * p.tile_step;
                for (int kb = 0; kb < K_BLOCKS; ++kb) {
                    ab::mbar_wait_nocall(&empty_bar[stage], phase ^ 1u);
                    ab::mbar_arrive_expect_tx(&full_bar[stage], tx_bytes);
                    uint8_t* st = smem_gen + stage * STAGE_BYTES;
                    ab::tma_load_2d(&tmap_q, &full_bar[stage], st, kb * BLOCK_K, 0, ab::kEvictLast);
                    if (p.n_halves == 2)
                        ab::tma_load_2d(&tmap_q, &full_bar[stage], st + A_HALF_BYTES, kb * BLOCK_K, HALF_M,
                                        ab::kEvictLast);
                    ab::tma_load_2d(&tmap_bank, &full_bar[stage], st + 2 * A_HALF_BYTES, kb * BLOCK_K,
                                    tile * TILE_N, ab::kEvictFirst);
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ===================== query half h: MMAs + threshold filter + candidate append =====================
    const uint32_t cw = (warp >> 2) - 1u;             // consumer warpgroup 0..3
    const uint32_t half = cw >> 1, sub = cw & 1u;
    const uint32_t wl = warp & 3u;
    if (static_cast<int>(half) >= p.n_halves) return;
    // this thread's two query rows e: r and r + 8
    int qrow[2];
    float bnd[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        qrow[e] = static_cast<int>(half * HALF_M + sub * 64 + wl * 16 + (lane >> 2) + e * 8);
        bnd[e] = qrow[e] < p.nq ? p.bound[qrow[e]] : INFINITY;
    }
    const int cq = static_cast<int>(2u * (lane & 3u));
    uint32_t stage = 0, phase = 0;
    for (int i = blockIdx.x; i < p.num_tiles; i += gridDim.x) {
        const int tile = p.tile_begin + i * p.tile_step;
        float acc[64];
        int prev_stage = -1;
        for (int kb = 0; kb < K_BLOCKS; ++kb) {
            ab::mbar_wait_nocall(&full_bar[stage], phase);
            const uint32_t st = smem_base + stage * STAGE_BYTES;
            ab::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
                const uint64_t bdesc = ab::wgmma_desc_sw128(st + 2 * A_HALF_BYTES + k * UMMA_K * 2);
                const uint64_t adesc = ab::wgmma_desc_sw128(st + half * A_HALF_BYTES + sub * 8192 + k * UMMA_K * 2);
                ab::wgmma_m64n128k16_ss<kBF16, 0, 0>(acc, adesc, bdesc, (kb | k) != 0 ? 1 : 0);
            }
            ab::wgmma_commit();
            // the previous stage's MMAs have retired once at most this stage's group is pending: release it
            ab::wgmma_wait<1>();
            ab::wgmma_reg_fence(acc);
            if (prev_stage >= 0 && wl == 0 && lane == 0) ab::mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = static_cast<int>(stage);
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1u;
            }
        }
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(acc);
        if (wl == 0 && lane == 0) ab::mbar_arrive(&empty_bar[prev_stage]);

        // row e of this thread: acc[4 j + 2 e + c] = passage tile * 128 + 8 j + 2 (lane % 4) + c
        const int id_base = tile * TILE_N + cq;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float* a = acc + 2 * e;
            float m = -INFINITY;
#pragma unroll
            for (int j = 0; j < 32; ++j) m = fmaxf(m, fmaxf(a[4 * j], a[4 * j + 1]));
            if (!(m >= bnd[e])) continue;
            uint32_t npass = 0;
#pragma unroll
            for (int j = 0; j < 32; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) npass += (a[4 * j + c] >= bnd[e] && id_base + 8 * j + c < p.n_rows) ? 1u : 0u;
            if (npass == 0) continue;
            uint64_t* my_cand = p.cand + static_cast<size_t>(qrow[e]) * p.capq;
            uint32_t pos = atomicAdd(&p.count[qrow[e]], npass);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const float v = a[4 * j + c];
                    const int id = id_base + 8 * j + c;
                    if (v >= bnd[e] && id < p.n_rows) {
                        if (pos < p.capq)
                            my_cand[pos] = pack_candidate(bits_to_key(round_to_bits<kBF16>(v)), static_cast<uint32_t>(id));
                        ++pos;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// prep: stage one query block (zero padded to QBLOCK rows), reset counters and bounds
// ---------------------------------------------------------------------------------------------
__global__ void mips_prep_kernel(const uint16_t* __restrict__ queries, int nq, uint16_t* __restrict__ qstage,
                                 uint32_t* __restrict__ count, float* __restrict__ bound) {
    const int total = QBLOCK * DIM / 8;  // 16-byte vectors
    const uint4* src = reinterpret_cast<const uint4*>(queries);
    uint4* dst = reinterpret_cast<uint4*>(qstage);
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < total; v += gridDim.x * blockDim.x) {
        const int row = v / (DIM / 8);
        dst[v] = (row < nq) ? src[v] : make_uint4(0, 0, 0, 0);
    }
    if (blockIdx.x == 0 && threadIdx.x < QBLOCK) {
        count[threadIdx.x] = 0;
        bound[threadIdx.x] = -INFINITY;
    }
}

// ---------------------------------------------------------------------------------------------
// merge of W sorted per-shard lists: thread per candidate, rank by counting predecessors
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool before(uint32_t ka, int64_t ia, uint32_t kb, int64_t ib) {
    return (ka > kb) || (ka == kb && ia < ib);
}

__global__ void topk_merge_kernel(const uint16_t* __restrict__ scores_in, const int64_t* __restrict__ ids_in,
                                  int64_t stride_s, int64_t stride_i, int world, int k, int q_begin,
                                  uint16_t* __restrict__ out_scores, int64_t* __restrict__ out_ids) {
    const int qo = blockIdx.x;       // output row
    const int q = q_begin + qo;      // row inside every shard list
    for (int e = threadIdx.x; e < world * k; e += blockDim.x) {
        const int w = e / k, j = e % k;
        const size_t row = static_cast<size_t>(q) * k;
        const uint16_t hb = scores_in[w * stride_s + row + j];
        const uint32_t key = bits_to_key(hb);
        const int64_t id = ids_in[w * stride_i + row + j];
        int rank = j;  // predecessors inside its own (sorted) list
        for (int w2 = 0; w2 < world; ++w2) {
            if (w2 == w) continue;
            const uint16_t* s2 = scores_in + w2 * stride_s + row;
            const int64_t* i2 = ids_in + w2 * stride_i + row;
            int lo = 0, hi = k;  // number of elements of list w2 that come before (key, id)
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (before(bits_to_key(s2[mid]), i2[mid], key, id))
                    lo = mid + 1;
                else
                    hi = mid;
            }
            rank += lo;
        }
        if (rank < k) {
            out_scores[static_cast<size_t>(qo) * k + rank] = hb;
            out_ids[static_cast<size_t>(qo) * k + rank] = id;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// casts
// ---------------------------------------------------------------------------------------------
template <bool kBF16>
__global__ void cast_f32_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, int64_t count) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < count;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x)
        dst[i] = static_cast<uint16_t>(round_to_bits<kBF16>(src[i]));
}

template <bool kBF16>
__global__ void widen_kernel(const uint16_t* __restrict__ src, float* __restrict__ dst, int64_t count) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < count;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x)
        dst[i] = bits_to_float<kBF16>(src[i]);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
struct Workspace {
    uint32_t* count;
    float* bound;
    int32_t* status;
    uint16_t* qstage;
    uint64_t* cand;
    uint32_t capq;
    // host-buffer path staging
    float* q_f32;
    uint16_t* q_16;
    uint16_t* o_s16;
    float* o_s32;
    int64_t* o_ids;
};


static size_t carve(Workspace* w, void* base, int64_t n, int nq, int k) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        size_t o = off;
        off = abh::align_up(off + bytes, 256);
        return o;
    };
    const uint32_t capq = capq_for(n, k);
    const size_t o_count = take(QBLOCK * sizeof(uint32_t));
    const size_t o_bound = take(QBLOCK * sizeof(float));
    const size_t o_status = take(sizeof(int32_t));
    const size_t o_qstage = take(static_cast<size_t>(QBLOCK) * DIM * 2);
    const size_t o_cand = take(static_cast<size_t>(QBLOCK) * capq * sizeof(uint64_t));
    const size_t o_qf32 = take(static_cast<size_t>(nq) * DIM * sizeof(float));
    const size_t o_q16 = take(static_cast<size_t>(nq) * DIM * 2);
    const size_t o_os16 = take(static_cast<size_t>(nq) * k * 2);
    const size_t o_os32 = take(static_cast<size_t>(nq) * k * sizeof(float));
    const size_t o_oids = take(static_cast<size_t>(nq) * k * sizeof(int64_t));
    if (w) {
        uint8_t* b = static_cast<uint8_t*>(base);
        w->count = reinterpret_cast<uint32_t*>(b + o_count);
        w->bound = reinterpret_cast<float*>(b + o_bound);
        w->status = reinterpret_cast<int32_t*>(b + o_status);
        w->qstage = reinterpret_cast<uint16_t*>(b + o_qstage);
        w->cand = reinterpret_cast<uint64_t*>(b + o_cand);
        w->capq = capq;
        w->q_f32 = reinterpret_cast<float*>(b + o_qf32);
        w->q_16 = reinterpret_cast<uint16_t*>(b + o_q16);
        w->o_s16 = reinterpret_cast<uint16_t*>(b + o_os16);
        w->o_s32 = reinterpret_cast<float*>(b + o_os32);
        w->o_ids = reinterpret_cast<int64_t*>(b + o_oids);
    }
    return off;
}

template <bool kBF16>
static int launch_scan(const CUtensorMap& tq, const CUtensorMap& tb, const ScanParams& p, cudaStream_t s) {
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(mips_scan_kernel<kBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SMEM_BYTES));
        attr_set = true;
    }
    if (p.num_tiles <= 0) return ATLAS_B200_OK;
    const int grid = p.num_tiles < abh::num_sms() ? p.num_tiles : abh::num_sms();
    mips_scan_kernel<kBF16><<<grid, NUM_THREADS, SMEM_BYTES, s>>>(tq, tb, p);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

static int check_common(const void* bank, int64_t n, int64_t ld, const void* queries, int nq, int k) {
    AB_REQUIRE(nq >= 0 && k >= 1, "nq must be >= 0 and k >= 1 (nq=%d k=%d)", nq, k);
    AB_REQUIRE(k <= ATLAS_B200_MAX_TOPK, "k=%d exceeds ATLAS_B200_MAX_TOPK=%d", k, ATLAS_B200_MAX_TOPK);
    AB_REQUIRE(n >= 1 && n < (1ll << 31) - TILE_N, "bank rows n=%lld out of range", (long long)n);
    // torch.topk raises when k > n (src/index.py:118)
    AB_REQUIRE(k <= n, "selected index k out of range: k=%d > n=%lld", k, (long long)n);
    AB_REQUIRE(ld >= DIM && ld % 8 == 0, "row stride ld=%lld must be >= 768 and a multiple of 8", (long long)ld);
    AB_REQUIRE(bank != nullptr && (reinterpret_cast<uintptr_t>(bank) & 15u) == 0, "bank must be 16-byte aligned");
    AB_REQUIRE(nq == 0 || (queries != nullptr && (reinterpret_cast<uintptr_t>(queries) & 15u) == 0),
               "queries must be 16-byte aligned");
    return ATLAS_B200_OK;
}

template <bool kBF16>
static int topk_impl(const void* bank, int64_t n, int64_t ld, const void* queries, int nq, int k, void* out_scores,
                     int64_t* out_ids, int64_t id_base, int64_t id_stride, int32_t* status, void* workspace,
                     size_t workspace_bytes, cudaStream_t s, bool exhaustive) {
    int rc = check_common(bank, n, ld, queries, nq, k);
    if (rc) return rc;
    if (status) AB_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int32_t), s));
    if (nq == 0) return ATLAS_B200_OK;
    Workspace w;
    const size_t need = carve(&w, workspace, n, nq, k);
    if (workspace == nullptr || workspace_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", workspace_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    const int tile_n = TILE_N;
    // tensor maps: query block (128-row boxes) + 128-row bank boxes
    CUtensorMap tq, tb;
    rc = abh::make_tmap_2d_16bit(&tq, w.qstage, QBLOCK, DIM, DIM, HALF_M, BLOCK_K, kBF16);
    if (rc) return rc;
    rc = abh::make_tmap_2d_16bit(&tb, bank, static_cast<uint64_t>(n), DIM, static_cast<uint64_t>(ld), TILE_N, BLOCK_K, kBF16);
    if (rc) return rc;

    const int total_tiles = static_cast<int>((n + tile_n - 1) / tile_n);
    const uint16_t* q16 = static_cast<const uint16_t*>(queries);
    uint16_t* os = static_cast<uint16_t*>(out_scores);

    for (int q0 = 0; q0 < nq; q0 += QBLOCK) {
        const int nqb = (nq - q0 < QBLOCK) ? (nq - q0) : QBLOCK;
        mips_prep_kernel<<<64, 256, 0, s>>>(q16 + static_cast<size_t>(q0) * DIM, nqb, w.qstage, w.count, w.bound);
        abh::count_launch();
        ScanParams p;
        p.n_rows = static_cast<int>(n);
        p.nq = nqb;
        p.n_halves = nqb > HALF_M ? 2 : 1;
        p.bound = w.bound;
        p.count = w.count;
        p.cand = w.cand;
        p.capq = w.capq;
        uint16_t* os_b = os + static_cast<size_t>(q0) * k;
        int64_t* oi_b = out_ids + static_cast<size_t>(q0) * k;
        auto scan = [&](const ScanParams& sp) -> int { return launch_scan<kBF16>(tq, tb, sp, s); };

        if (!exhaustive) {
            int first_tile = 0;
            if (n > static_cast<int64_t>(w.capq)) {
                // (1)+(2): first bound from a strided sample of ~2*sqrt(k*n) rows (every score kept)
                // Sample size: the bound-only select costs O(m) per query and the sweep that follows keeps ~k*n_next/m
                // candidates per query.  With the refinement sweep over the first tenth of the bank (below) the next part
                // is n/10 rows, so m = sqrt(k*n/10) balances the two selects (4 Mi rows, k = 40: m = 4096 instead of the
                // 26 k of the one-stage bound 2*sqrt(k*n): the 256-query threshold select does ~6 x less work);
                // without a refinement stage the one-stage optimum is kept.
                double m_two_stage = sqrt(static_cast<double>(k) * static_cast<double>(n) / 10.0);
                if (m_two_stage < 4096) m_two_stage = 4096;
                const bool refine = (total_tiles / 10) * static_cast<double>(tile_n) >= 8.0 * m_two_stage;
                double m = refine ? m_two_stage : 2.0 * sqrt(static_cast<double>(k) * static_cast<double>(n));
                if (m < 4096) m = 4096;
                if (m > w.capq / 2) m = w.capq / 2;
                int sample_tiles = static_cast<int>(m / tile_n);
                if (sample_tiles < 1) sample_tiles = 1;
                if (sample_tiles > total_tiles) sample_tiles = total_tiles;
                p.tile_begin = 0;
                p.tile_step = total_tiles / sample_tiles;
                p.num_tiles = sample_tiles;
                rc = scan(p);
                if (rc) return rc;
                mips_select_kernel<kBF16><<<nqb, SEL_THREADS, 0, s>>>(w.cand, w.count, w.capq, k, SEL_WRITE_BOUND,
                                                                     w.bound, nullptr, nullptr, 0, 0, nullptr);
                abh::count_launch();
                // (2b) refinement: sweep the first ~1/10 of the bank with that bound, then tighten the bound to
                // the k-th best seen so far (its winners stay in the lists) before sweeping the other 9/10.
                // Expected survivors per query: k*n_A/m in this part, k*n_B/n_A (~9k) in the rest.
                const int tiles_a = total_tiles / 10;
                if (tiles_a * static_cast<int64_t>(tile_n) >= 8 * static_cast<int64_t>(m)) {
                    p.tile_begin = 0;
                    p.tile_step = 1;
                    p.num_tiles = tiles_a;
                    abh::prof_begin(s, abh::PROF_SCAN);
                    rc = scan(p);
                    abh::prof_end(s, abh::PROF_SCAN, static_cast<double>(tiles_a) * tile_n * DIM * 2.0);
                    if (rc) return rc;
                    mips_select_kernel<kBF16><<<nqb, SEL_THREADS, 0, s>>>(w.cand, w.count, w.capq, k,
                                                                         SEL_WRITE_BOUND | SEL_CARRY, w.bound, nullptr,
                                                                         nullptr, 0, 0, status);
                    abh::count_launch();
                    first_tile = tiles_a;
                }
            }
            // (3)+(4): the main sweep and the final selection
            p.tile_begin = first_tile;
            p.tile_step = 1;
            p.num_tiles = total_tiles - first_tile;
            abh::prof_begin(s, abh::PROF_SCAN);
            rc = scan(p);
            abh::prof_end(s, abh::PROF_SCAN, static_cast<double>(total_tiles - first_tile) * tile_n * DIM * 2.0);
            if (rc) return rc;
            mips_select_kernel<kBF16><<<nqb, SEL_THREADS, 0, s>>>(w.cand, w.count, w.capq, k, SEL_EMIT, w.bound, os_b,
                                                                 oi_b, id_base, id_stride, status);
            abh::count_launch();
        } else {
            // chunked exact scan: every score of a chunk is a candidate, winners are carried forward
            int chunk_tiles = static_cast<int>((w.capq - static_cast<uint32_t>(k)) / tile_n);
            if (chunk_tiles < 1) chunk_tiles = 1;
            for (int t0 = 0; t0 < total_tiles; t0 += chunk_tiles) {
                const bool last = t0 + chunk_tiles >= total_tiles;
                p.tile_begin = t0;
                p.tile_step = 1;
                p.num_tiles = last ? total_tiles - t0 : chunk_tiles;
                rc = scan(p);
                if (rc) return rc;
                mips_select_kernel<kBF16><<<nqb, SEL_THREADS, 0, s>>>(w.cand, w.count, w.capq, k,
                                                                     last ? SEL_EMIT : SEL_CARRY, w.bound, os_b, oi_b,
                                                                     id_base, id_stride, nullptr);
                abh::count_launch();
            }
        }
    }
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // namespace mips

extern "C" {

size_t atlas_b200_mips_workspace_bytes(int64_t n, int32_t nq, int32_t k) {
    if (n < 1) n = 1;
    if (nq < 0) nq = 0;
    if (k < 1) k = 1;
    return mips::carve(nullptr, nullptr, n, nq, k);
}

int atlas_b200_mips_topk(const void* bank, int64_t n, int64_t ld, int32_t is_bf16, const void* queries, int32_t nq,
                         int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride,
                         int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16)
        return mips::topk_impl<true>(bank, n, ld, queries, nq, k, out_scores, out_ids, id_base, id_stride, status,
                                     workspace, workspace_bytes, s, false);
    return mips::topk_impl<false>(bank, n, ld, queries, nq, k, out_scores, out_ids, id_base, id_stride, status,
                                  workspace, workspace_bytes, s, false);
}

int atlas_b200_mips_topk_exhaustive(const void* bank, int64_t n, int64_t ld, int32_t is_bf16, const void* queries,
                                    int32_t nq, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                                    int64_t id_stride, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16)
        return mips::topk_impl<true>(bank, n, ld, queries, nq, k, out_scores, out_ids, id_base, id_stride, nullptr,
                                     workspace, workspace_bytes, s, true);
    return mips::topk_impl<false>(bank, n, ld, queries, nq, k, out_scores, out_ids, id_base, id_stride, nullptr,
                                  workspace, workspace_bytes, s, true);
}

int atlas_b200_topk_merge(const void* scores_in, const int64_t* ids_in, int64_t shard_stride_scores,
                          int64_t shard_stride_ids, int32_t is_bf16, int32_t world, int32_t nq_total, int32_t k,
                          int32_t q_begin, int32_t nq_out, void* out_scores, int64_t* out_ids, void* stream) {
    (void)is_bf16;  // the sortable-key transform is identical for both 16-bit formats
    AB_REQUIRE(world >= 1 && k >= 1 && nq_total >= 0 && nq_out >= 0 && q_begin >= 0 && q_begin + nq_out <= nq_total,
               "bad merge arguments (world=%d nq_total=%d k=%d q_begin=%d nq_out=%d)", world, nq_total, k, q_begin,
               nq_out);
    if (nq_out == 0) return ATLAS_B200_OK;
    mips::topk_merge_kernel<<<nq_out, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint16_t*>(scores_in), ids_in, shard_stride_scores, shard_stride_ids, world, k, q_begin,
        static_cast<uint16_t*>(out_scores), out_ids);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_cast_f32(const float* src, void* dst, int64_t count, int32_t to_bf16, void* stream) {
    if (count <= 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int64_t blocks = (count + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    if (to_bf16)
        mips::cast_f32_kernel<true><<<static_cast<int>(blocks), 256, 0, s>>>(src, static_cast<uint16_t*>(dst), count);
    else
        mips::cast_f32_kernel<false><<<static_cast<int>(blocks), 256, 0, s>>>(src, static_cast<uint16_t*>(dst), count);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_search_host(const void* bank, int64_t n, int64_t ld, int32_t is_bf16, const float* queries_host,
                           int32_t nq, int32_t k, float* out_scores_host, int64_t* out_ids_host, int64_t id_base,
                           int64_t id_stride, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = mips::check_common(bank, n, ld, reinterpret_cast<const void*>(16), nq, k);
    if (rc) return rc;
    if (nq == 0) return ATLAS_B200_OK;
    mips::Workspace w;
    const size_t need = mips::carve(&w, workspace, n, nq, k);
    if (workspace == nullptr || workspace_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", workspace_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    const int64_t qcount = static_cast<int64_t>(nq) * mips::DIM;
    AB_CUDA_CHECK(cudaMemcpyAsync(w.q_f32, queries_host, qcount * sizeof(float), cudaMemcpyHostToDevice, s));
    rc = atlas_b200_cast_f32(w.q_f32, w.q_16, qcount, is_bf16, stream);
    if (rc) return rc;
    rc = atlas_b200_mips_topk(bank, n, ld, is_bf16, w.q_16, nq, k, w.o_s16, w.o_ids, id_base, id_stride, w.status,
                              workspace, workspace_bytes, stream);
    if (rc) return rc;
    int32_t st = 0;
    AB_CUDA_CHECK(cudaMemcpyAsync(&st, w.status, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    const int64_t ocount = static_cast<int64_t>(nq) * k;
    int blocks = static_cast<int>((ocount + 255) / 256);
    if (blocks > 1024) blocks = 1024;
    if (is_bf16)
        mips::widen_kernel<true><<<blocks, 256, 0, s>>>(w.o_s16, w.o_s32, ocount);
    else
        mips::widen_kernel<false><<<blocks, 256, 0, s>>>(w.o_s16, w.o_s32, ocount);
    abh::count_launch();
    AB_CUDA_CHECK(cudaMemcpyAsync(out_scores_host, w.o_s32, ocount * sizeof(float), cudaMemcpyDeviceToHost, s));
    AB_CUDA_CHECK(cudaMemcpyAsync(out_ids_host, w.o_ids, ocount * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    AB_CUDA_CHECK(cudaStreamSynchronize(s));
    if (st != 0) {
        rc = atlas_b200_mips_topk_exhaustive(bank, n, ld, is_bf16, w.q_16, nq, k, w.o_s16, w.o_ids, id_base, id_stride,
                                             workspace, workspace_bytes, stream);
        if (rc) return rc;
        if (is_bf16)
            mips::widen_kernel<true><<<blocks, 256, 0, s>>>(w.o_s16, w.o_s32, ocount);
        else
            mips::widen_kernel<false><<<blocks, 256, 0, s>>>(w.o_s16, w.o_s32, ocount);
        abh::count_launch();
        AB_CUDA_CHECK(cudaMemcpyAsync(out_scores_host, w.o_s32, ocount * sizeof(float), cudaMemcpyDeviceToHost, s));
        AB_CUDA_CHECK(cudaMemcpyAsync(out_ids_host, w.o_ids, ocount * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        AB_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return ATLAS_B200_OK;
}

}  // extern "C"
