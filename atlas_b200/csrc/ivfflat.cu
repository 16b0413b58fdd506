// IVF-Flat row scan for sm_90a: the hot path of `DistributedFAISSIndex("ivfflat")` and ("flat") (layout: ivfflat.cuh,
// host code and rules: pq.cu, include/atlas_b200.h).
//
// A row's score is the flat index's: fp16(<q_fp16, x_fp16>), accumulated in fp32 on the tensor cores with the same
// operands, shape and K order as mips.cu's scan (A = queries, B = rows, wgmma m64n128k16), so a full scan returns the
// flat index's scores bit for bit.  No coarse term is added; the coarse terms only choose the probe sets.
//
// Roles (640 threads, persistent, 1 CTA / SM):
//   warpgroup 0     TMA producer (one thread): per CTA step of two 64-slot tiles (128 slots), for each of the 12 K-blocks,
//                   the two tiles' 64 x 128-byte row blocks and the block's query K-block (64 rows per active consumer,
//                   read from L2) through a 4-stage mbarrier ring (128B swizzle).
//   warpgroups 1-4  64 queries each (only ceil(nq / 64) of them take part): one wgmma m64n128k16 per k16 step into 64
//                   accumulator registers per thread, then the threshold filter and the append straight from the
//                   registers.  A slot's local row is read only when its score passes the bound; padding slots (row -1)
//                   are never appended.
// PROBED: the tiles come from the compacted items (ivf_probe.cuh).  One CTA serves every query of the block, and an item
// exists only for a list some query of the block probes, so no step is skipped; a slot is appended for query q only when
// q probes its tile's list.  The producer and the consumers derive the same item sequence from the same count (read once,
// before the loop), so the ring stays in step.
#include "common.cuh"
#include "host_common.h"
#include "ivf_probe.cuh"
#include "ivfflat.cuh"
#include "mips_select.cuh"
#include "wgmma.cuh"

namespace ivfflat {

constexpr int BLOCK_K = 64;                          // 128 bytes of fp16 = one swizzle row
constexpr int K_BLOCKS = FLAT_DIM / BLOCK_K;
constexpr int STEP_TILES = 2;                        // wgmma N = 128 slots
constexpr int WG_M = 64;                             // queries per consumer warpgroup
constexpr int CONSUMERS = FLAT_QBLOCK / WG_M;
constexpr int STAGES = 4;
constexpr int TILE_BYTES = FLAT_TILE * BLOCK_K * 2;  // one tile's rows of one K-block
constexpr int B_BYTES = STEP_TILES * TILE_BYTES;
constexpr int A_BYTES = WG_M * BLOCK_K * 2;          // one consumer's queries of one K-block
constexpr int STAGE_BYTES = B_BYTES + CONSUMERS * A_BYTES;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
constexpr int NUM_THREADS = 128 * (1 + CONSUMERS);
// 640 threads start with LAUNCH_REGS registers each (__launch_bounds__(640, 1)).  setmaxnreg.inc takes registers only from
// those released in the same CTA, so the producer gives up at least what the consumers add; with the extra registers the
// consumers' 64 accumulators and the epilogue fit without spilling.
constexpr int LAUNCH_REGS = 96;
constexpr int PRODUCER_REGS = 24;
constexpr int CONSUMER_REGS = 112;
static_assert(128 * (LAUNCH_REGS - PRODUCER_REGS) >= 128 * CONSUMERS * (CONSUMER_REGS - LAUNCH_REGS), "");

static_assert(FLAT_DIM % BLOCK_K == 0, "");

template <bool PROBED>
__global__ void __launch_bounds__(NUM_THREADS, 1)
ivfflat_scan_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_r,
                    const ScanParams p, const ivfsq::ProbeScan pr) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));
    const int n_cw = (p.nq + WG_M - 1) / WG_M;

    int pbegin = 0, pstep = 1, pnum = 0;
    if constexpr (PROBED) ivfp::resolve_items(*pr.item_count, p.tile_begin, p.tile_step, p.num_tiles, pbegin, pstep, pnum);
    const int n_items = PROBED ? pnum : p.num_tiles;
    const int steps = (n_items + STEP_TILES - 1) / STEP_TILES;
    // item i of this launch: its tile and (PROBED) its list; false past the last item
    auto item = [&](int i, int& tile, int& list) -> bool {
        if (i >= n_items) return false;
        if constexpr (PROBED) {
            const int2 it = pr.items[pbegin + i * pstep];
            list = it.x;
            tile = it.y;
        } else {
            list = 0;
            tile = p.tile_begin + i * p.tile_step;
        }
        return true;
    };

    if (threadIdx.x == 0) {
        ab::tma_prefetch_desc(&tmap_q);
        ab::tma_prefetch_desc(&tmap_r);
        for (int s = 0; s < STAGES; ++s) {
            ab::mbar_init(&full_bar[s], 1);
            ab::mbar_init(&empty_bar[s], static_cast<uint32_t>(n_cw));   // one arrive per active consumer warpgroup
        }
        ab::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        ab::setmaxnreg_dec<PRODUCER_REGS>();
        if (warp == 0 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            for (int g = blockIdx.x; g < steps; g += gridDim.x) {
                int tile[STEP_TILES] = {0, 0}, list[STEP_TILES] = {0, 0}, ntile = 0;
                bool has[STEP_TILES];
                for (int c = 0; c < STEP_TILES; ++c) ntile += (has[c] = item(g * STEP_TILES + c, tile[c], list[c])) ? 1 : 0;
                const uint32_t tx = static_cast<uint32_t>(ntile * TILE_BYTES + n_cw * A_BYTES);
                for (int kb = 0; kb < K_BLOCKS; ++kb) {
                    ab::mbar_wait_nocall(&empty_bar[stage], phase ^ 1u);
                    ab::mbar_arrive_expect_tx(&full_bar[stage], tx);
                    uint8_t* st = smem_gen + stage * STAGE_BYTES;
                    for (int c = 0; c < STEP_TILES; ++c)
                        if (has[c])
                            ab::tma_load_2d(&tmap_r, &full_bar[stage], st + c * TILE_BYTES, kb * BLOCK_K, tile[c] * FLAT_TILE,
                                            ab::kEvictFirst);
                    for (int w = 0; w < n_cw; ++w)
                        ab::tma_load_2d(&tmap_q, &full_bar[stage], st + B_BYTES + w * A_BYTES, kb * BLOCK_K, w * WG_M,
                                        ab::kEvictLast);
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: 64 queries x 128 slots per step =====================
    ab::setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = static_cast<int>(warp >> 2) - 1;
    if (cw >= n_cw) return;
    const int wl = static_cast<int>(warp & 3u);
    // this thread's two query rows e: r and r + 8
    int qrow[2];
    float bnd[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        qrow[e] = cw * WG_M + wl * 16 + static_cast<int>(lane >> 2) + e * 8;
        bnd[e] = qrow[e] < p.nq ? p.bound[qrow[e]] : INFINITY;
    }
    const int cq = static_cast<int>(2u * (lane & 3u));
    uint32_t stage = 0, phase = 0;
    for (int g = blockIdx.x; g < steps; g += gridDim.x) {
        float acc[64];
        int prev_stage = -1;
        for (int kb = 0; kb < K_BLOCKS; ++kb) {
            ab::mbar_wait_nocall(&full_bar[stage], phase);
            const uint32_t st = smem_base + stage * STAGE_BYTES;
            ab::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / 16; ++k) {
                const uint64_t bdesc = ab::wgmma_desc_sw128(st + k * 32);
                const uint64_t adesc = ab::wgmma_desc_sw128(st + B_BYTES + cw * A_BYTES + k * 32);
                ab::wgmma_m64n128k16_ss<false, 0, 0>(acc, adesc, bdesc, (kb | k) != 0 ? 1 : 0);
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

        // the step's tiles, read after the MMAs so that they hold no registers across them
        int tile[STEP_TILES] = {0, 0}, list[STEP_TILES] = {0, 0};
        bool has[STEP_TILES];
#pragma unroll
        for (int c = 0; c < STEP_TILES; ++c) has[c] = item(g * STEP_TILES + c, tile[c], list[c]);
        // row e of this thread: acc[4 j + 2 e + c] = slot 8 j + 2 (lane % 4) + c of the step, i.e. slot
        // 8 (j % 8) + 2 (lane % 4) + c of tile j / 8
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            if (qrow[e] >= p.nq) continue;
            bool live[STEP_TILES];
            int sbase[STEP_TILES];     // slot of j % 8 = 0, c = 0 (n_tiles * FLAT_TILE < 2^31)
#pragma unroll
            for (int h = 0; h < STEP_TILES; ++h) {
                live[h] = has[h] && (!PROBED || ivfp::probes(pr.probed, list[h], qrow[e]));
                sbase[h] = tile[h] * FLAT_TILE + cq;
            }
            uint32_t npass = 0;
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c)
                    if (live[j / 8] && acc[4 * j + 2 * e + c] >= bnd[e] && __ldg(p.slot_rows + sbase[j / 8] + 8 * (j % 8) + c) >= 0)
                        ++npass;
            if (npass == 0) continue;
            uint64_t* my_cand = p.cand + static_cast<size_t>(qrow[e]) * p.capq;
            uint32_t pos = atomicAdd(&p.count[qrow[e]], npass);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const float v = acc[4 * j + 2 * e + c];
                    if (!live[j / 8] || !(v >= bnd[e])) continue;
                    const int32_t row = __ldg(p.slot_rows + sbase[j / 8] + 8 * (j % 8) + c);
                    if (row < 0) continue;
                    if (pos < p.capq)
                        my_cand[pos] = mips::pack_candidate(mips::bits_to_key(mips::round_to_bits<false>(v)),
                                                            static_cast<uint32_t>(row));
                    ++pos;
                }
            }
        }
    }
}

template <bool PROBED>
static int launch(const CUtensorMap& tq, const CUtensorMap& tr, const ScanParams& p, const ivfsq::ProbeScan& pr,
                  cudaStream_t s) {
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(ivfflat_scan_kernel<PROBED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SMEM_BYTES));
        attr_set = true;
    }
    const int steps = (p.num_tiles + STEP_TILES - 1) / STEP_TILES;
    const int grid = steps < abh::num_sms() ? steps : abh::num_sms();
    ivfflat_scan_kernel<PROBED><<<grid, NUM_THREADS, SMEM_BYTES, s>>>(tq, tr, p, pr);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int launch_scan(const ScanParams& p, const ivfsq::ProbeScan* probe, cudaStream_t s) {
    if (p.num_tiles <= 0 || p.nq <= 0) return ATLAS_B200_OK;
    CUtensorMap tq, tr;
    int rc = abh::make_tmap_2d_16bit(&tq, p.qstage, FLAT_QBLOCK, FLAT_DIM, FLAT_DIM, WG_M, BLOCK_K, false);
    if (rc) return rc;
    rc = abh::make_tmap_2d_16bit(&tr, p.rows, static_cast<uint64_t>(p.n_tiles) * FLAT_TILE, FLAT_DIM, FLAT_DIM, FLAT_TILE,
                                 BLOCK_K, false);
    if (rc) return rc;
    return probe ? launch<true>(tq, tr, p, *probe, s) : launch<false>(tq, tr, p, ivfsq::ProbeScan{}, s);
}

}  // namespace ivfflat
