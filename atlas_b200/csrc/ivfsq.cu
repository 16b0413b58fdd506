// IVF-SQ code scan for sm_90a: the hot path of `DistributedFAISSIndex("ivfsq")` (layout and rules: ivfsq.cuh, pq.cu).
//
// A 4-bit SQ score is a dense dot product: s(q, x) = T[q][list] + C[q] + 2^-e_q * sum_d w^[q][d] * (code_d - 8), with the
// codes small integers and the per-dimension scale folded into the fp16 query operand w^.  So the scan is a GEMM whose
// A operand (64 slots x 16 dims per step) is decoded from nibbles straight into registers - wgmma's register-A form -
// and whose B operand is the query block, N = NQ queries.
//
// Roles (384 threads, persistent, 1 CTA / SM):
//   warp 0          TMA producer (one thread): the CTA's query block [NQ x 768] once into shared memory, where it stays
//                   for the whole sweep (128B swizzle, K-major, 12 K-blocks); then, per CTA step of two tiles (128
//                   slots), the 64 x 32-byte code K-blocks of both tiles through an mbarrier ring as deep as the rest
//                   of shared memory allows.
//   warpgroups 1-2  one 64-slot tile each per step: per K-block the quad lane loads 8 code bytes of each of its two
//                   fragment rows, converts the nibbles to fp16 pairs code - 8 (lop3 with the 0x6400 magic, then subtract 1032)
//                   and issues four wgmma m64nNQk16 with A from registers; then the epilogue
//                   acc * 2^-e_q + C[q] + T[list][q], the threshold filter and the append in mips_select.cuh's format.
// Keeping the query block resident means it is read from L2 once per CTA instead of once per tile.  A block of more
// than 128 queries is split over grid.y (NQ <= 128 keeps the block and the ring in 227 KB of shared memory), so the
// codes are then read once per 128 queries.
#include "common.cuh"
#include "host_common.h"
#include "ivf_probe.cuh"
#include "ivfsq.cuh"
#include "mips_select.cuh"
#include "wgmma.cuh"

namespace ivfsq {

constexpr int K_BLOCKS = SQ_DIM / 64;
constexpr int CONSUMERS = 2;
constexpr int TILE_KB_BYTES = SQ_TILE * SQ_KBLOCK_BYTES;      // 2048: one tile's codes of one K-block
constexpr int STAGE_BYTES = CONSUMERS * TILE_KB_BYTES;
constexpr int NUM_THREADS = 128 * (1 + CONSUMERS);

constexpr int SMEM_LIMIT = 227 * 1024 - 4096;      // dynamic shared memory, leaving room for the static part

// ring depth: whatever shared memory the resident query block leaves (7 stages at 128 queries), at most 32 stages
// (128 KB of codes in flight per SM for small query blocks, where the sweep is bound by HBM latency and bandwidth)
template <int NQ>
__host__ __device__ constexpr int stages() {
    return (SMEM_LIMIT - NQ * 128 * K_BLOCKS - 1024) / STAGE_BYTES < 32 ? (SMEM_LIMIT - NQ * 128 * K_BLOCKS - 1024) / STAGE_BYTES
                                                                          : 32;
}
template <int NQ>
__host__ __device__ constexpr int smem_bytes() { return NQ * 128 * K_BLOCKS + stages<NQ>() * STAGE_BYTES + 1024; }

// fp16 pair code - 8 of the nibbles at bits 0 and 16 of w / at bits 4 and 20 of w.  Centred codes keep the running
// fp32 sum of the MMA small: the tensor cores' accumulation does not round to nearest, and with codes 0..15 its error
// grows with the sum's common offset.  The offset 8 sum_d w^ is part of C[q].
__device__ __forceinline__ uint32_t nib_lo(uint32_t w) {
    const uint32_t h = (w & 0x000F000Fu) | 0x64006400u;     // 1024 + n
    uint32_t r;
    asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(h), "r"(0x64086408u));      // - 1032
    return r;
}
__device__ __forceinline__ uint32_t nib_hi(uint32_t w) {
    const uint32_t h = (w & 0x00F000F0u) | 0x64006400u;     // 1024 + 16 n
    uint32_t r;
    asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(r) : "r"(h), "r"(0x2C002C00u), "r"(0xD480D480u));   // / 16 - 72
    return r;
}

template <int NQ>
__device__ __forceinline__ void mma_step(float (&acc)[NQ / 2], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
    if constexpr (NQ == 8) ab::wgmma_m64n8k16_rs_f16<0>(acc, a, bdesc, scale_d);
    else if constexpr (NQ == 16) ab::wgmma_m64n16k16_rs_f16<0>(acc, a, bdesc, scale_d);
    else if constexpr (NQ == 32) ab::wgmma_m64n32k16_rs_f16<0>(acc, a, bdesc, scale_d);
    else if constexpr (NQ == 64) ab::wgmma_m64n64k16_rs<false, 0>(acc, a, bdesc, scale_d);
    else ab::wgmma_m64n128k16_rs_f16<0>(acc, a, bdesc, scale_d);
}

// PROBED: the tiles come from the compacted items (ivf_probe.cuh); a step whose two items no query of this CTA's group
// probes is skipped.  The producer and both consumers derive the same item sequence from the same count (read once,
// before the loop) and the same probe bits, so the mbarrier ring stays in step.
template <int NQ, bool PROBED>
__global__ void __launch_bounds__(NUM_THREADS, 1)
ivfsq_scan_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_c, const ScanParams p,
                  const ProbeScan pr) {
    constexpr int STAGES = stages<NQ>();
    static_assert(STAGES >= 4, "");
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];
    __shared__ __align__(8) uint64_t q_bar;
    __shared__ float s_scale[NQ], s_c[NQ], s_bnd[NQ];

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));
    constexpr int Q_KB_BYTES = NQ * 128;
    const uint8_t* ring_gen = smem_gen + K_BLOCKS * Q_KB_BYTES;

    const int q0 = blockIdx.y * NQ;
    const int nqg = min(NQ, p.nq - q0);
    int pbegin = 0, pstep = 1, pnum = 0;
    if constexpr (PROBED) ivfp::resolve_items(*pr.item_count, p.tile_begin, p.tile_step, p.num_tiles, pbegin, pstep, pnum);
    const int steps = ((PROBED ? pnum : p.num_tiles) + CONSUMERS - 1) / CONSUMERS;
    // PROBED: item i of this launch, its tile and list, and whether this CTA's queries need it
    auto probed_item = [&](int i, int& tile, int& list) -> bool {
        if (i >= pnum) return false;
        const int2 it = pr.items[pbegin + i * pstep];
        list = it.x;
        tile = it.y;
        return ivfp::group_probes(pr.probed, list, q0, nqg);
    };

    if (threadIdx.x == 0) {
        ab::tma_prefetch_desc(&tmap_q);
        ab::tma_prefetch_desc(&tmap_c);
        for (int s = 0; s < STAGES; ++s) {
            ab::mbar_init(&full_bar[s], 1);
            ab::mbar_init(&empty_bar[s], CONSUMERS);
        }
        ab::mbar_init(&q_bar, 1);
        ab::fence_barrier_init();
    }
    if (threadIdx.x < NQ) {
        const int q = threadIdx.x;
        s_scale[q] = q < nqg ? p.scale[q0 + q] : 0.f;
        s_c[q] = q < nqg ? p.cterm[q0 + q] : 0.f;
        s_bnd[q] = q < nqg ? p.bound[q0 + q] : INFINITY;
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        if (warp == 0 && lane == 0) {
            ab::mbar_arrive_expect_tx(&q_bar, K_BLOCKS * Q_KB_BYTES);
            for (int kb = 0; kb < K_BLOCKS; ++kb)
                ab::tma_load_2d(&tmap_q, &q_bar, smem_gen + kb * Q_KB_BYTES, kb * 64, q0, ab::kEvictLast);
            uint32_t stage = 0, phase = 0;
            for (int g = blockIdx.x; g < steps; g += gridDim.x) {
                if constexpr (PROBED) {
                    int tile[CONSUMERS], list[CONSUMERS], ntile = 0;
                    bool has[CONSUMERS];
                    for (int c = 0; c < CONSUMERS; ++c)
                        ntile += (has[c] = probed_item(g * CONSUMERS + c, tile[c], list[c])) ? 1 : 0;
                    if (ntile == 0) continue;
                    for (int kb = 0; kb < K_BLOCKS; ++kb) {
                        ab::mbar_wait_nocall(&empty_bar[stage], phase ^ 1u);
                        ab::mbar_arrive_expect_tx(&full_bar[stage], static_cast<uint32_t>(ntile * TILE_KB_BYTES));
                        for (int c = 0; c < CONSUMERS; ++c) {
                            if (!has[c]) continue;
                            ab::tma_load_2d(&tmap_c, &full_bar[stage], smem_gen + K_BLOCKS * Q_KB_BYTES +
                                            stage * STAGE_BYTES + c * TILE_KB_BYTES, kb * SQ_KBLOCK_BYTES, tile[c] * SQ_TILE,
                                            ab::kEvictFirst);
                        }
                        if (++stage == STAGES) {
                            stage = 0;
                            phase ^= 1u;
                        }
                    }
                    continue;
                }
                const int ntile = min(CONSUMERS, p.num_tiles - g * CONSUMERS);
                for (int kb = 0; kb < K_BLOCKS; ++kb) {
                    ab::mbar_wait_nocall(&empty_bar[stage], phase ^ 1u);
                    ab::mbar_arrive_expect_tx(&full_bar[stage], static_cast<uint32_t>(ntile * TILE_KB_BYTES));
                    for (int c = 0; c < ntile; ++c) {
                        const int tile = p.tile_begin + (g * CONSUMERS + c) * p.tile_step;
                        ab::tma_load_2d(&tmap_c, &full_bar[stage], smem_gen + K_BLOCKS * Q_KB_BYTES + stage * STAGE_BYTES +
                                        c * TILE_KB_BYTES, kb * SQ_KBLOCK_BYTES, tile * SQ_TILE, ab::kEvictFirst);
                    }
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: one 64-slot tile per step =====================
    const int cw = static_cast<int>(warp >> 2) - 1;
    const int wl = static_cast<int>(warp & 3u);
    const int frag_row = wl * 16 + static_cast<int>(lane >> 2);    // fragment rows frag_row and frag_row + 8
    const int quad = static_cast<int>(lane & 3u);
    ab::mbar_wait_nocall(&q_bar, 0);
    uint32_t stage = 0, phase = 0;
    for (int g = blockIdx.x; g < steps; g += gridDim.x) {
        int tile, my_list = 0;
        bool has;
        if constexpr (PROBED) {
            has = probed_item(g * CONSUMERS + cw, tile, my_list);
            int other_tile, other_list;
            if (!has && !probed_item(g * CONSUMERS + (1 - cw), other_tile, other_list)) continue;   // the producer skips it too
        } else {
            const int item = g * CONSUMERS + cw;
            has = item < p.num_tiles;
            tile = p.tile_begin + item * p.tile_step;
        }
        float acc[NQ / 2];
#pragma unroll 1
        for (int kb = 0; kb < K_BLOCKS; ++kb) {
            ab::mbar_wait_nocall(&full_bar[stage], phase);
            uint2 v0 = make_uint2(0, 0), v1 = make_uint2(0, 0);
            if (has) {
                const uint8_t* cs = ring_gen + stage * STAGE_BYTES + cw * TILE_KB_BYTES;
                v0 = *reinterpret_cast<const uint2*>(cs + frag_row * SQ_KBLOCK_BYTES + quad * 8);
                v1 = *reinterpret_cast<const uint2*>(cs + (frag_row + 8) * SQ_KBLOCK_BYTES + quad * 8);
            }
            // the stage is read only through these loads: release it before the MMAs
            ab::named_bar_sync(1 + cw, 128);
            if (wl == 0 && lane == 0) ab::mbar_arrive(&empty_bar[stage]);
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1u;
            }
            if (!has) continue;
            uint32_t a[4][4];
#pragma unroll
            for (int w = 0; w < 2; ++w) {
                const uint32_t r0 = w ? v0.y : v0.x, r1 = w ? v1.y : v1.x;
                a[2 * w][0] = nib_lo(r0);
                a[2 * w][1] = nib_lo(r1);
                a[2 * w][2] = nib_hi(r0);
                a[2 * w][3] = nib_hi(r1);
                a[2 * w + 1][0] = nib_lo(r0 >> 8);
                a[2 * w + 1][1] = nib_lo(r1 >> 8);
                a[2 * w + 1][2] = nib_hi(r0 >> 8);
                a[2 * w + 1][3] = nib_hi(r1 >> 8);
            }
            ab::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t bdesc = ab::wgmma_desc_sw128(smem_base + kb * Q_KB_BYTES + k * 32);
                mma_step<NQ>(acc, a[k], bdesc, (kb | k) != 0 ? 1 : 0);
            }
            ab::wgmma_commit();
            ab::wgmma_wait<0>();
            ab::wgmma_reg_fence(acc);
        }
        if (!has) continue;

        // epilogue: acc[4 j + 2 e + c] = (slot frag_row + 8 e, query 8 j + 2 quad + c)
        const int list = PROBED ? my_list : p.tile_lists[tile];
        const float* trow = p.tterm + static_cast<int64_t>(list) * p.ldt + q0;
        int row[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) row[e] = p.slot_rows[static_cast<int64_t>(tile) * SQ_TILE + frag_row + 8 * e];
#pragma unroll
        for (int j = 0; j < NQ / 8; ++j) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int q = 8 * j + 2 * quad + c;
                bool pass[2] = {false, false};
                float v[2] = {0.f, 0.f};
                if (q < nqg) {
                    const float base = trow[q] + s_c[q];
                    const bool probed = !PROBED || ivfp::probes(pr.probed, list, q0 + q);
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        v[e] = fmaf(acc[4 * j + 2 * e + c], s_scale[q], base);
                        pass[e] = row[e] >= 0 && probed && v[e] >= s_bnd[q];
                    }
                }
                const uint32_t np = (pass[0] ? 1u : 0u) + (pass[1] ? 1u : 0u);
                if (!__any_sync(0xffffffffu, np != 0)) continue;
                // the 8 lanes of this quad position share query q: one atomic per (warp, query)
                uint32_t incl = np;
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
                    if (static_cast<int>(lane) >= o) incl += y;
                }
                const int last = 28 + quad;
                const uint32_t total = __shfl_sync(0xffffffffu, incl, last);
                uint32_t base_pos = 0;
                if (static_cast<int>(lane) == last && total) base_pos = atomicAdd(&p.count[q0 + q], total);
                base_pos = __shfl_sync(0xffffffffu, base_pos, last);
                uint32_t pos = base_pos + incl - np;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    if (!pass[e]) continue;
                    if (pos < p.capq)
                        p.cand[static_cast<size_t>(q0 + q) * p.capq + pos] = mips::pack_candidate(
                            mips::bits_to_key(mips::round_to_bits<false>(v[e])), static_cast<uint32_t>(row[e]));
                    ++pos;
                }
            }
        }
    }
}

template <int NQ, bool PROBED>
static int launch_nq(const CUtensorMap& tq, const CUtensorMap& tc, const ScanParams& p, const ProbeScan& pr, cudaStream_t s) {
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(ivfsq_scan_kernel<NQ, PROBED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           smem_bytes<NQ>()));
        attr_set = true;
    }
    const int groups = (p.nq + NQ - 1) / NQ;
    const int steps = (p.num_tiles + CONSUMERS - 1) / CONSUMERS;
    int gx = abh::num_sms() / groups;
    if (gx > steps) gx = steps;
    if (gx < 1) gx = 1;
    ivfsq_scan_kernel<NQ, PROBED><<<dim3(gx, groups), NUM_THREADS, smem_bytes<NQ>(), s>>>(tq, tc, p, pr);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

template <bool PROBED>
static int launch_cols(int nq_cols, const CUtensorMap& tq, const CUtensorMap& tc, const ScanParams& p, const ProbeScan& pr,
                       cudaStream_t s) {
    switch (nq_cols) {
        case 8: return launch_nq<8, PROBED>(tq, tc, p, pr, s);
        case 16: return launch_nq<16, PROBED>(tq, tc, p, pr, s);
        case 32: return launch_nq<32, PROBED>(tq, tc, p, pr, s);
        case 64: return launch_nq<64, PROBED>(tq, tc, p, pr, s);
        default: return launch_nq<128, PROBED>(tq, tc, p, pr, s);
    }
}

int launch_scan(const ScanParams& p, const ProbeScan* probe, cudaStream_t s) {
    if (p.num_tiles <= 0 || p.nq <= 0) return ATLAS_B200_OK;
    // query columns per CTA: the block's query count rounded up to a power of two >= 8, at most 128
    int nq_cols = 8;
    while (nq_cols < p.nq && nq_cols < 128) nq_cols <<= 1;
    CUtensorMap tq, tc;
    int rc = abh::make_tmap_2d_16bit(&tq, p.what, SQ_QBLOCK, SQ_DIM, SQ_DIM, static_cast<uint32_t>(nq_cols), 64, false);
    if (rc) return rc;
    rc = abh::make_tmap_2d_bytes(&tc, p.codes, static_cast<uint64_t>(p.n_tiles) * SQ_TILE, SQ_CODE_BYTES, SQ_CODE_BYTES,
                                 SQ_TILE, SQ_KBLOCK_BYTES);
    if (rc) return rc;
    return probe ? launch_cols<true>(nq_cols, tq, tc, p, *probe, s) : launch_cols<false>(nq_cols, tq, tc, p, ProbeScan{}, s);
}

}  // namespace ivfsq
