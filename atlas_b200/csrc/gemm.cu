// Dense linear layers of Contriever (BERT) and FiD (T5) on Hopper warpgroup MMAs (wgmma):
//     C[M, N] = epilogue( A[M, K] . W[N, K]^T )        A, W, C 16-bit (fp16 or bf16), fp32 accumulate
// W is the nn.Linear weight as stored ([out_features, in_features]), i.e. both operands are K-major
// and stream through TMA boxes with the 128-byte swizzle straight into wgmma shared-memory descriptors.
//
// Replaces the cuBLAS GEMM + separate ATen elementwise kernels behind
//   BertSelfAttention q/k/v, BertSelfOutput.dense, BertIntermediate.dense (+erf-GELU),
//   BertOutput.dense                                     (src/modeling_bert.py:280-466)
//   T5Attention q/k/v/o, T5DenseGatedGeluDense wi_0/wi_1 (+gelu_new gate)/wo, T5DenseReluDense wi (+ReLU)/wo, lm_head
//                                                        (src/modeling_t5.py:256-289,418-531,1642-1647)
// Fused epilogues (a template parameter of the kernel, applied to the fp32 accumulator registers):
//   EPI_NONE      C = acc
//   EPI_BIAS      C = acc + bias[n]
//   EPI_GELU      C = gelu_erf(acc + bias[n])                      (ACT2FN["gelu"], modeling_bert.py:444)
//   EPI_RESIDUAL  C = acc + bias[n] + R[m, n]                      (dense + residual, LN follows)
//   EPI_GATED     C[m, j] = gelu_new(acc[m, 2j]) * acc[m, 2j+1]    (W rows interleaved wi_0/wi_1;
//                                                                   modeling_t5.py:281-285, fp32 GELU)
//   EPI_RELU      C = max(acc + bias[n], 0)                        (T5 v1.0 T5DenseReluDense, modeling_t5.py:263-265;
//                                                                   with row_ss the row scale comes first: relu(s acc))
//
// Persistent, warp-specialised, one CTA per SM (grid = #SMs): warpgroup 0 is the TMA producer (one thread; setmaxnreg
// gives its registers to the consumers), warpgroups 1 and 2 are consumers.  Three schedules:
//   wide (gemm_wide_kernel; the encoder-sized K-major launches with the plain epilogue: the q|k|v projection, the
//     cross-attention K|V projection, the input-gradient GEMMs of training): both consumers share one 128 x 256 tile,
//     64 rows each, one wgmma m64n256k16 per k16 step on a shared W block, then a TMA-store epilogue through a 32 KB
//     staging buffer per consumer that overlaps the next tile's mainloop.  3 stages of 48 KB.  It implements every
//     epilogue (ATLAS_B200_GEMM_SCHEDULE=wide runs it for all encoder-sized launches); the rule sends it only the plain one.
//   ping-pong (gemm_pp_kernel; the other K-major launches of at least 2 x #SMs 128 x 128 tiles, i.e. the encoder
//     projections with a fused bias / activation / residual / gate, and the LM head at 256 rows x 32128, whose 251
//     column tiles would pad to 252 at 256 wide): each consumer owns whole 128 x 128 tiles, two wgmma m64n128k16 per k16 step
//     sharing the W descriptor; a CTA's work items alternate between the consumers, which take turns in the mainloop, so
//     one consumer's epilogue runs under the other's MMAs.  The epilogue goes through a per-consumer 32 KB staging buffer
//     (128-byte swizzle) and a TMA store; EPI_RESIDUAL's residual tile is loaded into that buffer by the producer during
//     the item's mainloop.  5 stages of 32 KB.
//   cooperative (gemm_kernel; smaller launches - the decoder's other 256-row GEMMs, Contriever's query batch - and
//     the MN-major weight-gradient / split-K path): both consumers share one 128 x BLOCK_N tile (BLOCK_N = 256 once there
//     are enough tiles to fill the SMs, else 128), 64 rows each, wgmma m64nBLOCK_Nk16, then the epilogue straight from the
//     accumulator registers to global memory (EPI_RESIDUAL: the tile's residual rows are prefetched into L2 before its
//     mainloop and read in batches of independent loads).  A ring of 64-wide K stages (~200 KB).
// The choice depends only on the shape and epilogue (and, for EPI_RESIDUAL, on a 16-byte aligned residual, which its
// tensor map needs): select_schedule, reported by atlas_b200_linear_schedule.  All schedules run each output element
// through the same sequence of k16 MMAs and the same epilogue arithmetic (epilogue_pair), so they give bit-identical results.
#include "common.cuh"
#include "host_common.h"
#include "wgmma.cuh"

#include <math.h>
#include <stdlib.h>
#include <string.h>

namespace gemm {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int UMMA_K = 16;      // K of one wgmma
constexpr int CONSUMERS = 2;    // consumer warpgroups
constexpr int THREADS = 128 * (1 + CONSUMERS);

enum Epilogue { EPI_NONE = 0, EPI_BIAS = 1, EPI_GELU = 2, EPI_RESIDUAL = 3, EPI_GATED = 4, EPI_RELU = 5 };

template <int BLOCK_N>
struct Cfg {
    static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
    static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (200 * 1024) / STAGE_BYTES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
};

struct Params {
    int M, N, K;
    int ldc;              // elements; for EPI_GATED C has N/2 columns
    int ldr;              // residual row stride
    const uint16_t* bias;      // [N] 16-bit or nullptr
    const uint16_t* residual;  // [M, ldr] 16-bit or nullptr
    uint16_t* C;
    // fused T5 RMSNorm (src/modeling_t5.py:244-253) around the GEMM:
    //   row_ss  [M] fp32 sum of squares of the A rows (or nullptr): acc[m, :] *= rsqrt(row_ss[m] / K + rs_eps) before the
    //           epilogue, i.e. the GEMM consumes the UN-normalised rows with the norm weight folded into W
    //   out_ss  [M] fp32 (or nullptr): += sum over this launch's columns of (16-bit rounded output)^2, the statistic the
    //           next RMSNorm needs, accumulated with one atomicAdd per row, quad and tile
    const float* row_ss;
    float* out_ss;
    float rs_eps;
    // split-K (weight gradients: few output tiles, very long contraction): work item = (tile, split); split s covers the
    // k-blocks [s * kb_per_split, (s + 1) * kb_per_split) and stores its fp32 partial tile to C32 + s * M * N (row stride N);
    // splitk_reduce_kernel sums the partials and rounds once.  splits == 1 / C32 == nullptr: the ordinary epilogues.
    int splits, kb_per_split;
    float* C32;
    int l2_prefetch;      // producer prefetches the next work item's A rows into L2 (off for the weight gradients)
    const int32_t* m_dev; // optional: the number of valid rows lives in device memory (<= M): only ceil(*m_dev / tile) row blocks
                          // are computed (compacted activations under a CUDA graph: the launch shape stays static)
};

template <bool kBF16>
__device__ __forceinline__ float to_f32(uint16_t h) {
    if constexpr (kBF16) return __bfloat162float(__ushort_as_bfloat16(h));
    return __half2float(__ushort_as_half(h));
}
template <bool kBF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    return ab::pack2_rn<kBF16>(a, b);
}

// erf-GELU (ACT2FN["gelu"]): 0.5 x (1 + erf(x / sqrt 2)).  erf by Abramowitz-Stegun 7.1.26 (|abs error| <= 1.5e-7, i.e.
// fp32-level on 1 + erf): t = 1 / (1 + p|z|), erf|z| = 1 - (a1 t + ... + a5 t^5) e^(-z^2) -- one MUFU.RCP, one MUFU.EX2 and
// six FMAs instead of erff's ~25-instruction two-branch polynomial (the 128 x 256 GELU epilogue was as long as the MMAs).
__device__ __forceinline__ float gelu_erf(float x) {
    const float z = fabsf(x) * 0.70710678118654752f;
    float t, e;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z * z));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float erfc_abs = poly * t * e;                       // 1 - erf(|z|)
    const float one_plus_erf = x >= 0.f ? 2.0f - erfc_abs : erfc_abs;
    return 0.5f * x * one_plus_erf;
}
// transformers' "gelu_new": 0.5*x*(1+tanh(sqrt(2/pi)*(x+0.044715*x^3)))
// = x * sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3): 1 + tanh(u) = 2 / (1 + e^(-2u)).  One MUFU.EX2 and one
// MUFU.RCP (both ~1e-7 relative) instead of tanhf's ~30-instruction path: the 128 x 256 gated epilogue (16 k GELUs
// per tile) was longer than the tile's MMAs.  e^(-2u) = inf for very negative x gives x / inf = -0 (true value ~0).
__device__ __forceinline__ float gelu_new(float x) {
    const float u2 = x * (1.5957691216057308f + 0.07135481627260025f * x * x);    // 2u
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * u2));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return x * r;
}

// ---- the fused epilogue, shared by both schedules: the same fp32 operations in the same order, one rounding to 16 bits
// rsqrt(row_ss / K + eps) of output row `row` (fused RMSNorm), or 1
__device__ __forceinline__ float row_scale(const Params& p, int row, bool row_ok) {
    return (p.row_ss != nullptr && row_ok) ? rsqrtf(__ldg(p.row_ss + row) / static_cast<float>(p.K) + p.rs_eps) : 1.0f;
}
// accumulators (v0, v1) of columns (col, col + 1) -> the packed 16-bit pair to store; `res` is the packed residual pair
// (EPI_RESIDUAL).  EPI_GATED: columns (2c, 2c+1) = (x.wi_0[c], x.wi_1[c]) -> one output, in the low half.
template <bool kBF16, int kEpi>
__device__ __forceinline__ uint32_t epilogue_pair(const Params& p, float v0, float v1, float rscale, int col, uint32_t res) {
    v0 *= rscale;
    v1 *= rscale;
    if constexpr (kEpi == EPI_GATED) return pack2<kBF16>(gelu_new(v0) * v1, 0.f);
    if (kEpi != EPI_NONE && p.bias != nullptr) {
        const uint32_t b = __ldg(reinterpret_cast<const uint32_t*>(p.bias + col));
        v0 += to_f32<kBF16>(static_cast<uint16_t>(b & 0xFFFFu));
        v1 += to_f32<kBF16>(static_cast<uint16_t>(b >> 16));
    }
    if constexpr (kEpi == EPI_GELU) {
        v0 = gelu_erf(v0);
        v1 = gelu_erf(v1);
    } else if constexpr (kEpi == EPI_RESIDUAL) {
        v0 += to_f32<kBF16>(static_cast<uint16_t>(res & 0xFFFFu));
        v1 += to_f32<kBF16>(static_cast<uint16_t>(res >> 16));
    } else if constexpr (kEpi == EPI_RELU) {
        // written as a select so that NaN propagates like torch.relu (fmaxf would return 0)
        v0 = v0 < 0.f ? 0.f : v0;
        v1 = v1 < 0.f ? 0.f : v1;
    }
    return pack2<kBF16>(v0, v1);
}
// out_ss: squares of the values as STORED (what a separate norm would read)
template <bool kBF16>
__device__ __forceinline__ float add_sq_pair(uint32_t o, float ss) {
    const float a = to_f32<kBF16>(static_cast<uint16_t>(o & 0xFFFFu));
    const float b = to_f32<kBF16>(static_cast<uint16_t>(o >> 16));
    return fmaf(a, a, fmaf(b, b, ss));
}
// the four threads of a quad hold the same row: one atomicAdd per row and quad (every lane of the warp calls this)
__device__ __forceinline__ void out_ss_add(const Params& p, int row, bool row_ok, uint32_t lane, float ss) {
    ss += __shfl_xor_sync(0xffffffffu, ss, 1);
    ss += __shfl_xor_sync(0xffffffffu, ss, 2);
    if (row_ok && (lane & 3u) == 0u) atomicAdd(p.out_ss + row, ss);
}

// kTN = false: C = A[M, K] . W[N, K]^T, both operands K-major (activations x nn.Linear weight).
// kTN = true : C[M, N] = A[K, M]^T . W[K, N]: both operands MN-major, i.e. the contraction runs over the ROWS of two
//              row-major matrices - the weight gradient dW[N_out, K_in] = dY[tokens, N_out]^T . X[tokens, K_in] without
//              transposing either activation matrix (rows past K are zero-filled by TMA: no padding needed).
//              wgmma reads 16-bit MN-major tiles through its transpose flags: boxes of {64 MN elements, 64 K rows}, MN
//              blocks 8 KB apart (descriptor LBO).
// kEpi: the epilogue (EPI_*), a compile-time choice; the MN-major path runs EPI_NONE (or the split-K partial store).
template <bool kBF16, int BLOCK_N, bool kTN, int kEpi>
__global__ void __launch_bounds__(THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const Params p) {
    using C = Cfg<BLOCK_N>;
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[C::STAGES];
    __shared__ __align__(8) uint64_t empty_bar[C::STAGES];

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));

    const int m_rows = p.m_dev != nullptr ? min(p.M, max(__ldg(p.m_dev), 0)) : p.M;     // identical in every role
    const int num_m = (m_rows + BLOCK_M - 1) / BLOCK_M;
    const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
    const int num_tiles = num_m * num_n * p.splits;     // work items: (tile, split), split fastest
    const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

    if (threadIdx.x == 0) {
        ab::tma_prefetch_desc(&tmap_a);
        ab::tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < C::STAGES; ++s) {
            ab::mbar_init(&full_bar[s], 1);
            ab::mbar_init(&empty_bar[s], CONSUMERS);          // one arrive per consumer warpgroup
        }
        ab::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== producer warpgroup (one thread issues the TMA loads) =====================
        ab::setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const int tile = t / p.splits, split = t % p.splits;
                const int m_blk = tile / num_n, n_blk = tile % num_n;
                const int a_row = m_blk * BLOCK_M;
                const int b_row = n_blk * BLOCK_N;
                const int kb0 = split * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
                // L2 prefetch of the A rows of this CTA's NEXT work item when it starts a new row block
                int pf_row = -1;
                if constexpr (!kTN) {
                    const int t2 = t + static_cast<int>(gridDim.x);
                    if (p.l2_prefetch && t2 < num_tiles && (t2 / p.splits) % num_n == 0) pf_row = ((t2 / p.splits) / num_n) * BLOCK_M;
                }
                for (int kb = kb0; kb < kb1; ++kb) {
                    if (pf_row >= 0) ab::tma_prefetch_2d(&tmap_a, kb * BLOCK_K, pf_row);
                    ab::mbar_wait_nocall(&empty_bar[stage], phase ^ 1u);
                    uint8_t* st = smem_gen + stage * C::STAGE_BYTES;
                    ab::mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
                    if constexpr (kTN) {
#pragma unroll
                        for (int j = 0; j < BLOCK_M / 64; ++j)
                            ab::tma_load_2d(&tmap_a, &full_bar[stage], st + j * 8192, a_row + 64 * j, kb * BLOCK_K,
                                            ab::kEvictNormal);
#pragma unroll
                        for (int j = 0; j < BLOCK_N / 64; ++j)
                            ab::tma_load_2d(&tmap_b, &full_bar[stage], st + C::A_BYTES + j * 8192, b_row + 64 * j,
                                            kb * BLOCK_K, ab::kEvictNormal);
                    } else {
                        ab::tma_load_2d(&tmap_a, &full_bar[stage], st, kb * BLOCK_K, a_row, ab::kEvictNormal);
                        ab::tma_load_2d(&tmap_b, &full_bar[stage], st + C::A_BYTES, kb * BLOCK_K, b_row, ab::kEvictLast);
                    }
                    if (++stage == C::STAGES) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroups: 64 rows x BLOCK_N columns each =====================
    ab::setmaxnreg_inc<232>();
    const uint32_t wg = (warp >> 2) - 1u;              // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
    const uint32_t wl = warp & 3u;                     // warp inside the warpgroup
    constexpr int NACC = BLOCK_N / 2;
    constexpr int RES_BATCH = 8;                       // residual loads in flight per thread
    uint32_t stage = 0, phase = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int tile = t / p.splits, split = t % p.splits;
        const int m_blk = tile / num_n, n_blk = tile % num_n;
        const int kb0 = split * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
        const int r0 = m_blk * BLOCK_M + static_cast<int>(wg * 64u + wl * 16u + (lane >> 2));
        const int cq = static_cast<int>(2u * (lane & 3u));
        if constexpr (kEpi == EPI_RESIDUAL) {
            // pull this thread's residual rows into L2 while the mainloop runs: the activations are larger than L2, and the
            // epilogue would otherwise wait out DRAM latency on them (each lane of a quad takes a quarter of the row segment)
            const int col = n_blk * BLOCK_N + static_cast<int>(lane & 3u) * (BLOCK_N / 4);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h;
                if (row < p.M && col < p.N)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + static_cast<size_t>(row) * p.ldr + col));
            }
        }
        float acc[NACC];
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        int prev_stage = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            ab::mbar_wait_nocall(&full_bar[stage], phase);
            const uint32_t st = smem_base + stage * C::STAGE_BYTES;
            ab::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
                uint64_t adesc, bdesc;
                if constexpr (kTN) {
                    adesc = ab::wgmma_desc_sw128(st + wg * 8192u + k * 2048u, 8192);
                    bdesc = ab::wgmma_desc_sw128(st + C::A_BYTES + k * 2048u, 8192);
                } else {
                    adesc = ab::wgmma_desc_sw128(st + wg * 8192u + k * 32u);
                    bdesc = ab::wgmma_desc_sw128(st + C::A_BYTES + k * 32u);
                }
                if constexpr (BLOCK_N == 256)
                    ab::wgmma_m64n256k16_ss<kBF16, kTN ? 1 : 0, kTN ? 1 : 0>(acc, adesc, bdesc, 1);
                else
                    ab::wgmma_m64n128k16_ss<kBF16, kTN ? 1 : 0, kTN ? 1 : 0>(acc, adesc, bdesc, 1);
            }
            ab::wgmma_commit();
            // the previous stage's MMAs have retired once at most this stage's group is pending: release it
            ab::wgmma_wait<1>();
            ab::wgmma_reg_fence(acc);
            if (prev_stage >= 0 && wl == 0 && lane == 0) ab::mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = static_cast<int>(stage);
            if (++stage == C::STAGES) {
                stage = 0;
                phase ^= 1u;
            }
        }
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(acc);
        if (prev_stage >= 0 && wl == 0 && lane == 0) ab::mbar_arrive(&empty_bar[prev_stage]);

        // ---- epilogue straight from the accumulator registers: rows r0 and r0 + 8, column pairs 8 j + 2 (lane % 4)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            const bool row_ok = row < p.M;
            const float rscale = row_scale(p, row, row_ok);
            float ss_out = 0.f;
            if (row_ok) {
#pragma unroll
              for (int jb = 0; jb < BLOCK_N / 8; jb += RES_BATCH) {
                // a batch of independent residual loads issued together, ahead of the batch's stores.  Plain (coherent) loads:
                // the compiler treats them as possibly aliasing the stores and keeps them in place, whereas read-only (.nc)
                // loads get sunk to their uses, one dependent memory latency per column pair.
                uint32_t res[RES_BATCH];
                if constexpr (kEpi == EPI_RESIDUAL) {
#pragma unroll
                    for (int jj = 0; jj < RES_BATCH; ++jj) {
                        const int col = n_blk * BLOCK_N + 8 * (jb + jj) + cq;
                        res[jj] = col < p.N ? *reinterpret_cast<const uint32_t*>(p.residual + static_cast<size_t>(row) * p.ldr + col)
                                            : 0u;
                    }
                }
#pragma unroll
                for (int jj = 0; jj < RES_BATCH; ++jj) {
                    const int j = jb + jj;
                    const int col = n_blk * BLOCK_N + 8 * j + cq;
                    if (col >= p.N) continue;
                    const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                    if constexpr (kTN) {
                        if (p.C32 != nullptr) {   // split-K partial: raw fp32 accumulator
                            *reinterpret_cast<float2*>(p.C32 + (static_cast<size_t>(split) * p.M + row) * p.N + col) =
                                make_float2(v0, v1);
                            continue;
                        }
                    }
                    const uint32_t o = epilogue_pair<kBF16, kEpi>(p, v0, v1, rscale, col,
                                                                  kEpi == EPI_RESIDUAL ? res[jj] : 0u);
                    if constexpr (kEpi == EPI_GATED) {
                        p.C[static_cast<size_t>(row) * p.ldc + (col >> 1)] = static_cast<uint16_t>(o & 0xFFFFu);
                        continue;
                    }
                    *reinterpret_cast<uint32_t*>(p.C + static_cast<size_t>(row) * p.ldc + col) = o;
                    if (p.out_ss != nullptr) ss_out = add_sq_pair<kBF16>(o, ss_out);
                }
              }
            }
            if (p.out_ss != nullptr) out_ss_add(p, row, row_ok, lane, ss_out);
        }
    }
}

// ===================== ping-pong schedule (K-major, 128 x 128 tiles, encoder-sized launches) =====================
namespace pp {
constexpr int BLOCK_N = 128;
constexpr int STAGE_BYTES = (BLOCK_M + BLOCK_N) * BLOCK_K * 2;      // 32 KB: A 128 x 64, W 128 x 64
constexpr int EPI_BYTES = BLOCK_M * BLOCK_N * 2;                    // 32 KB staging tile per consumer: two 128 x 64 boxes
constexpr int STAGES = (227 * 1024 - 1024 - CONSUMERS * EPI_BYTES) / STAGE_BYTES;    // 5
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + CONSUMERS * EPI_BYTES + 1024;
// named barriers: consumer c waits on ORDER_BAR + c for its turn in the mainloop; EPI_BAR + c syncs its 128 threads
constexpr uint32_t ORDER_BAR = 1, EPI_BAR = 3;
// byte offset of element (r, c) in a 128-row box of 64 16-bit columns written with the 128-byte swizzle (what TMA
// reads and writes): 16-byte chunk c / 8 of row r lands at chunk (c / 8) ^ (r % 8)
__device__ __forceinline__ uint32_t sw128_offset(int r, int c) {
    return static_cast<uint32_t>(r * 128 + ((((c >> 3) ^ r) & 7) << 4) + ((c & 7) << 1));
}
}  // namespace pp

// Each consumer warpgroup owns whole 128 x 128 tiles: the CTA's work items alternate between the consumers (item i ->
// consumer i % 2).  The producer loads the stages of every item in order into one ring; the consumers take turns in the
// mainloop (named barriers), so one consumer's epilogue runs while the other issues MMAs.  The epilogue writes the tile
// into the consumer's shared-memory staging buffer, and one thread stores it with TMA through the tensor map of C, whose
// extent clips ragged edges (and keeps a strided view's neighbouring columns untouched).  EPI_RESIDUAL: the producer
// loads the residual tile into that buffer with TMA during the item's mainloop; the epilogue adds it in place.
template <bool kBF16, int kEpi>
__global__ void __launch_bounds__(THREADS, 1)
gemm_pp_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r, const Params p) {
    using namespace pp;
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];
    __shared__ __align__(8) uint64_t res_full[CONSUMERS];     // residual tile landed in the staging buffer
    __shared__ __align__(8) uint64_t res_empty[CONSUMERS];    // staging buffer read out by the previous TMA store

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));
    uint8_t* epi_gen = smem_gen + STAGES * STAGE_BYTES;

    const int m_rows = p.m_dev != nullptr ? min(p.M, max(__ldg(p.m_dev), 0)) : p.M;     // identical in every role
    const int num_m = (m_rows + BLOCK_M - 1) / BLOCK_M;
    const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
    const int num_tiles = num_m * num_n;
    const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

    if (threadIdx.x == 0) {
        ab::tma_prefetch_desc(&tmap_a);
        ab::tma_prefetch_desc(&tmap_b);
        ab::tma_prefetch_desc(&tmap_c);
        if constexpr (kEpi == EPI_RESIDUAL) ab::tma_prefetch_desc(&tmap_r);
        for (int s = 0; s < STAGES; ++s) {
            ab::mbar_init(&full_bar[s], 1);
            ab::mbar_init(&empty_bar[s], 1);                  // one consumer per stage
        }
        for (int c = 0; c < CONSUMERS; ++c) {
            ab::mbar_init(&res_full[c], 1);
            ab::mbar_init(&res_empty[c], 1);
        }
        ab::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== producer warpgroup (one thread issues the TMA loads) =====================
        ab::setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            int i = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++i) {
                const int m_blk = t / num_n, n_blk = t % num_n;
                const int a_row = m_blk * BLOCK_M;
                const int b_row = n_blk * BLOCK_N;
                // L2 prefetch of the A rows of this CTA's NEXT work item when it starts a new row block
                int pf_row = -1;
                const int t2 = t + static_cast<int>(gridDim.x);
                if (p.l2_prefetch && t2 < num_tiles && t2 % num_n == 0) pf_row = (t2 / num_n) * BLOCK_M;
                bool res_issued = false;
                for (int kb = 0; kb < num_kb; ++kb) {
                    if (pf_row >= 0) ab::tma_prefetch_2d(&tmap_a, kb * BLOCK_K, pf_row);
                    ab::mbar_wait_nocall(&empty_bar[stage], phase ^ 1u);
                    uint8_t* st = smem_gen + stage * STAGE_BYTES;
                    ab::mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
                    ab::tma_load_2d(&tmap_a, &full_bar[stage], st, kb * BLOCK_K, a_row, ab::kEvictNormal);
                    ab::tma_load_2d(&tmap_b, &full_bar[stage], st + BLOCK_M * BLOCK_K * 2, kb * BLOCK_K, b_row,
                                    ab::kEvictLast);
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1u;
                    }
                    if constexpr (kEpi == EPI_RESIDUAL) {
                        // the residual tile, as early in the item's mainloop as its consumer's staging buffer is free (the
                        // store of that consumer's previous tile has read it).  The buffer is probed after each k-block
                        // and waited for only after the last one, so the stage loads never stall on it.
                        const int c = i & 1;
                        const uint32_t par = ((static_cast<uint32_t>(i >> 1)) & 1u) ^ 1u;
                        if (!res_issued && (kb == num_kb - 1 || ab::mbar_test_wait(&res_empty[c], par))) {
                            ab::mbar_wait_nocall(&res_empty[c], par);
                            res_issued = true;
                            uint8_t* buf = epi_gen + c * EPI_BYTES;
                            ab::mbar_arrive_expect_tx(&res_full[c], EPI_BYTES);
                            ab::tma_load_2d(&tmap_r, &res_full[c], buf, b_row, a_row, ab::kEvictFirst);
                            ab::tma_load_2d(&tmap_r, &res_full[c], buf + EPI_BYTES / 2, b_row + 64, a_row, ab::kEvictFirst);
                        }
                    }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroups: whole 128 x 128 tiles, alternating =====================
    ab::setmaxnreg_inc<232>();
    const uint32_t wg = (warp >> 2) - 1u;              // consumer 0 / 1
    const uint32_t wl = warp & 3u;                     // warp inside the warpgroup
    const uint32_t ctid = threadIdx.x & 127u;
    uint8_t* buf = epi_gen + wg * EPI_BYTES;
    const int cq = static_cast<int>(2u * (lane & 3u));
    const int stride = static_cast<int>(gridDim.x);
    int i = static_cast<int>(wg);
    for (int t = blockIdx.x + i * stride; t < num_tiles; t += 2 * stride, i += 2) {
        const int m_blk = t / num_n, n_blk = t % num_n;
        // this item's first stage: every item has num_kb k-blocks, loaded in item order
        const int pos = i * num_kb;
        uint32_t stage = static_cast<uint32_t>(pos % STAGES), phase = static_cast<uint32_t>((pos / STAGES) & 1);
        // wait for the other consumer to have issued the previous item's mainloop.  Consumer 0's first item has no
        // predecessor.  This barrier also covers the previous store of this consumer's staging buffer: the thread that
        // issued it arrives here only after waiting for the store to have read the buffer.
        if (i > 0) ab::named_bar_sync(ORDER_BAR + wg, 256);
        float acc[2][64];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < 64; ++q) acc[h][q] = 0.f;
        int prev_stage = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
            ab::mbar_wait_nocall(&full_bar[stage], phase);
            const uint32_t st = smem_base + stage * STAGE_BYTES;
            ab::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
                const uint64_t bdesc = ab::wgmma_desc_sw128(st + BLOCK_M * BLOCK_K * 2 + k * 32u);
                ab::wgmma_m64n128k16_ss<kBF16, 0, 0>(acc[0], ab::wgmma_desc_sw128(st + k * 32u), bdesc, 1);
                ab::wgmma_m64n128k16_ss<kBF16, 0, 0>(acc[1], ab::wgmma_desc_sw128(st + 8192u + k * 32u), bdesc, 1);
            }
            ab::wgmma_commit();
            // the previous stage's MMAs have retired once at most this stage's group is pending: release it
            ab::wgmma_wait<1>();
            ab::wgmma_reg_fence(acc[0]);
            ab::wgmma_reg_fence(acc[1]);
            if (prev_stage >= 0 && ctid == 0) ab::mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = static_cast<int>(stage);
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1u;
            }
        }
        // the other consumer's turn (if it has a next item)
        if (t + stride < num_tiles) ab::named_bar_arrive(ORDER_BAR + (wg ^ 1u), 256);
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(acc[0]);
        ab::wgmma_reg_fence(acc[1]);
        if (prev_stage >= 0 && ctid == 0) ab::mbar_arrive(&empty_bar[prev_stage]);

        // ---- epilogue into the staging buffer: rows 64 mh + 16 wl + lane / 4 (+ 8), column pairs 8 j + 2 (lane % 4)
        if constexpr (kEpi == EPI_RESIDUAL) ab::mbar_wait_nocall(&res_full[wg], static_cast<uint32_t>((i >> 1) & 1));
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = mh * 64 + static_cast<int>(wl * 16u + (lane >> 2)) + 8 * h;    // row in the tile
                const int row = m_blk * BLOCK_M + r;
                const bool row_ok = row < p.M;
                const float rscale = row_scale(p, row, row_ok);
                float ss_out = 0.f;
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; ++j) {
                    const int c = 8 * j + cq;                                                  // column in the tile
                    const int col = n_blk * BLOCK_N + c;
                    if (col >= p.N) continue;                  // past the edge: the TMA store clips it
                    uint8_t* dst = buf + (c >> 6) * (EPI_BYTES / 2) + sw128_offset(r, c & 63);
                    const uint32_t res = kEpi == EPI_RESIDUAL ? *reinterpret_cast<const uint32_t*>(dst) : 0u;
                    const uint32_t o = epilogue_pair<kBF16, kEpi>(p, acc[mh][4 * j + 2 * h], acc[mh][4 * j + 2 * h + 1],
                                                                  rscale, col, res);
                    if constexpr (kEpi == EPI_GATED) {
                        *reinterpret_cast<uint16_t*>(buf + sw128_offset(r, c >> 1)) = static_cast<uint16_t>(o & 0xFFFFu);
                    } else {
                        *reinterpret_cast<uint32_t*>(dst) = o;
                        if (p.out_ss != nullptr) ss_out = add_sq_pair<kBF16>(o, ss_out);
                    }
                }
                if (kEpi != EPI_GATED && p.out_ss != nullptr) out_ss_add(p, row, row_ok, lane, ss_out);
            }
        }
        ab::fence_proxy_async_smem();                  // generic-proxy writes -> visible to the TMA store
        ab::named_bar_sync(EPI_BAR + wg, 128);
        if (ctid == 0) {
            if constexpr (kEpi == EPI_GATED) {
                ab::tma_store_2d(&tmap_c, buf, n_blk * (BLOCK_N / 2), m_blk * BLOCK_M);
            } else {
                ab::tma_store_2d(&tmap_c, buf, n_blk * BLOCK_N, m_blk * BLOCK_M);
                ab::tma_store_2d(&tmap_c, buf + EPI_BYTES / 2, n_blk * BLOCK_N + 64, m_blk * BLOCK_M);
            }
            ab::tma_store_commit();
            ab::tma_store_wait_read();
            if constexpr (kEpi == EPI_RESIDUAL) ab::mbar_arrive(&res_empty[wg]);
        }
    }
    if (ctid == 0) ab::tma_store_wait_all();
}

// ===================== wide schedule (K-major, 128 x 256 tiles, encoder-sized launches) =====================
namespace wd {
constexpr int BLOCK_N = 256;
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;                      // 16 KB
constexpr int STAGE_BYTES = (BLOCK_M + BLOCK_N) * BLOCK_K * 2;      // 48 KB: A 128 x 64, W 256 x 64
constexpr int BOX_BYTES = 64 * 64 * 2;                              // one 64-row x 64-column box of C / the residual
constexpr int EPI_BYTES = 64 * BLOCK_N * 2;                         // 32 KB staging per consumer: its 64 rows, four boxes
constexpr int STAGES = (227 * 1024 - 1024 - CONSUMERS * EPI_BYTES) / STAGE_BYTES;    // 3
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + CONSUMERS * EPI_BYTES + 1024;
constexpr uint32_t EPI_BAR = 1;                                     // EPI_BAR + c syncs consumer c's 128 threads
}  // namespace wd

// Both consumers work on the same 128 x 256 tile: each stage holds one A block (128 x 64) and one W block (256 x 64), and
// consumer c runs one wgmma m64n256k16 per k16 step on A rows [64 c, 64 c + 64) against the whole W block.  Per FLOP this
// reads half the W bytes from shared memory that a 128 x 128 tile (two m64n128 sharing a W slice) does, and fills half
// as many bytes per FLOP by TMA.  Each consumer releases a stage on its own (empty_bar counts two arrivals).  The epilogue
// writes the consumer's 64 x 256 slice into its own 32 KB staging buffer (four 64 x 64 boxes, 128-byte swizzle) and one
// thread stores it with TMA; the consumer starts the next tile's mainloop without waiting for the store, and waits for it
// to have read the buffer only during that mainloop.  EPI_RESIDUAL: the producer loads the consumer's residual slice into
// the staging buffer during the tile's mainloop, as soon as the previous store has read it.  The two consumers reach their
// epilogues together; starting consumer 1 two k-blocks after consumer 0 (all the 3-stage ring allows) was measured and
// did not shorten any encoder shape (see select_schedule), so they run in step.
template <bool kBF16, int kEpi>
__global__ void __launch_bounds__(THREADS, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r, const Params p) {
    using namespace wd;
    using pp::sw128_offset;
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];
    __shared__ __align__(8) uint64_t res_full[CONSUMERS];     // residual slice landed in the staging buffer
    __shared__ __align__(8) uint64_t res_empty[CONSUMERS];    // staging buffer read out by the previous TMA store

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));
    uint8_t* epi_gen = smem_gen + STAGES * STAGE_BYTES;

    const int m_rows = p.m_dev != nullptr ? min(p.M, max(__ldg(p.m_dev), 0)) : p.M;     // identical in every role
    const int num_m = (m_rows + BLOCK_M - 1) / BLOCK_M;
    const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
    const int num_tiles = num_m * num_n;
    const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;
    const int n_out = kEpi == EPI_GATED ? p.N / 2 : p.N;                 // columns of C
    constexpr int OUT_BOXES = kEpi == EPI_GATED ? 2 : 4;                // 64-column boxes of C per tile

    if (threadIdx.x == 0) {
        ab::tma_prefetch_desc(&tmap_a);
        ab::tma_prefetch_desc(&tmap_b);
        ab::tma_prefetch_desc(&tmap_c);
        if constexpr (kEpi == EPI_RESIDUAL) ab::tma_prefetch_desc(&tmap_r);
        for (int s = 0; s < STAGES; ++s) {
            ab::mbar_init(&full_bar[s], 1);
            ab::mbar_init(&empty_bar[s], CONSUMERS);          // one arrive per consumer warpgroup
        }
        for (int c = 0; c < CONSUMERS; ++c) {
            ab::mbar_init(&res_full[c], 1);
            ab::mbar_init(&res_empty[c], 1);
        }
        ab::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== producer warpgroup (one thread issues the TMA loads) =====================
        ab::setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            int i = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++i) {
                const int m_blk = t / num_n, n_blk = t % num_n;
                const int a_row = m_blk * BLOCK_M;
                const int b_row = n_blk * BLOCK_N;
                // L2 prefetch of the A rows of this CTA's NEXT work item when it starts a new row block
                int pf_row = -1;
                const int t2 = t + static_cast<int>(gridDim.x);
                if (p.l2_prefetch && t2 < num_tiles && t2 % num_n == 0) pf_row = (t2 / num_n) * BLOCK_M;
                bool res_issued[CONSUMERS] = {false, false};
                for (int kb = 0; kb < num_kb; ++kb) {
                    if (pf_row >= 0) ab::tma_prefetch_2d(&tmap_a, kb * BLOCK_K, pf_row);
                    ab::mbar_wait_nocall(&empty_bar[stage], phase ^ 1u);
                    uint8_t* st = smem_gen + stage * STAGE_BYTES;
                    ab::mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
                    ab::tma_load_2d(&tmap_a, &full_bar[stage], st, kb * BLOCK_K, a_row, ab::kEvictNormal);
                    ab::tma_load_2d(&tmap_b, &full_bar[stage], st + A_BYTES, kb * BLOCK_K, b_row, ab::kEvictLast);
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1u;
                    }
                    if constexpr (kEpi == EPI_RESIDUAL) {
                        // each consumer's residual slice, as early in the tile's mainloop as its staging buffer is free.
                        // The buffer is probed after each k-block and waited for only after the last one, so the stage
                        // loads never stall on it.  Boxes wholly past the edge of R are not loaded (their columns are
                        // skipped by the epilogue, their rows clipped by the store).
                        const uint32_t par = (static_cast<uint32_t>(i) & 1u) ^ 1u;
                        for (int c = 0; c < CONSUMERS; ++c) {
                            if (res_issued[c] || !(kb == num_kb - 1 || ab::mbar_test_wait(&res_empty[c], par))) continue;
                            ab::mbar_wait_nocall(&res_empty[c], par);
                            res_issued[c] = true;
                            uint8_t* buf = epi_gen + c * EPI_BYTES;
                            const int r_row = a_row + 64 * c;
                            int boxes = 0;
                            if (r_row < p.M)
                                for (int b = 0; b < 4 && b_row + 64 * b < p.N; ++b) ++boxes;
                            ab::mbar_arrive_expect_tx(&res_full[c], boxes * BOX_BYTES);
                            for (int b = 0; b < boxes; ++b)
                                ab::tma_load_2d(&tmap_r, &res_full[c], buf + b * BOX_BYTES, b_row + 64 * b, r_row,
                                                ab::kEvictFirst);
                        }
                    }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroups: 64 rows x 256 columns each of every tile =====================
    ab::setmaxnreg_inc<232>();
    const uint32_t wg = (warp >> 2) - 1u;              // rows [64 wg, 64 wg + 64) of the tile
    const uint32_t wl = warp & 3u;                     // warp inside the warpgroup
    const uint32_t ctid = threadIdx.x & 127u;
    uint8_t* buf = epi_gen + wg * EPI_BYTES;
    const int cq = static_cast<int>(2u * (lane & 3u));
    uint32_t stage = 0, phase = 0;
    int i = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++i) {
        const int m_blk = t / num_n, n_blk = t % num_n;
        float acc[BLOCK_N / 2];
#pragma unroll
        for (int q = 0; q < BLOCK_N / 2; ++q) acc[q] = 0.f;
        int prev_stage = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
            ab::mbar_wait_nocall(&full_bar[stage], phase);
            const uint32_t st = smem_base + stage * STAGE_BYTES;
            ab::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / UMMA_K; ++k)
                ab::wgmma_m64n256k16_ss<kBF16, 0, 0>(acc, ab::wgmma_desc_sw128(st + wg * 8192u + k * 32u),
                                                     ab::wgmma_desc_sw128(st + A_BYTES + k * 32u), 1);
            ab::wgmma_commit();
            // the previous tile's TMA store has had this tile's first k-block to read the staging buffer: wait for it
            // here, under the MMAs just issued, and hand the buffer to the residual load
            if (kb == 0 && i > 0 && ctid == 0) {
                ab::tma_store_wait_read();
                if constexpr (kEpi == EPI_RESIDUAL) ab::mbar_arrive(&res_empty[wg]);
            }
            // the previous stage's MMAs have retired once at most this stage's group is pending: release it
            ab::wgmma_wait<1>();
            ab::wgmma_reg_fence(acc);
            if (prev_stage >= 0 && ctid == 0) ab::mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = static_cast<int>(stage);
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1u;
            }
        }
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(acc);
        if (prev_stage >= 0 && ctid == 0) ab::mbar_arrive(&empty_bar[prev_stage]);

        // ---- epilogue into the staging buffer: rows 16 wl + lane / 4 (+ 8) of the slice, column pairs 8 j + 2 (lane % 4)
        if constexpr (kEpi == EPI_RESIDUAL) ab::mbar_wait_nocall(&res_full[wg], static_cast<uint32_t>(i & 1));
        else if (i > 0) ab::named_bar_sync(EPI_BAR + wg, 128);    // the previous store has read the buffer
        const int row0 = m_blk * BLOCK_M + static_cast<int>(wg) * 64;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = static_cast<int>(wl * 16u + (lane >> 2)) + 8 * h;                   // row in the slice
            const int row = row0 + r;
            const bool row_ok = row < p.M;
            const float rscale = row_scale(p, row, row_ok);
            // out_ss: one partial sum per 128 columns, the same sums in the same order as the 128 x 128 schedules
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                float ss_out = 0.f;
#pragma unroll
                for (int j = 16 * half; j < 16 * half + 16; ++j) {
                    const int c = 8 * j + cq;                                                  // column in the tile
                    const int col = n_blk * BLOCK_N + c;
                    if (col >= p.N) continue;                  // past the edge: the TMA store clips it
                    uint8_t* dst = buf + (c >> 6) * BOX_BYTES + sw128_offset(r, c & 63);
                    const uint32_t res = kEpi == EPI_RESIDUAL ? *reinterpret_cast<const uint32_t*>(dst) : 0u;
                    const uint32_t o = epilogue_pair<kBF16, kEpi>(p, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], rscale,
                                                                  col, res);
                    if constexpr (kEpi == EPI_GATED) {
                        const int co = c >> 1;
                        *reinterpret_cast<uint16_t*>(buf + (co >> 6) * BOX_BYTES + sw128_offset(r, co & 63)) =
                            static_cast<uint16_t>(o & 0xFFFFu);
                    } else {
                        *reinterpret_cast<uint32_t*>(dst) = o;
                        if (p.out_ss != nullptr) ss_out = add_sq_pair<kBF16>(o, ss_out);
                    }
                }
                if (kEpi != EPI_GATED && p.out_ss != nullptr) out_ss_add(p, row, row_ok, lane, ss_out);
            }
        }
        ab::fence_proxy_async_smem();                  // generic-proxy writes -> visible to the TMA store
        ab::named_bar_sync(EPI_BAR + wg, 128);
        if (ctid == 0) {
            // boxes wholly past the edge of C are not stored (the tensor map clips the rest)
            const int c0 = n_blk * (BLOCK_N / (kEpi == EPI_GATED ? 2 : 1));
            if (row0 < p.M)
                for (int b = 0; b < OUT_BOXES && c0 + 64 * b < n_out; ++b)
                    ab::tma_store_2d(&tmap_c, buf + b * BOX_BYTES, c0 + 64 * b, row0);
            ab::tma_store_commit();
        }
    }
    if (ctid == 0) ab::tma_store_wait_all();
}

template <bool kBF16, int BLOCK_N, bool kTN, int kEpi>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const Params& p, cudaStream_t s) {
    using C = Cfg<BLOCK_N>;
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(gemm_kernel<kBF16, BLOCK_N, kTN, kEpi>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           C::SMEM_BYTES));
        attr_set = true;
    }
    const int tiles = ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N) * p.splits;
    const int grid = tiles < abh::num_sms() ? tiles : abh::num_sms();
    abh::prof_begin(s, abh::PROF_LINEAR);
    gemm_kernel<kBF16, BLOCK_N, kTN, kEpi><<<grid, THREADS, C::SMEM_BYTES, s>>>(ta, tb, p);
    if (p.m_dev != nullptr) abh::prof_end_dyn(s, abh::PROF_LINEAR, 2.0 * static_cast<double>(p.N) * p.K, p.m_dev, p.M);
    else abh::prof_end(s, abh::PROF_LINEAR, 2.0 * p.M * static_cast<double>(p.N) * p.K);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

// K-major launch of one epilogue: 16-bit type and tile width chosen at run time
template <int kEpi>
static int launch_n(bool bf16, bool wide, const CUtensorMap& ta, const CUtensorMap& tb, const Params& p, cudaStream_t s) {
    if (bf16) return wide ? launch<true, 256, false, kEpi>(ta, tb, p, s) : launch<true, 128, false, kEpi>(ta, tb, p, s);
    return wide ? launch<false, 256, false, kEpi>(ta, tb, p, s) : launch<false, 128, false, kEpi>(ta, tb, p, s);
}

template <bool kBF16, int kEpi>
static int launch_pp(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& tr, const Params& p,
                     cudaStream_t s) {
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(gemm_pp_kernel<kBF16, kEpi>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           pp::SMEM_BYTES));
        attr_set = true;
    }
    const int tiles = ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + pp::BLOCK_N - 1) / pp::BLOCK_N);
    const int grid = tiles < abh::num_sms() ? tiles : abh::num_sms();
    abh::prof_begin(s, abh::PROF_LINEAR);
    gemm_pp_kernel<kBF16, kEpi><<<grid, THREADS, pp::SMEM_BYTES, s>>>(ta, tb, tc, tr, p);
    if (p.m_dev != nullptr) abh::prof_end_dyn(s, abh::PROF_LINEAR, 2.0 * static_cast<double>(p.N) * p.K, p.m_dev, p.M);
    else abh::prof_end(s, abh::PROF_LINEAR, 2.0 * p.M * static_cast<double>(p.N) * p.K);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

template <int kEpi>
static int launch_pp_t(bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& tr,
                       const Params& p, cudaStream_t s) {
    return bf16 ? launch_pp<true, kEpi>(ta, tb, tc, tr, p, s) : launch_pp<false, kEpi>(ta, tb, tc, tr, p, s);
}

template <bool kBF16, int kEpi>
static int launch_wide(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& tr,
                       const Params& p, cudaStream_t s) {
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(gemm_wide_kernel<kBF16, kEpi>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           wd::SMEM_BYTES));
        attr_set = true;
    }
    const int tiles = ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + wd::BLOCK_N - 1) / wd::BLOCK_N);
    const int grid = tiles < abh::num_sms() ? tiles : abh::num_sms();
    abh::prof_begin(s, abh::PROF_LINEAR);
    gemm_wide_kernel<kBF16, kEpi><<<grid, THREADS, wd::SMEM_BYTES, s>>>(ta, tb, tc, tr, p);
    if (p.m_dev != nullptr) abh::prof_end_dyn(s, abh::PROF_LINEAR, 2.0 * static_cast<double>(p.N) * p.K, p.m_dev, p.M);
    else abh::prof_end(s, abh::PROF_LINEAR, 2.0 * p.M * static_cast<double>(p.N) * p.K);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

template <int kEpi>
static int launch_wide_t(bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& tr,
                         const Params& p, cudaStream_t s) {
    return bf16 ? launch_wide<true, kEpi>(ta, tb, tc, tr, p, s) : launch_wide<false, kEpi>(ta, tb, tc, tr, p, s);
}

// The schedule of a K-major launch (values of atlas_b200_linear_schedule).  res_aligned: EPI_RESIDUAL's residual base is
// 16-byte aligned, which the TMA-staged schedules need for its tensor map.  Measured at the bench's encoder sizes (77,696
// packed rows, H100 SXM 80 GB at 700 W, tools/prof_ops.py gemm_sched; wide vs ping-pong, two runs each):
//   plain      q|k|v N 2304 K 768   401 vs 472-480 us    cross K|V N 1536   286-293 vs 344-376 us
//              mainloop N 2304 K 4096 (M 61,440)   1675-1682 vs 2160-2218 us                       -> wide
//   residual   o-proj N 768 K 768   262 vs 226-230 us    wo N 768 K 2048 + out_ss   490-495 vs 427-434 us -> ping-pong
//   gated      N 4096 K 768         891-893 vs 875-901 us                                           -> ping-pong
//   bias       N 2304 K 768         624-676 vs 626-632 us                                           -> ping-pong
//   GELU       N 3072 K 768         1023-1034 vs 978-1022 us                                        -> ping-pong
//   ReLU       N 3072 K 768         860-871 vs 865-891 us                                           -> ping-pong
// A fused epilogue is as fast or faster on ping-pong, which hides it under the other consumer's MMAs; wide only wins where
// the epilogue is a plain store.  Wide also needs the 256-wide tiles to pad no more columns than 128-wide ones
// (N % 256 == 0 or > 128).
// ATLAS_B200_GEMM_SCHEDULE=pingpong|wide overrides the choice between the two for every launch that may run either (for
// timing them against each other on the same shapes: tools/prof_ops.py gemm_sched).
static int select_schedule(int64_t M, int64_t N, int64_t K, int epilogue, bool res_aligned) {
    (void)K;
    static const char* force = getenv("ATLAS_B200_GEMM_SCHEDULE");
    const int64_t tiles128 = ((M + 127) / 128) * ((N + 127) / 128);
    if (tiles128 >= 2 * abh::num_sms() && (epilogue != EPI_RESIDUAL || res_aligned)) {
        if (force != nullptr && strcmp(force, "pingpong") == 0) return ATLAS_B200_GEMM_PINGPONG;
        if (force != nullptr && strcmp(force, "wide") == 0) return ATLAS_B200_GEMM_WIDE;
        return epilogue == EPI_NONE && (N + 255) / 256 * 2 == (N + 127) / 128 ? ATLAS_B200_GEMM_WIDE : ATLAS_B200_GEMM_PINGPONG;
    }
    if (N >= 256 && ((M + 127) / 128) * ((N + 255) / 256) >= abh::num_sms()) return ATLAS_B200_GEMM_COOPERATIVE_256;
    return ATLAS_B200_GEMM_COOPERATIVE_128;
}

// out[i] = round16(sum_s part[s][i]) for the M*N outputs of a split-K GEMM (8 outputs per thread)
template <bool kBF16>
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ part, uint16_t* __restrict__ out, int64_t ldc, int M, int N, int splits) {
    const int64_t vecs = static_cast<int64_t>(M) * (N / 8);
    for (int64_t idx = blockIdx.x * 256ll + threadIdx.x; idx < vecs; idx += gridDim.x * 256ll) {
        const int64_t row = idx / (N / 8);
        const int col = static_cast<int>(idx % (N / 8)) * 8;
        float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int sidx = 0; sidx < splits; ++sidx) {
            const float4* src = reinterpret_cast<const float4*>(part + (static_cast<size_t>(sidx) * M + row) * N + col);
            const float4 x = __ldg(src), y = __ldg(src + 1);
            a[0] += x.x; a[1] += x.y; a[2] += x.z; a[3] += x.w;
            a[4] += y.x; a[5] += y.y; a[6] += y.z; a[7] += y.w;
        }
        *reinterpret_cast<uint4*>(out + row * ldc + col) =
            make_uint4(pack2<kBF16>(a[0], a[1]), pack2<kBF16>(a[2], a[3]), pack2<kBF16>(a[4], a[5]), pack2<kBF16>(a[6], a[7]));
    }
}

}  // namespace gemm

extern "C" {

int atlas_b200_linear_rows(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, const void* residual,
                           int64_t ldr, void* C, int64_t ldc, int32_t M, int32_t N, int32_t K, int32_t epilogue,
                           int32_t is_bf16, const float* row_ss, float* out_ss, float rs_eps, const int32_t* m_dev, void* stream) {
    using namespace gemm;
    AB_REQUIRE(M >= 0 && N > 0 && K > 0, "bad GEMM shape M=%d N=%d K=%d", M, N, K);
    if (M == 0) return ATLAS_B200_OK;
    AB_REQUIRE(N % 8 == 0 && K % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0 && ldc % 8 == 0,
               "N, K and the leading dimensions must be multiples of 8 (16-byte rows)");
    AB_REQUIRE(epilogue >= EPI_NONE && epilogue <= EPI_RELU, "unknown epilogue %d", epilogue);
    AB_REQUIRE(epilogue != EPI_RESIDUAL || (residual != nullptr && ldr % 8 == 0), "EPI_RESIDUAL needs a residual");
    // epilogue_pair reads the bias, and the cooperative epilogue the residual, as 32-bit pairs of 16-bit values
    AB_REQUIRE(bias == nullptr || epilogue == EPI_NONE || epilogue == EPI_GATED || (reinterpret_cast<uintptr_t>(bias) & 3u) == 0,
               "the bias must be 4-byte aligned");
    AB_REQUIRE(epilogue != EPI_RESIDUAL || (reinterpret_cast<uintptr_t>(residual) & 3u) == 0,
               "the residual must be 4-byte aligned");
    AB_REQUIRE(epilogue != EPI_GATED || N % 32 == 0, "EPI_GATED needs N %% 32 == 0");
    AB_REQUIRE((reinterpret_cast<uintptr_t>(C) & 15u) == 0, "C must be 16-byte aligned");
    AB_REQUIRE(out_ss == nullptr || epilogue != EPI_GATED, "out_ss is not available with the gated epilogue");
    Params p;
    p.splits = 1;
    p.kb_per_split = (K + BLOCK_K - 1) / BLOCK_K;
    p.C32 = nullptr;
    p.l2_prefetch = 1;
    p.m_dev = m_dev;
    p.row_ss = row_ss;
    p.out_ss = out_ss;
    p.rs_eps = rs_eps;
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = static_cast<int>(ldc);
    p.ldr = static_cast<int>(ldr);
    p.bias = static_cast<const uint16_t*>(bias);
    p.residual = static_cast<const uint16_t*>(residual);
    p.C = static_cast<uint16_t*>(C);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int sched = select_schedule(M, N, K, epilogue, (reinterpret_cast<uintptr_t>(residual) & 15u) == 0);
    const bool pingpong = sched == ATLAS_B200_GEMM_PINGPONG;
    const bool wide = sched == ATLAS_B200_GEMM_COOPERATIVE_256;
    const int block_n = (wide || sched == ATLAS_B200_GEMM_WIDE) ? 256 : 128;
    CUtensorMap ta, tb;
    int rc = abh::make_tmap_2d_16bit(&ta, A, static_cast<uint64_t>(M), static_cast<uint64_t>(K),
                                     static_cast<uint64_t>(lda), BLOCK_M, BLOCK_K, is_bf16 != 0);
    if (rc) return rc;
    rc = abh::make_tmap_2d_16bit(&tb, W, static_cast<uint64_t>(N), static_cast<uint64_t>(K), static_cast<uint64_t>(ldw),
                                 static_cast<uint32_t>(block_n), BLOCK_K, is_bf16 != 0);
    if (rc) return rc;
    if (pingpong || sched == ATLAS_B200_GEMM_WIDE) {
        // C (N / 2 columns for EPI_GATED) and the residual in boxes of 64 columns: 128 rows (ping-pong: a whole tile per
        // consumer) or 64 rows (wide: a consumer's slice of the tile)
        CUtensorMap tc, tr;
        const uint64_t n_out = static_cast<uint64_t>(epilogue == EPI_GATED ? N / 2 : N);
        const uint32_t box_rows = pingpong ? BLOCK_M : 64;
        rc = abh::make_tmap_2d_16bit(&tc, C, static_cast<uint64_t>(M), n_out, static_cast<uint64_t>(ldc), box_rows, 64,
                                     is_bf16 != 0);
        if (rc) return rc;
        if (epilogue == EPI_RESIDUAL) {
            rc = abh::make_tmap_2d_16bit(&tr, residual, static_cast<uint64_t>(M), static_cast<uint64_t>(N),
                                         static_cast<uint64_t>(ldr), box_rows, 64, is_bf16 != 0);
            if (rc) return rc;
        } else {
            tr = tc;                                   // unused
        }
        if (!pingpong) {
            switch (epilogue) {
                case EPI_NONE: return launch_wide_t<EPI_NONE>(is_bf16 != 0, ta, tb, tc, tr, p, s);
                case EPI_BIAS: return launch_wide_t<EPI_BIAS>(is_bf16 != 0, ta, tb, tc, tr, p, s);
                case EPI_GELU: return launch_wide_t<EPI_GELU>(is_bf16 != 0, ta, tb, tc, tr, p, s);
                case EPI_RESIDUAL: return launch_wide_t<EPI_RESIDUAL>(is_bf16 != 0, ta, tb, tc, tr, p, s);
                case EPI_RELU: return launch_wide_t<EPI_RELU>(is_bf16 != 0, ta, tb, tc, tr, p, s);
                default: return launch_wide_t<EPI_GATED>(is_bf16 != 0, ta, tb, tc, tr, p, s);
            }
        }
        switch (epilogue) {
            case EPI_NONE: return launch_pp_t<EPI_NONE>(is_bf16 != 0, ta, tb, tc, tr, p, s);
            case EPI_BIAS: return launch_pp_t<EPI_BIAS>(is_bf16 != 0, ta, tb, tc, tr, p, s);
            case EPI_GELU: return launch_pp_t<EPI_GELU>(is_bf16 != 0, ta, tb, tc, tr, p, s);
            case EPI_RESIDUAL: return launch_pp_t<EPI_RESIDUAL>(is_bf16 != 0, ta, tb, tc, tr, p, s);
            case EPI_RELU: return launch_pp_t<EPI_RELU>(is_bf16 != 0, ta, tb, tc, tr, p, s);
            default: return launch_pp_t<EPI_GATED>(is_bf16 != 0, ta, tb, tc, tr, p, s);
        }
    }
    switch (epilogue) {
        case EPI_NONE: return launch_n<EPI_NONE>(is_bf16 != 0, wide, ta, tb, p, s);
        case EPI_BIAS: return launch_n<EPI_BIAS>(is_bf16 != 0, wide, ta, tb, p, s);
        case EPI_GELU: return launch_n<EPI_GELU>(is_bf16 != 0, wide, ta, tb, p, s);
        case EPI_RESIDUAL: return launch_n<EPI_RESIDUAL>(is_bf16 != 0, wide, ta, tb, p, s);
        case EPI_RELU: return launch_n<EPI_RELU>(is_bf16 != 0, wide, ta, tb, p, s);
        default: return launch_n<EPI_GATED>(is_bf16 != 0, wide, ta, tb, p, s);
    }
}

int atlas_b200_linear_schedule(int32_t M, int32_t N, int32_t K, int32_t epilogue) {
    return gemm::select_schedule(M, N, K, epilogue, true);
}

// (tile shape, number of K splits) of a weight-gradient GEMM: minimise the number of waves of work items per split
static void wgrad_plan(int32_t tokens, int32_t N, int32_t K, int* block_n, int* splits, int* kb_per_split) {
    using namespace gemm;
    *block_n = K >= 256 ? 256 : 128;
    const int64_t tiles = static_cast<int64_t>((N + BLOCK_M - 1) / BLOCK_M) * ((K + *block_n - 1) / *block_n);
    const int groups = abh::num_sms();
    const int num_kb = (tokens + BLOCK_K - 1) / BLOCK_K;
    int best = 1;
    double best_t = 1e30;
    for (int sp = 1; sp <= 16 && sp * 8 <= num_kb; ++sp) {     // every split keeps >= 8 k-blocks (512 tokens)
        const int64_t waves = (tiles * sp + groups - 1) / groups;
        const double t = static_cast<double>(waves) / sp + 0.02 * sp;   // + the partial-tile store / reduce cost
        if (t < best_t - 1e-9) {
            best_t = t;
            best = sp;
        }
    }
    const int per = (num_kb + best - 1) / best;
    *kb_per_split = per > 0 ? per : 1;
    *splits = num_kb > 0 ? (num_kb + *kb_per_split - 1) / *kb_per_split : 1;   // no empty split
}

size_t atlas_b200_linear_wgrad_workspace_bytes(int32_t tokens, int32_t N, int32_t K) {
    int block_n, splits, per;
    wgrad_plan(tokens, N, K, &block_n, &splits, &per);
    return splits > 1 ? static_cast<size_t>(splits) * N * K * sizeof(float) : 0;
}

int atlas_b200_linear_wgrad(const void* dY, int64_t lddy, const void* X, int64_t ldx, void* dW, int64_t lddw, int32_t tokens,
                            int32_t N, int32_t K, int32_t is_bf16, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace gemm;
    AB_REQUIRE(tokens >= 0 && N > 0 && K > 0, "bad wgrad shape tokens=%d N=%d K=%d", tokens, N, K);
    AB_REQUIRE(N % 8 == 0 && K % 8 == 0 && lddy % 8 == 0 && ldx % 8 == 0 && lddw % 8 == 0,
               "wgrad: N, K and the leading dimensions must be multiples of 8 (16-byte rows)");
    AB_REQUIRE((reinterpret_cast<uintptr_t>(dW) & 15u) == 0, "dW must be 16-byte aligned");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (tokens == 0) {
        AB_CUDA_CHECK(cudaMemset2DAsync(dW, static_cast<size_t>(lddw) * 2, 0, static_cast<size_t>(K) * 2, N, s));
        return ATLAS_B200_OK;
    }
    Params p;
    p.l2_prefetch = 0;
    p.m_dev = nullptr;
    p.row_ss = nullptr;
    p.out_ss = nullptr;
    p.rs_eps = 0.f;
    p.M = N;            // output rows  = out_features
    p.N = K;            // output cols  = in_features
    p.K = tokens;       // contraction  = tokens
    p.ldc = static_cast<int>(lddw);
    p.ldr = 0;
    p.bias = nullptr;
    p.residual = nullptr;
    p.C = static_cast<uint16_t*>(dW);
    int block_n, splits, per;
    wgrad_plan(tokens, N, K, &block_n, &splits, &per);
    const bool wide = block_n == 256;
    const size_t need = static_cast<size_t>(splits) * N * K * sizeof(float);
    if (splits > 1 && (workspace == nullptr || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15u) != 0)) {
        splits = 1;                                      // no (usable) scratch: one CTA group walks the whole contraction
        per = (tokens + BLOCK_K - 1) / BLOCK_K;
    }
    p.splits = splits;
    p.kb_per_split = per;
    p.C32 = splits > 1 ? static_cast<float*>(workspace) : nullptr;
    CUtensorMap ta, tb;
    // both maps: rows = tokens, box = {64 columns, 64 tokens}
    int rc = abh::make_tmap_2d_16bit(&ta, dY, static_cast<uint64_t>(tokens), static_cast<uint64_t>(N),
                                     static_cast<uint64_t>(lddy), BLOCK_K, 64, is_bf16 != 0);
    if (rc) return rc;
    rc = abh::make_tmap_2d_16bit(&tb, X, static_cast<uint64_t>(tokens), static_cast<uint64_t>(K), static_cast<uint64_t>(ldx),
                                 BLOCK_K, 64, is_bf16 != 0);
    if (rc) return rc;
    if (is_bf16) rc = wide ? launch<true, 256, true, EPI_NONE>(ta, tb, p, s) : launch<true, 128, true, EPI_NONE>(ta, tb, p, s);
    else rc = wide ? launch<false, 256, true, EPI_NONE>(ta, tb, p, s) : launch<false, 128, true, EPI_NONE>(ta, tb, p, s);
    if (rc || splits == 1) return rc;
    const int64_t vecs = static_cast<int64_t>(N) * (K / 8);
    const int64_t blocks = (vecs + 255) / 256, cap = static_cast<int64_t>(abh::num_sms()) * 8;
    const int grid = static_cast<int>(blocks < cap ? blocks : cap);
    if (is_bf16) splitk_reduce_kernel<true><<<grid, 256, 0, s>>>(p.C32, p.C, p.ldc, N, K, splits);
    else splitk_reduce_kernel<false><<<grid, 256, 0, s>>>(p.C32, p.C, p.ldc, N, K, splits);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
