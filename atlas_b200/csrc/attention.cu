// Fused multi-head attention (head_dim 64, <= 576 keys per segment) on Hopper warpgroup MMAs for the Contriever and FiD
// encoders and the FiD decoder's self- and cross-attention:
//     O[b, i, h, :] = softmax_j( scale * Q[b,i,h,:].K[b,j,h,:] + rel_bias[h, j-i] + key_mask[b, j] (+ causal) ) V[b, j, h, :]
// Replaces, per layer, two batched cuBLAS GEMMs + the materialised [B, H, L, L] score / probability tensors +
// the ATen softmax / mask / bias kernels of
//     BertSelfAttention.forward  src/modeling_bert.py:328-366   (scale 1/8, additive key mask, fp32 softmax)
//     T5Attention.forward        src/modeling_t5.py:478-524      (no scaling, relative-position bias + mask
//                                                                 added to the scores, fp32 softmax)
// Q, K, V are read IN PLACE from the fused projection output ([tokens, n_cols] row-major, head h at a column offset)
// through TMA boxes of {64 columns, 64 rows} with the 128-byte swizzle; nothing is transposed or re-laid-out:
//   S = Q K^T : wgmma m64n64k16, A = Q rows (K-major), B = K rows (K-major)          -> fp32 S in registers
//   O += P V  : wgmma m64n64k16, A = P from REGISTERS (the S fragment rounded to 16 bits),
//               B = V rows as they lie in memory = MN-major operand (transpose flag)
// One CTA = one (segment, head, 128-row query tile): the segment's K and V (<= 576 keys, 72 KB each) and the query tile land in
// shared memory through one mbarrier; two warpgroups own 64 query rows each and sweep the 64-key blocks with an online
// (flash-attention) softmax in the log2 domain.  Key blocks whose keys are all masked out (key_block_live) are skipped: their
// probabilities are exactly 0 in fp32.
//
// Segments of 577 to 4096 keys (the FiD encoder on long passages) run on attention_long_kernel below: the same per-block
// arithmetic, with K and V streamed through a ring of shared-memory slots instead of held resident.  Its per-block code
// (attend_block) is a copy of attention_kernel's loop body rather than shared with it: calling one inlined function from both
// kernels changes how ptxas allocates attention_kernel (124 -> 122 registers, different SASS), so attention_kernel keeps
// its own loop and stays instruction-for-instruction what it was.
//
// The padding-compacted encoders (segment b keeps the first n_b of its 64-row tiles, stored back to back) run on
// attention_packed_kernel below: a persistent kernel over (segment, head) items with the same per-block arithmetic.
#include "common.cuh"
#include "dropout.cuh"
#include "host_common.h"
#include "wgmma.cuh"

#include <algorithm>
#include <math.h>
#include <stdlib.h>

namespace attn {

constexpr int D = 64;            // head dim
constexpr int BQ = 128;          // query rows per CTA (two warpgroups x 64)
constexpr int BK = 64;           // keys per block
constexpr int MAX_BLOCKS = 9;
constexpr int MAX_LK = MAX_BLOCKS * BK;        // 576
constexpr int THREADS = 256;
constexpr int TILE_BYTES = BK * D * 2;         // 8 KB: 64 rows x 128 bytes
constexpr int Q_BYTES = BQ * D * 2;
constexpr int KV_BYTES = MAX_LK * D * 2;
constexpr int SMEM_BYTES = 1024 + Q_BYTES + 2 * KV_BYTES;
constexpr float LOG2E = 1.4426950408889634f;

struct Params {
    int B, H, Lq, Lk;
    int q_col0, k_col0, v_col0;  // column of head 0 in the Q / K / V row buffers
    uint16_t* O;
    int64_t ldo;
    const float* add_mask;    // [B, Lk] additive key mask (0 or -10000 / -1e9 ...) or nullptr
    const float* bias_delta;  // [H, Lq + Lk - 1]: bias for (j - i) + (Lq - 1), or nullptr
    float scale;
    float causal_value;       // 0 = not causal; otherwise the additive value for j > i (reference: -10000)
    // split-KV (decoder cross-attention over n_ctx*L keys): segment b reads the queries of batch b / q_div and
    // writes UN-normalised fp32 partial outputs + (row max, row sum) for combine_splits_kernel
    int q_div;
    float* o_partial;         // [B*Lq, H*64] fp32 or nullptr
    float* ml_partial;        // [B*Lq, H, 2] fp32
    float* lse_out;           // [B, H, Lq] fp32 row log-sum-exp (natural log) for the backward pass, or nullptr
    abdrop::Key drop;         // attention-probability dropout (training path); thr16 == 0: off
    const uint8_t* blk_live;  // [B, ceil(Lk / 64)] or nullptr: 0 = every key of the block is masked out
    int n_qt;                 // query tiles per segment (grid.x)
};

template <bool kBF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    return ab::pack2_rn<kBF16>(a, b);
}

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// attention_long_kernel's step over one live 64-key block kb, the loop body of attention_kernel (see the header): for this
// thread's query rows i0 and i0 + 8 (warpgroup g of the 128-row tile at sQ; the block's K and V in slot `slot` of sK / sV),
// S = Q K^T, t = S * scale2 + mask + bias in the log2 domain, the online-softmax update of (m_run, l_run, o) and O += P V
// with P from registers.  s_mask is indexed by key, s_bias by key - min(i, Lq - 1) + bias_off.
template <bool kBF16>
__device__ __forceinline__ void attend_block(float (&o)[32], float (&m_run)[2], float (&l_run)[2], const uint32_t sQ,
                                             const uint32_t g, const uint32_t sK, const uint32_t sV, const int slot,
                                             const float* s_mask, const float* s_bias,
                                             const int bias_off, const bool has_bias, const int kb, const int i0, const int cq,
                                             const float scale2, const bool dropping, const Params& p, const int b, const int h,
                                             const uint32_t lane) {
    float sc[32];
    ab::wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
        const uint64_t adesc = ab::wgmma_desc_sw128(sQ + g * 8192u + k * 32u);
        const uint64_t bdesc = ab::wgmma_desc_sw128(sK + slot * TILE_BYTES + k * 32u);
        ab::wgmma_m64n64k16_ss<kBF16, 0, 0>(sc, adesc, bdesc, k);
    }
    ab::wgmma_commit();
    ab::wgmma_wait<0>();
    ab::wgmma_reg_fence(sc);

    // t = S * scale2 + (mask + bias) in the log2 domain; new row maxima
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int key = kb * BK + 8 * j + cq + c;
            const float mk = s_mask[key];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float a = mk;
                if (has_bias) a += s_bias[key - min(i0 + 8 * hh, p.Lq - 1) + bias_off];   // rows past Lq are not stored
                const float t = fmaf(sc[4 * j + 2 * hh + c], scale2, a);
                sc[4 * j + 2 * hh + c] = t;
                mx[hh] = fmaxf(mx[hh], t);
            }
        }
    }
    float corr[2], base[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
        base[hh] = mx[hh] == -INFINITY ? 0.f : mx[hh];
        corr[hh] = ex2_approx(m_run[hh] - base[hh]);     // 0 for the first block (m_run = -inf)
        m_run[hh] = mx[hh];
        l_run[hh] *= corr[hh];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        o[4 * j] *= corr[0];
        o[4 * j + 1] *= corr[0];
        o[4 * j + 2] *= corr[1];
        o[4 * j + 3] *= corr[1];
    }
    // p = 2^(t - m); the row sum takes every probability, the P operand only the kept ones (dropout)
    uint32_t pa[16];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        uint32_t w[2][4];
        if (dropping) {
            const uint64_t R = (static_cast<uint64_t>(b / p.q_div) * p.H + h) * p.Lq + min(i0 + 8 * hh, p.Lq - 1);
#pragma unroll
            for (int gg = 0; gg < 2; ++gg) {
                const uint32_t G = static_cast<uint32_t>(((b % p.q_div) * p.Lk + kb * BK + gg * 32) >> 5);
                abdrop::attn_words(p.drop, R, G, static_cast<uint32_t>(lane & 3u), w[gg]);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float e0 = ex2_approx(sc[4 * j + 2 * hh] - base[hh]);
            const float e1 = ex2_approx(sc[4 * j + 2 * hh + 1] - base[hh]);
            l_run[hh] += e0 + e1;
            float k0 = e0, k1 = e1;
            if (dropping) {
                const uint32_t word = w[j >> 2][j & 3];
                k0 = abdrop::keep_lo(p.drop, word) ? e0 : 0.f;
                k1 = abdrop::keep_hi(p.drop, word) ? e1 : 0.f;
            }
            // A fragment of k16 step j / 2: a0 = (r, keys 0-7), a1 = (r + 8, keys 0-7), a2 / a3 = keys 8-15
            pa[4 * (j >> 1) + 2 * (j & 1) + hh] = pack2<kBF16>(k0, k1);
        }
    }
    ab::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
        const uint32_t a[4] = {pa[4 * k], pa[4 * k + 1], pa[4 * k + 2], pa[4 * k + 3]};
        const uint64_t bdesc = ab::wgmma_desc_sw128(sV + slot * TILE_BYTES + k * 2048u, 8192);
        ab::wgmma_m64n64k16_rs<kBF16, 1>(o, a, bdesc, 1);
    }
    ab::wgmma_commit();
    ab::wgmma_wait<0>();
    ab::wgmma_reg_fence(o);
}

// grid = (query tiles, H, B)
template <bool kBF16>
__global__ void __launch_bounds__(THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const Params p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t load_bar;
    __shared__ float s_mask[MAX_LK];                 // key mask * log2e, -inf past Lk
    __shared__ float s_bias[2 * MAX_LK + BK];        // (bias by (j - i) + (Lq - 1) [+ causal]) * log2e
    __shared__ uint32_t s_live;

    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));
    const uint32_t sQ = smem_base, sK = smem_base + Q_BYTES, sV = sK + KV_BYTES;

    const int nkb = (p.Lk + BK - 1) / BK;
    // live key blocks (bit j = block j); none flagged live = all live
    uint32_t live = (1u << nkb) - 1u;
    if (p.blk_live != nullptr) {
        const bool lv = static_cast<int>(lane) < nkb && __ldg(p.blk_live + static_cast<size_t>(b) * nkb + lane) != 0;
        const uint32_t m = __ballot_sync(0xffffffffu, lv);
        if (m != 0u) live = m;
    }
    const int q_row0 = (b / p.q_div) * p.Lq;
    const int k_row0 = b * p.Lk;
    const int o_row0 = b * p.Lq;

    if (threadIdx.x == 0) {
        ab::mbar_init(&load_bar, 1);
        ab::fence_barrier_init();
        s_live = live;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        ab::tma_prefetch_desc(&tmap_q);
        int nload = 0;
        for (int kb = 0; kb < nkb; ++kb) nload += (live >> kb) & 1u;
        ab::mbar_arrive_expect_tx(&load_bar, static_cast<uint32_t>(2 * TILE_BYTES + 2 * nload * TILE_BYTES));
        for (int t = 0; t < 2; ++t)
            ab::tma_load_2d(&tmap_q, &load_bar, smem_gen + t * TILE_BYTES, p.q_col0 + h * D, q_row0 + qt * BQ + t * BK,
                            ab::kEvictFirst);
        for (int kb = 0; kb < nkb; ++kb) {
            if (!((live >> kb) & 1u)) continue;
            ab::tma_load_2d(&tmap_k, &load_bar, smem_gen + Q_BYTES + kb * TILE_BYTES, p.k_col0 + h * D, k_row0 + kb * BK,
                            ab::kEvictNormal);
            ab::tma_load_2d(&tmap_v, &load_bar, smem_gen + Q_BYTES + KV_BYTES + kb * TILE_BYTES, p.v_col0 + h * D,
                            k_row0 + kb * BK, ab::kEvictNormal);
        }
    }
    // mask / bias tables while the loads are in flight
    const bool has_bias = (p.bias_delta != nullptr) || (p.causal_value != 0.f);
    for (int j = threadIdx.x; j < nkb * BK; j += THREADS)
        s_mask[j] = (j < p.Lk) ? (p.add_mask ? p.add_mask[static_cast<size_t>(b) * p.Lk + j] * LOG2E : 0.f) : -INFINITY;
    if (has_bias) {
        const int n_valid = p.Lq + p.Lk - 1;
        for (int d = threadIdx.x; d < 2 * MAX_LK + BK; d += THREADS) {   // entries past the valid offsets stay finite (0)
            float v = 0.f;
            if (d < n_valid) {
                v = p.bias_delta ? p.bias_delta[static_cast<size_t>(h) * n_valid + d] : 0.f;
                if (p.causal_value != 0.f && d > p.Lq - 1) v += p.causal_value;   // j > i
            }
            s_bias[d] = v * LOG2E;
        }
    }
    __syncthreads();
    ab::mbar_wait(&load_bar, 0, 40);

    // ---- warpgroup g: query rows 64 g .. 64 g + 63 of the tile; this thread: rows r and r + 8, key pairs 8 j + 2 (lane % 4)
    const uint32_t g = warp >> 2, wl = warp & 3u;
    const int i0 = qt * BQ + static_cast<int>(g * 64u + wl * 16u + (lane >> 2));   // query index of row r (in the segment)
    const int cq = static_cast<int>(2u * (lane & 3u));
    const float scale2 = p.scale * LOG2E;
    const bool dropping = p.drop.thr16 != 0u;
    float o[32];
#pragma unroll
    for (int x = 0; x < 32; ++x) o[x] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    for (int kb = 0; kb < nkb; ++kb) {
        if (!((live >> kb) & 1u)) continue;
        float sc[32];
        ab::wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; ++k) {
            const uint64_t adesc = ab::wgmma_desc_sw128(sQ + g * 8192u + k * 32u);
            const uint64_t bdesc = ab::wgmma_desc_sw128(sK + kb * TILE_BYTES + k * 32u);
            ab::wgmma_m64n64k16_ss<kBF16, 0, 0>(sc, adesc, bdesc, k);
        }
        ab::wgmma_commit();
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(sc);

        // t = S * scale2 + (mask + bias) in the log2 domain; new row maxima
        float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int key = kb * BK + 8 * j + cq + c;
                const float mk = s_mask[key];
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float a = mk;
                    if (has_bias) a += s_bias[key - min(i0 + 8 * hh, p.Lq - 1) + (p.Lq - 1)];   // rows past Lq are not stored
                    const float t = fmaf(sc[4 * j + 2 * hh + c], scale2, a);
                    sc[4 * j + 2 * hh + c] = t;
                    mx[hh] = fmaxf(mx[hh], t);
                }
            }
        }
        float corr[2], base[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
            base[hh] = mx[hh] == -INFINITY ? 0.f : mx[hh];
            corr[hh] = ex2_approx(m_run[hh] - base[hh]);     // 0 for the first block (m_run = -inf)
            m_run[hh] = mx[hh];
            l_run[hh] *= corr[hh];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[4 * j] *= corr[0];
            o[4 * j + 1] *= corr[0];
            o[4 * j + 2] *= corr[1];
            o[4 * j + 3] *= corr[1];
        }
        // p = 2^(t - m); the row sum takes every probability, the P operand only the kept ones (dropout)
        uint32_t pa[16];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            uint32_t w[2][4];
            if (dropping) {
                const uint64_t R = (static_cast<uint64_t>(b / p.q_div) * p.H + h) * p.Lq + min(i0 + 8 * hh, p.Lq - 1);
#pragma unroll
                for (int gg = 0; gg < 2; ++gg) {
                    const uint32_t G = static_cast<uint32_t>(((b % p.q_div) * p.Lk + kb * BK + gg * 32) >> 5);
                    abdrop::attn_words(p.drop, R, G, static_cast<uint32_t>(lane & 3u), w[gg]);
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float e0 = ex2_approx(sc[4 * j + 2 * hh] - base[hh]);
                const float e1 = ex2_approx(sc[4 * j + 2 * hh + 1] - base[hh]);
                l_run[hh] += e0 + e1;
                float k0 = e0, k1 = e1;
                if (dropping) {
                    const uint32_t word = w[j >> 2][j & 3];
                    k0 = abdrop::keep_lo(p.drop, word) ? e0 : 0.f;
                    k1 = abdrop::keep_hi(p.drop, word) ? e1 : 0.f;
                }
                // A fragment of k16 step j / 2: a0 = (r, keys 0-7), a1 = (r + 8, keys 0-7), a2 / a3 = keys 8-15
                pa[4 * (j >> 1) + 2 * (j & 1) + hh] = pack2<kBF16>(k0, k1);
            }
        }
        ab::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
            const uint32_t a[4] = {pa[4 * k], pa[4 * k + 1], pa[4 * k + 2], pa[4 * k + 3]};
            const uint64_t bdesc = ab::wgmma_desc_sw128(sV + kb * TILE_BYTES + k * 2048u, 8192);
            ab::wgmma_m64n64k16_rs<kBF16, 1>(o, a, bdesc, 1);
        }
        ab::wgmma_commit();
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(o);
    }

    // ---- output: full row sums across the quad, then normalised 16-bit rows or split-KV partials
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        float l = l_run[hh];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const int i = i0 + 8 * hh;
        if (i >= p.Lq) continue;
        const size_t orow = static_cast<size_t>(o_row0) + i;
        if (p.o_partial != nullptr) {
            const float ik = p.drop.inv_keep;
            float* dst = p.o_partial + orow * (static_cast<size_t>(p.H) * D) + h * D + cq;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[4 * j + 2 * hh] * ik, o[4 * j + 2 * hh + 1] * ik);
            if ((lane & 3u) == 0u) {
                float* ml = p.ml_partial + (orow * p.H + h) * 2;
                ml[0] = m_run[hh] * (1.0f / LOG2E);
                ml[1] = l;
            }
        } else {
            const float inv = p.drop.inv_keep / l;
            if (p.lse_out != nullptr && (lane & 3u) == 0u)
                p.lse_out[(static_cast<size_t>(b) * p.H + h) * p.Lq + i] = m_run[hh] * (1.0f / LOG2E) + __logf(l);
            uint16_t* dst = p.O + orow * p.ldo + h * D + cq;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2<kBF16>(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
        }
    }
}

// ---- attention_long_kernel: the same contract for Lk up to LONG_MAX_LK keys (no split-KV partials, no packed layout).  K and V
// stream through a LONG_STAGES-deep ring of 64-key tiles: one producer warp issues their TMA loads (full / empty mbarriers),
// the two consumer warpgroups of attention_kernel sweep the live blocks with attend_block.  The CTA's slice of the bias table
// (offsets of its 128 query rows to every key) and the key mask are staged in shared memory once.
constexpr int LONG_MAX_LK = 4096;              // Lq + Lk - 1 <= 8192: the bias table of the backward (attention_bwd.cu)
constexpr int LONG_STAGES = 4;
constexpr int LONG_THREADS = THREADS + 32;     // two consumer warpgroups + one producer warp
constexpr int LONG_BIAS = LONG_MAX_LK + BQ;    // >= (keys rounded up to 64) + 127 offsets
constexpr int LONG_SMEM_BYTES = 1024 + Q_BYTES + 2 * LONG_STAGES * TILE_BYTES + (LONG_MAX_LK + LONG_BIAS) * 4;

// grid = (query tiles, H, B)
template <bool kBF16>
__global__ void __launch_bounds__(LONG_THREADS, 1)
attention_long_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                      const __grid_constant__ CUtensorMap tmap_v, const Params p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t q_bar, full_bar[LONG_STAGES], empty_bar[LONG_STAGES];
    __shared__ uint8_t s_live[LONG_MAX_LK / BK];

    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));
    // Q | K ring | V ring | key mask | bias slice
    const uint32_t sQ = smem_base, sK = smem_base + Q_BYTES, sV = sK + LONG_STAGES * TILE_BYTES;
    float* s_mask = reinterpret_cast<float*>(smem_gen + Q_BYTES + 2 * LONG_STAGES * TILE_BYTES);
    float* s_bias = s_mask + LONG_MAX_LK;

    const int nkb = (p.Lk + BK - 1) / BK;
    const bool producer = warp == THREADS / 32;
    if (threadIdx.x == 0) {
        ab::mbar_init(&q_bar, 1);
        for (int s = 0; s < LONG_STAGES; ++s) {
            ab::mbar_init(&full_bar[s], 1);
            ab::mbar_init(&empty_bar[s], THREADS / 32);     // one arrival per consumer warp
        }
        ab::fence_barrier_init();
    }
    // live key blocks; none flagged live = all live
    bool lv = false;
    if (static_cast<int>(threadIdx.x) < nkb) {
        lv = p.blk_live == nullptr || __ldg(p.blk_live + static_cast<size_t>(b) * nkb + threadIdx.x) != 0;
        s_live[threadIdx.x] = lv;
    }
    const bool all_live = __syncthreads_or(lv) == 0;

    // producer: the query tile, then the live K / V blocks; the first LONG_STAGES go out before the tables are staged
    int next_kb = 0, n_issued = 0;
    auto produce = [&](int max_issued) {
        for (; next_kb < nkb && n_issued < max_issued; ++next_kb) {
            if (!all_live && !s_live[next_kb]) continue;
            const int s = n_issued % LONG_STAGES;
            if (n_issued >= LONG_STAGES) ab::mbar_wait(&empty_bar[s], ((n_issued / LONG_STAGES) & 1) ^ 1, 51);
            ab::mbar_arrive_expect_tx(&full_bar[s], static_cast<uint32_t>(2 * TILE_BYTES));
            const int row = b * p.Lk + next_kb * BK;
            ab::tma_load_2d(&tmap_k, &full_bar[s], smem_gen + Q_BYTES + s * TILE_BYTES, p.k_col0 + h * D, row,
                            ab::kEvictNormal);
            ab::tma_load_2d(&tmap_v, &full_bar[s], smem_gen + Q_BYTES + (LONG_STAGES + s) * TILE_BYTES, p.v_col0 + h * D,
                            row, ab::kEvictNormal);
            ++n_issued;
        }
    };
    if (producer && lane == 0) {
        ab::tma_prefetch_desc(&tmap_q);
        ab::mbar_arrive_expect_tx(&q_bar, static_cast<uint32_t>(2 * TILE_BYTES));
        for (int t = 0; t < 2; ++t)
            ab::tma_load_2d(&tmap_q, &q_bar, smem_gen + t * TILE_BYTES, p.q_col0 + h * D, b * p.Lq + qt * BQ + t * BK,
                            ab::kEvictFirst);
        produce(LONG_STAGES);
    }
    // mask and the bias slice: offsets d_lo .. d_lo + 64 nkb + 126 of the [H, Lq + Lk - 1] table, d_lo = that of the tile's
    // last (clamped) row to key 0; entries past the valid offsets stay finite (0)
    const bool has_bias = (p.bias_delta != nullptr) || (p.causal_value != 0.f);
    for (int j = threadIdx.x; j < nkb * BK; j += LONG_THREADS)
        s_mask[j] = (j < p.Lk) ? (p.add_mask ? p.add_mask[static_cast<size_t>(b) * p.Lk + j] * LOG2E : 0.f) : -INFINITY;
    const int bias_off = min(qt * BQ + BQ - 1, p.Lq - 1);
    if (has_bias) {
        const int n_valid = p.Lq + p.Lk - 1;
        const int d_lo = (p.Lq - 1) - bias_off;
        for (int t = threadIdx.x; t < nkb * BK + BQ - 1; t += LONG_THREADS) {
            const int d = d_lo + t;
            float v = 0.f;
            if (d < n_valid) {
                v = p.bias_delta ? p.bias_delta[static_cast<size_t>(h) * n_valid + d] : 0.f;
                if (p.causal_value != 0.f && d > p.Lq - 1) v += p.causal_value;   // j > i
            }
            s_bias[t] = v * LOG2E;
        }
    }
    __syncthreads();
    if (producer) {
        if (lane == 0) produce(nkb);
        return;
    }
    ab::mbar_wait(&q_bar, 0, 50);

    const uint32_t g = warp >> 2, wl = warp & 3u;
    const int i0 = qt * BQ + static_cast<int>(g * 64u + wl * 16u + (lane >> 2));
    const int cq = static_cast<int>(2u * (lane & 3u));
    const float scale2 = p.scale * LOG2E;
    const bool dropping = p.drop.thr16 != 0u;
    float o[32];
#pragma unroll
    for (int x = 0; x < 32; ++x) o[x] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    int n_used = 0;
    for (int kb = 0; kb < nkb; ++kb) {
        if (!all_live && !s_live[kb]) continue;
        const int s = n_used % LONG_STAGES;
        ab::mbar_wait(&full_bar[s], (n_used / LONG_STAGES) & 1, 52);
        attend_block<kBF16>(o, m_run, l_run, sQ, g, sK, sV, s, s_mask, s_bias, bias_off, has_bias, kb, i0, cq, scale2,
                            dropping, p, b, h, lane);
        __syncwarp();
        if (lane == 0) ab::mbar_arrive(&empty_bar[s]);     // this warp's MMAs on the slot have completed
        ++n_used;
    }

#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        float l = l_run[hh];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const int i = i0 + 8 * hh;
        if (i >= p.Lq) continue;
        const float inv = p.drop.inv_keep / l;
        if (p.lse_out != nullptr && (lane & 3u) == 0u)
            p.lse_out[(static_cast<size_t>(b) * p.H + h) * p.Lq + i] = m_run[hh] * (1.0f / LOG2E) + __logf(l);
        uint16_t* dst = p.O + (static_cast<size_t>(b) * p.Lq + i) * p.ldo + h * D + cq;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2<kBF16>(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
    }
}

// ---- attention_packed_kernel: self-attention over the packed rows of the padding-compacted encoders.  Segment b keeps its
// first n_b = popcount(keep[b, :]) 64-row tiles, stored back to back from row 64 * tile_off[b * nb] of qkv / out; its n_b query
// tiles attend to its n_b key tiles.  Persistent: CTA c owns head h = c % H (its bias row is staged once) and the segments
// c / H, c / H + G, ... (G = grid / H).  One producer warp loads, per (segment, head) item, the item's K and V tiles ONCE into
// one of two item slots (the next item's slot fills while the consumers work on the current one) and the item's 64-row query
// tiles into a ring of PK_Q_STAGES tiles.  The CTA's query tiles are numbered across its items; consumer warpgroup g takes the
// ones with number % 2 == g.  Per key block the arithmetic is attention_kernel's (same blocks, same order, same fp32
// operations), only the issue order differs: S_{j+1} = Q K_{j+1}^T and O += P_j V_j are in flight while the softmax of block
// j + 1 runs.  Shared memory at L = 384: 2 slots x 12 tiles (192 KB) + 3 query tiles (24 KB) + bias row and masks (6 KB).
constexpr int PK_MAX_TILES = 6;                // L <= 384
constexpr int PK_Q_STAGES = 3;
constexpr int PK_THREADS = THREADS + 32;       // two consumer warpgroups + one producer warp

struct PackedParams {
    int S, H, L, G;
    int q_col0, k_col0, v_col0;
    uint16_t* O;
    int64_t ldo;
    const float* add_mask;     // [S, L] or nullptr
    const float* bias_delta;   // [H, 2L - 1] or nullptr
    const uint8_t* keep;       // [S, L / 64]
    const int32_t* tile_off;   // [S * L / 64]
    float scale;
};

static size_t packed_smem_bytes(int L) {
    const int nt = L / BK;
    return 1024 + static_cast<size_t>(2 * 2 * nt + PK_Q_STAGES) * TILE_BYTES + static_cast<size_t>(2 * L + 2 * L) * 4;
}

template <bool kBF16>
__global__ void __launch_bounds__(PK_THREADS, 1)
attention_packed_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                        const __grid_constant__ CUtensorMap tmap_v, const PackedParams p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_kv[2], empty_kv[2], full_q[PK_Q_STAGES], empty_q[PK_Q_STAGES];
    __shared__ int2 s_item[2];                     // per slot: (tiles n, first packed row)

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t smem_base = (ab::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ab::smem_u32(smem_raw));
    const int nt = p.L / BK;
    const uint32_t slot_bytes = 2u * nt * TILE_BYTES;  // K tiles | V tiles
    // K/V slot 0 | K/V slot 1 | query ring | bias row (2L - 1 offsets) | key mask per slot
    const uint32_t sKV = smem_base, sQ = sKV + 2u * slot_bytes;
    float* s_bias = reinterpret_cast<float*>(smem_gen + 2u * slot_bytes + PK_Q_STAGES * TILE_BYTES);
    float* s_mask = s_bias + 2 * p.L;

    const int h = static_cast<int>(blockIdx.x) % p.H;
    const int b0 = static_cast<int>(blockIdx.x) / p.H;
    const int n_items = (p.S - b0 + p.G - 1) / p.G;
    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) {
            ab::mbar_init(&full_kv[s], 32);                 // every producer lane arrives after staging its part of the mask
            ab::mbar_init(&empty_kv[s], THREADS / 32);      // one arrival per consumer warp
        }
        for (int s = 0; s < PK_Q_STAGES; ++s) {
            ab::mbar_init(&full_q[s], 1);
            ab::mbar_init(&empty_q[s], 4);                  // the 4 warps of the consuming warpgroup
        }
        ab::fence_barrier_init();
    }
    const bool has_bias = p.bias_delta != nullptr;
    if (has_bias)
        for (int d = threadIdx.x; d < 2 * p.L - 1; d += PK_THREADS)
            s_bias[d] = p.bias_delta[static_cast<size_t>(h) * (2 * p.L - 1) + d] * LOG2E;
    __syncthreads();

    if (warp == THREADS / 32) {
        // producer: item k's K / V into slot k % 2 once item k - 2 has left it; query tiles in order into the ring.  The two
        // streams wait on different barriers, so neither blocks the other: poll both.
        int kv_k = 0, q_k = 0, q_t = 0, qi = 0;
        if (lane == 0) {
            ab::tma_prefetch_desc(&tmap_q);
            ab::tma_prefetch_desc(&tmap_k);
            ab::tma_prefetch_desc(&tmap_v);
        }
        while (q_k < n_items) {
            bool issued = false;
            if (kv_k < n_items) {
                const int slot = kv_k & 1;
                int ready = kv_k < 2 || ab::mbar_test_wait(&empty_kv[slot], ((kv_k >> 1) & 1) ^ 1);
                ready = __shfl_sync(0xffffffffu, ready, 0);
                if (ready) {
                    const int b = b0 + kv_k * p.G;
                    const bool kp = static_cast<int>(lane) < nt && __ldg(p.keep + static_cast<size_t>(b) * nt + lane) != 0;
                    const uint32_t m = __ballot_sync(0xffffffffu, kp);
                    const int n = m != 0u ? __popc(m) : nt;
                    const int row0 = 64 * __ldg(p.tile_off + static_cast<size_t>(b) * nt);
                    float* mk = s_mask + slot * p.L;
                    for (int j = lane; j < n * BK; j += 32)
                        mk[j] = p.add_mask ? p.add_mask[static_cast<size_t>(b) * p.L + j] * LOG2E : 0.f;
                    if (lane == 0) {
                        s_item[slot] = make_int2(n, row0);
                        ab::mbar_arrive_expect_tx(&full_kv[slot], static_cast<uint32_t>(2 * n * TILE_BYTES));
                        for (int t = 0; t < n; ++t) {
                            ab::tma_load_2d(&tmap_k, &full_kv[slot], smem_gen + slot * slot_bytes + t * TILE_BYTES,
                                            p.k_col0 + h * D, row0 + t * BK, ab::kEvictFirst);
                            ab::tma_load_2d(&tmap_v, &full_kv[slot], smem_gen + slot * slot_bytes + (nt + t) * TILE_BYTES,
                                            p.v_col0 + h * D, row0 + t * BK, ab::kEvictFirst);
                        }
                    } else {
                        ab::mbar_arrive(&full_kv[slot]);
                    }
                    __syncwarp();
                    ++kv_k;
                    issued = true;
                }
            }
            if (q_k < kv_k) {
                const int s = qi % PK_Q_STAGES;
                int ready = qi < PK_Q_STAGES || ab::mbar_test_wait(&empty_q[s], ((qi / PK_Q_STAGES) & 1) ^ 1);
                ready = __shfl_sync(0xffffffffu, ready, 0);
                if (ready) {
                    const int2 it = s_item[q_k & 1];
                    if (lane == 0) {
                        ab::mbar_arrive_expect_tx(&full_q[s], static_cast<uint32_t>(TILE_BYTES));
                        ab::tma_load_2d(&tmap_q, &full_q[s], smem_gen + 2u * slot_bytes + s * TILE_BYTES, p.q_col0 + h * D,
                                        it.y + q_t * BK, ab::kEvictFirst);
                    }
                    ++qi;
                    if (++q_t == it.x) q_t = 0, ++q_k;
                    issued = true;
                }
            }
            if (!issued) __nanosleep(32);
        }
        return;
    }

    // ---- consumers: warpgroup g; this thread: rows r and r + 8 of the 64-row query tile, key pairs 8 j + 2 (lane % 4)
    const uint32_t g = warp >> 2, wl = warp & 3u;
    const int cq = static_cast<int>(2u * (lane & 3u));
    const float scale2 = p.scale * LOG2E;
    int q0 = 0;                                            // number of the item's first query tile
    for (int k = 0; k < n_items; ++k) {
        const int slot = k & 1;
        ab::mbar_wait_nocall(&full_kv[slot], (k >> 1) & 1);
        const int2 it = s_item[slot];
        const int n = it.x;
        const float* mk = s_mask + slot * p.L;
        const uint32_t sK = sKV + slot * slot_bytes, sV = sK + nt * TILE_BYTES;
        for (int qi = q0 + ((static_cast<int>(g) - q0) & 1); qi < q0 + n; qi += 2) {
            const int s = qi % PK_Q_STAGES;
            const uint32_t sQs = sQ + s * TILE_BYTES;
            const int i0 = (qi - q0) * BK + static_cast<int>(wl * 16u + (lane >> 2));   // segment row of row r
            ab::mbar_wait_nocall(&full_q[s], (qi / PK_Q_STAGES) & 1);

            float o[32], sc[32];
            uint32_t pa[16];
            float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, corr[2];
            auto issue_s = [&](int kb) {
#pragma unroll
                for (int kk = 0; kk < D / 16; ++kk)
                    ab::wgmma_m64n64k16_ss<kBF16, 0, 0>(sc, ab::wgmma_desc_sw128(sQs + kk * 32u),
                                                        ab::wgmma_desc_sw128(sK + kb * TILE_BYTES + kk * 32u), kk);
                ab::wgmma_commit();
            };
            auto issue_pv = [&](int kb) {
#pragma unroll
                for (int kk = 0; kk < BK / 16; ++kk)
                    ab::wgmma_m64n64k16_rs<kBF16, 1>(o, *reinterpret_cast<const uint32_t(*)[4]>(&pa[4 * kk]),
                                                     ab::wgmma_desc_sw128(sV + kb * TILE_BYTES + kk * 2048u, 8192), 1);
                ab::wgmma_commit();
            };
            // block kb's softmax on the completed S in sc: sc <- p = 2^(t - m), (m_run, l_run) updated, corr for o
            auto softmax = [&](int kb) {
                ab::wgmma_reg_fence(sc);
                // t = S * scale2 + (mask + bias) in the log2 domain; new row maxima
                float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int key = kb * BK + 8 * j + cq + c;
                        const float mkv = mk[key];
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            float a = mkv;
                            if (has_bias) a += s_bias[key - (i0 + 8 * hh) + (p.L - 1)];
                            const float t = fmaf(sc[4 * j + 2 * hh + c], scale2, a);
                            sc[4 * j + 2 * hh + c] = t;
                            mx[hh] = fmaxf(mx[hh], t);
                        }
                    }
                }
                float base[2];
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
                    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
                    base[hh] = mx[hh] == -INFINITY ? 0.f : mx[hh];
                    corr[hh] = ex2_approx(m_run[hh] - base[hh]);     // 0 for the first block (m_run = -inf)
                    m_run[hh] = mx[hh];
                    l_run[hh] *= corr[hh];
                }
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float e0 = ex2_approx(sc[4 * j + 2 * hh] - base[hh]);
                        const float e1 = ex2_approx(sc[4 * j + 2 * hh + 1] - base[hh]);
                        l_run[hh] += e0 + e1;
                        sc[4 * j + 2 * hh] = e0;
                        sc[4 * j + 2 * hh + 1] = e1;
                    }
                }
            };
            // o *= corr, then P = p rounded to 16 bits as the A fragment of k16 step j / 2: a0 = (r, keys 0-7),
            // a1 = (r + 8, keys 0-7), a2 / a3 = keys 8-15
            auto rescale_and_pack = [&]() {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    o[4 * j] *= corr[0];
                    o[4 * j + 1] *= corr[0];
                    o[4 * j + 2] *= corr[1];
                    o[4 * j + 3] *= corr[1];
                }
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        pa[4 * (j >> 1) + 2 * (j & 1) + hh] = pack2<kBF16>(sc[4 * j + 2 * hh], sc[4 * j + 2 * hh + 1]);
            };

#pragma unroll
            for (int x = 0; x < 32; ++x) o[x] = 0.f;
            ab::wgmma_fence();
            issue_s(0);
            ab::wgmma_wait<0>();
            softmax(0);
            rescale_and_pack();
            for (int kb = 1; kb < n; ++kb) {
                // S_kb and O += P_{kb-1} V_{kb-1} in flight; the softmax of block kb runs under the P V
                ab::wgmma_fence();
                issue_s(kb);
                issue_pv(kb - 1);
                ab::wgmma_wait<1>();
                softmax(kb);
                ab::wgmma_wait<0>();
                ab::wgmma_reg_fence(o);
#pragma unroll
                for (int x = 0; x < 16; ++x) asm volatile("" : "+r"(pa[x])::"memory");   // P_{kb-1} was read until here
                rescale_and_pack();
            }
            ab::wgmma_fence();
            issue_pv(n - 1);
            __syncwarp();
            if (lane == 0) ab::mbar_arrive(&empty_q[s]);     // every S of the query tile is complete
            ab::wgmma_wait<0>();
            ab::wgmma_reg_fence(o);

#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float l = l_run[hh];
                l += __shfl_xor_sync(0xffffffffu, l, 1);
                l += __shfl_xor_sync(0xffffffffu, l, 2);
                const float inv = 1.0f / l;
                uint16_t* dst = p.O + (static_cast<size_t>(it.y) + i0 + 8 * hh) * p.ldo + h * D + cq;
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2<kBF16>(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
            }
        }
        q0 += n;
        __syncwarp();
        if (lane == 0) ab::mbar_arrive(&empty_kv[slot]);     // this warp's MMAs on the slot have completed
    }
}

template <bool kBF16>
static int make_tmaps(CUtensorMap& tq, CUtensorMap& tk, CUtensorMap& tv, const void* q, int64_t ldq, const void* k, int64_t ldk,
                      const void* v, int64_t ldv, int q_rows, int k_rows, const Params& p) {
    int rc = abh::make_tmap_2d_16bit(&tq, q, static_cast<uint64_t>(q_rows), static_cast<uint64_t>(p.q_col0 + p.H * D),
                                     static_cast<uint64_t>(ldq), BK, D, kBF16);
    if (rc) return rc;
    rc = abh::make_tmap_2d_16bit(&tk, k, static_cast<uint64_t>(k_rows), static_cast<uint64_t>(p.k_col0 + p.H * D),
                                 static_cast<uint64_t>(ldk), BK, D, kBF16);
    if (rc) return rc;
    return abh::make_tmap_2d_16bit(&tv, v, static_cast<uint64_t>(k_rows), static_cast<uint64_t>(p.v_col0 + p.H * D),
                                   static_cast<uint64_t>(ldv), BK, D, kBF16);
}

template <bool kBF16>
static int launch_long(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const Params& p,
                       cudaStream_t s) {
    CUtensorMap tq, tk, tv;
    const int rc = make_tmaps<kBF16>(tq, tk, tv, q, ldq, k, ldk, v, ldv, p.B * p.Lq, p.B * p.Lk, p);
    if (rc) return rc;
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(attention_long_kernel<kBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           LONG_SMEM_BYTES));
        attr_set = true;
    }
    attention_long_kernel<kBF16><<<dim3(static_cast<unsigned>(p.n_qt), static_cast<unsigned>(p.H), static_cast<unsigned>(p.B)),
                                   LONG_THREADS, LONG_SMEM_BYTES, s>>>(tq, tk, tv, p);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

template <bool kBF16>
static int launch(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, int q_rows, int k_rows,
                  const Params& p, cudaStream_t s) {
    CUtensorMap tq, tk, tv;
    const int rc = make_tmaps<kBF16>(tq, tk, tv, q, ldq, k, ldk, v, ldv, q_rows, k_rows, p);
    if (rc) return rc;
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel<kBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set = true;
    }
    attention_kernel<kBF16><<<dim3(static_cast<unsigned>(p.n_qt), static_cast<unsigned>(p.H), static_cast<unsigned>(p.B)),
                              THREADS, SMEM_BYTES, s>>>(tq, tk, tv, p);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

template <bool kBF16>
static int launch_packed(const void* qkv, int64_t ld, int rows, const Params& tp, const PackedParams& p, cudaStream_t s) {
    CUtensorMap tq, tk, tv;
    const int rc = make_tmaps<kBF16>(tq, tk, tv, qkv, ld, qkv, ld, qkv, ld, rows, rows, tp);
    if (rc) return rc;
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(attention_packed_kernel<kBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(packed_smem_bytes(PK_MAX_TILES * BK))));
        attr_set = true;
    }
    attention_packed_kernel<kBF16><<<static_cast<unsigned>(p.G * p.H), PK_THREADS, packed_smem_bytes(p.L), s>>>(tq, tk, tv, p);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

static Params base_params(int B, int H, int Lq, int Lk, int q_col0, int k_col0, int v_col0, void* out, int64_t ldo,
                          const float* add_mask, const float* bias_delta, float scale, float causal_value) {
    Params p;
    p.B = B, p.H = H, p.Lq = Lq, p.Lk = Lk;
    p.q_col0 = q_col0, p.k_col0 = k_col0, p.v_col0 = v_col0;
    p.O = static_cast<uint16_t*>(out);
    p.ldo = ldo;
    p.add_mask = add_mask;
    p.bias_delta = bias_delta;
    p.scale = scale;
    p.causal_value = causal_value;
    p.q_div = 1;
    p.o_partial = nullptr;
    p.ml_partial = nullptr;
    p.lse_out = nullptr;
    p.drop = abdrop::make_key(0.f, 0, 0);
    p.blk_live = nullptr;
    p.n_qt = (Lq + BQ - 1) / BQ;
    return p;
}

// out[b, i, h, :] = sum_s w_s O_s / sum_s w_s l_s with w_s = exp(m_s - max_s m_s); one warp per (b, i, h)
template <bool kBF16>
__global__ void combine_splits_kernel(const float* __restrict__ o_partial, const float* __restrict__ ml, int B, int splits,
                                      int Lq, int H, uint16_t* __restrict__ out, int64_t ldo, float* __restrict__ lse_out) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= B * Lq * H) return;
    const int h = w % H, i = (w / H) % Lq, b = w / (H * Lq);
    float M = -INFINITY;
    for (int s = 0; s < splits; ++s) {
        const size_t row = (static_cast<size_t>(b) * splits + s) * Lq + i;
        M = fmaxf(M, ml[(row * H + h) * 2]);
    }
    float acc0 = 0.f, acc1 = 0.f, den = 0.f;
    for (int s = 0; s < splits; ++s) {
        const size_t row = (static_cast<size_t>(b) * splits + s) * Lq + i;
        const float wgt = exp2f((ml[(row * H + h) * 2] - M) * LOG2E);
        den += wgt * ml[(row * H + h) * 2 + 1];
        const float2 o = reinterpret_cast<const float2*>(o_partial + row * (static_cast<size_t>(H) * D) + h * D)[lane];
        acc0 += wgt * o.x;
        acc1 += wgt * o.y;
    }
    const float inv = 1.0f / den;
    if (lse_out != nullptr && lane == 0) lse_out[(static_cast<size_t>(b) * H + h) * Lq + i] = M + __logf(den);
    reinterpret_cast<uint32_t*>(out + (static_cast<size_t>(b) * Lq + i) * ldo + h * D)[lane] =
        pack2<kBF16>(acc0 * inv, acc1 * inv);
}

}  // namespace attn

extern "C" {

int atlas_b200_attention(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                         const void* v, int64_t ldv, int32_t v_col0, void* out, int64_t ldo, const float* add_mask,
                         const float* bias_delta, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                         float causal_value, int32_t q_div, float* o_partial, float* ml_partial, int32_t is_bf16,
                         void* stream) {
    return atlas_b200_attention_ex(q, ldq, q_col0, k, ldk, k_col0, v, ldv, v_col0, out, ldo, add_mask, bias_delta, B, H, Lq,
                                   Lk, scale, causal_value, q_div, o_partial, ml_partial, nullptr, is_bf16, stream);
}

int atlas_b200_attention_ex(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                            const void* v, int64_t ldv, int32_t v_col0, void* out, int64_t ldo, const float* add_mask,
                            const float* bias_delta, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                            float causal_value, int32_t q_div, float* o_partial, float* ml_partial, float* lse_out,
                            int32_t is_bf16, void* stream) {
    return atlas_b200_attention_train(q, ldq, q_col0, k, ldk, k_col0, v, ldv, v_col0, out, ldo, add_mask, bias_delta, B, H, Lq,
                                      Lk, scale, causal_value, q_div, o_partial, ml_partial, lse_out, 0.f, 0, 0, nullptr,
                                      is_bf16, stream);
}

// Self-attention over the PACKED rows of the padding-compacted FiD encoder (atlas_b200_segment_tile_scan): segment b keeps the
// first popcount(keep[b, :]) of its L / 64 tiles, stored back to back from row 64 * tile_off[b * (L / 64)] of qkv / out.
int atlas_b200_attention_packed(const void* qkv, int64_t ld, int32_t q_col0, int32_t k_col0, int32_t v_col0, void* out, int64_t ldo,
                                const float* add_mask, const float* bias_delta, const uint8_t* keep, const int32_t* tile_off,
                                int32_t B, int32_t H, int32_t L, float scale, int32_t is_bf16, void* stream) {
    using namespace attn;
    AB_REQUIRE(B > 0 && H > 0 && L > 0 && L % 64 == 0 && L <= 384 && keep != nullptr && tile_off != nullptr,
               "attention_packed: 0 < L <= 384, L %% 64 == 0 and the segment tables are required (got L=%d)", L);
    AB_REQUIRE(ld % 8 == 0 && ldo % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 && v_col0 % 8 == 0,
               "attention_packed: strides and column offsets must be multiples of 8 elements");
    AB_REQUIRE(static_cast<int64_t>(B) * L < (1ll << 31), "attention_packed: more than 2^31 rows");
    cudaStream_t ls = static_cast<cudaStream_t>(stream);
    const Params tp = base_params(B, H, L, L, q_col0, k_col0, v_col0, out, ldo, add_mask, bias_delta, scale, 0.f);
    PackedParams p;
    p.S = B, p.H = H, p.L = L;
    // CTAs per head: one CTA per SM in all, every CTA with at least one segment
    p.G = std::max(1, std::min(B, abh::num_sms() / H));
    p.q_col0 = q_col0, p.k_col0 = k_col0, p.v_col0 = v_col0;
    p.O = static_cast<uint16_t*>(out);
    p.ldo = ldo;
    p.add_mask = add_mask;
    p.bias_delta = bias_delta;
    p.keep = keep;
    p.tile_off = tile_off;
    p.scale = scale;
    // the packed rows of all segments: at most B * L (the tensor maps only bound the TMA boxes)
    const int rows = B * L;
    abh::prof_begin(ls, abh::PROF_ATTENTION);
    const int lrc = is_bf16 ? launch_packed<true>(qkv, ld, rows, tp, p, ls) : launch_packed<false>(qkv, ld, rows, tp, p, ls);
    if (lrc) return lrc;
    // dense-equivalent work, like the masked-block skipping of the padded layout
    abh::prof_end(ls, abh::PROF_ATTENTION, 4.0 * B * H * static_cast<double>(L) * L * attn::D);
    abh::count_launch();
    return ATLAS_B200_OK;
}

int atlas_b200_attention_train(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                               const void* v, int64_t ldv, int32_t v_col0, void* out, int64_t ldo, const float* add_mask,
                               const float* bias_delta, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                               float causal_value, int32_t q_div, float* o_partial, float* ml_partial, float* lse_out,
                               float dropout_p, uint64_t seed, uint64_t offset, const uint8_t* key_block_live,
                               int32_t is_bf16, void* stream) {
    using namespace attn;
    AB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention: need 0 <= dropout_p < 1 (got %f)", dropout_p);
    const abdrop::Key drop = abdrop::make_key(dropout_p, seed, offset);
    const bool dropping = drop.thr16 != 0u;
    AB_REQUIRE(!dropping || q_div == 1 || Lk % 32 == 0,
               "attention: dropout over split keys needs a split length that is a multiple of 32 (got %d)", Lk);
    AB_REQUIRE(lse_out == nullptr || o_partial == nullptr, "attention: lse_out is produced by attention_combine in split mode");
    AB_REQUIRE(q_div >= 1 && B % q_div == 0, "attention: q_div must divide the number of key segments");
    AB_REQUIRE((o_partial == nullptr) == (ml_partial == nullptr), "attention: partial outputs come in pairs");
    AB_REQUIRE(B >= 0 && H > 0 && Lq > 0 && Lk > 0 && Lk <= MAX_LK, "attention: need 0 < Lk <= %d (got Lq=%d Lk=%d)",
               MAX_LK, Lq, Lk);
    AB_REQUIRE(Lq + Lk - 1 <= 2 * MAX_LK, "attention: Lq + Lk too large for the bias table");
    AB_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 &&
                   v_col0 % 8 == 0,
               "attention: strides and column offsets must be multiples of 8 elements");
    if (B == 0) return ATLAS_B200_OK;
    Params p = base_params(B, H, Lq, Lk, q_col0, k_col0, v_col0, out, ldo, add_mask, bias_delta, scale, causal_value);
    p.q_div = q_div;
    p.o_partial = o_partial;
    p.ml_partial = ml_partial;
    p.lse_out = lse_out;
    p.drop = drop;
    p.blk_live = key_block_live;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    abh::prof_begin(s, abh::PROF_ATTENTION);
    const int lrc = is_bf16 ? launch<true>(q, ldq, k, ldk, v, ldv, (B / q_div) * Lq, B * Lk, p, s)
                            : launch<false>(q, ldq, k, ldk, v, ldv, (B / q_div) * Lq, B * Lk, p, s);
    if (lrc) return lrc;
    abh::prof_end(s, abh::PROF_ATTENTION, 4.0 * B * H * static_cast<double>(Lq) * Lk * D);
    abh::count_launch();
    return ATLAS_B200_OK;
}

int atlas_b200_attention_long(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                              const void* v, int64_t ldv, int32_t v_col0, void* out, int64_t ldo, const float* add_mask,
                              const float* bias_delta, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                              float causal_value, float* lse_out, float dropout_p, uint64_t seed, uint64_t offset,
                              const uint8_t* key_block_live, int32_t is_bf16, void* stream) {
    using namespace attn;
    AB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention_long: need 0 <= dropout_p < 1 (got %f)", dropout_p);
    AB_REQUIRE(B >= 0 && H > 0 && Lq > 0 && Lk > 0 && Lk <= LONG_MAX_LK, "attention_long: need 0 < Lk <= %d (got Lq=%d Lk=%d)",
               LONG_MAX_LK, Lq, Lk);
    AB_REQUIRE(Lq + Lk - 1 <= 2 * LONG_MAX_LK, "attention_long: Lq + Lk - 1 = %d exceeds the bias table (%d)", Lq + Lk - 1,
               2 * LONG_MAX_LK);
    AB_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 &&
                   v_col0 % 8 == 0,
               "attention_long: strides and column offsets must be multiples of 8 elements");
    AB_REQUIRE(static_cast<int64_t>(B) * Lq < (1ll << 31) && static_cast<int64_t>(B) * Lk < (1ll << 31),
               "attention_long: more than 2^31 rows");
    if (B == 0) return ATLAS_B200_OK;
    Params p = base_params(B, H, Lq, Lk, q_col0, k_col0, v_col0, out, ldo, add_mask, bias_delta, scale, causal_value);
    p.lse_out = lse_out;
    p.drop = abdrop::make_key(dropout_p, seed, offset);
    p.blk_live = key_block_live;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    abh::prof_begin(s, abh::PROF_ATTENTION);
    const int lrc = is_bf16 ? launch_long<true>(q, ldq, k, ldk, v, ldv, p, s) : launch_long<false>(q, ldq, k, ldk, v, ldv, p, s);
    if (lrc) return lrc;
    abh::prof_end(s, abh::PROF_ATTENTION, 4.0 * B * H * static_cast<double>(Lq) * Lk * D);
    abh::count_launch();
    return ATLAS_B200_OK;
}

int atlas_b200_attention_combine(const float* o_partial, const float* ml_partial, int32_t B, int32_t splits, int32_t Lq,
                                 int32_t H, void* out, int64_t ldo, int32_t is_bf16, void* stream) {
    return atlas_b200_attention_combine_ex(o_partial, ml_partial, B, splits, Lq, H, out, ldo, nullptr, is_bf16, stream);
}

int atlas_b200_attention_combine_ex(const float* o_partial, const float* ml_partial, int32_t B, int32_t splits, int32_t Lq,
                                    int32_t H, void* out, int64_t ldo, float* lse_out, int32_t is_bf16, void* stream) {
    AB_REQUIRE(B >= 0 && splits >= 1 && Lq > 0 && H > 0 && ldo % 2 == 0, "attention_combine: bad shape");
    if (B == 0) return ATLAS_B200_OK;
    const int warps = B * Lq * H;
    const int grid = (warps * 32 + 255) / 256;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16)
        attn::combine_splits_kernel<true><<<grid, 256, 0, s>>>(o_partial, ml_partial, B, splits, Lq, H,
                                                               static_cast<uint16_t*>(out), ldo, lse_out);
    else
        attn::combine_splits_kernel<false><<<grid, 256, 0, s>>>(o_partial, ml_partial, B, splits, Lq, H,
                                                                static_cast<uint16_t*>(out), ldo, lse_out);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
