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
// arithmetic, with K and V streamed through a ring of shared-memory slots instead of held resident.
//
// The padding-compacted encoders (segment b keeps the first n_b of its 64-row tiles, stored back to back, L <= 576): the
// no-grad attention up to 384 tokens runs on attention_packed_kernel below, a persistent kernel over (segment, head) items with
// the same per-block arithmetic; with lse or dropout (the training forward) and at 448 to 576 tokens attention_kernel runs
// with packed-row addressing (Params::tile_off), its positions, mask, bias, dropout rows and lse those of the padded layout.
//
// All three kernels run that arithmetic through the same functions (issue_s, block_softmax, rescale_and_pack, drop_probs,
// issue_pv, write_rows), so their results agree bit for bit where their inputs do.
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
    // packed rows (atlas_b200_attention_packed, self-attention with Lq = Lk): segment b is its kept 64-row tiles, blk_live =
    // keep (a prefix of the segment), stored back to back from row 64 * tile_off[b * nkb] of q / k / v / out; nullptr: the
    // padded layout.  Positions, mask, bias, dropout rows and lse stay those of the padded layout.
    const int32_t* tile_off;
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

// ---- The per-block arithmetic, shared by the three kernels.  A warpgroup owns 64 query rows; this thread holds rows r and
// r + 8 of them (segment rows i0 and i0 + 8) and, of each 8-key group j of a 64-key block, the keys 8 j + cq + c, cq =
// 2 (lane % 4), c = 0, 1: element 4 j + 2 hh + c of the fragments sc (S, then t, then p) and o is (row r + 8 hh, key c).

// S = Q K^T for one 64-key block: the warpgroup's 64-row query tile at sQ, the block's K tile at sK; one commit group
template <bool kBF16>
__device__ __forceinline__ void issue_s(float (&sc)[32], const uint32_t sQ, const uint32_t sK) {
#pragma unroll
    for (int k = 0; k < D / 16; ++k)
        ab::wgmma_m64n64k16_ss<kBF16, 0, 0>(sc, ab::wgmma_desc_sw128(sQ + k * 32u), ab::wgmma_desc_sw128(sK + k * 32u), k);
    ab::wgmma_commit();
}

// O += P V for one 64-key block: P from registers (rescale_and_pack), the block's V tile at sV as it lies in memory (the
// MN-major operand); one commit group
template <bool kBF16>
__device__ __forceinline__ void issue_pv(float (&o)[32], const uint32_t (&pa)[16], const uint32_t sV) {
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
        ab::wgmma_m64n64k16_rs<kBF16, 1>(o, *reinterpret_cast<const uint32_t(*)[4]>(&pa[4 * k]),
                                         ab::wgmma_desc_sw128(sV + k * 2048u, 8192), 1);
    ab::wgmma_commit();
}

// The online softmax of one block on its completed S (keys key0 + 8 j + c, key0 = 64 kb + cq): t = S * scale2 + mask[key]
// + bias[hh][key] in the log2 domain (bias[hh] = the staged bias row of row r + 8 hh, read only if has_bias), the new row
// maxima over the quad, sc <- p = 2^(t - base) and l_run <- l_run * corr + sum p.  corr = 2^(m_old - base) is o's rescale.
__device__ __forceinline__ void block_softmax(float (&sc)[32], float (&m_run)[2], float (&l_run)[2], float (&corr)[2],
                                              const float* mask, const float* const (&bias)[2], const bool has_bias,
                                              const int key0, const float scale2) {
    ab::wgmma_reg_fence(sc);
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int key = key0 + 8 * j + c;
            const float mk = mask[key];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float a = mk;
                if (has_bias) a += bias[hh][key];
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
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float e0 = ex2_approx(sc[4 * j + 2 * hh] - base[hh]);
            const float e1 = ex2_approx(sc[4 * j + 2 * hh + 1] - base[hh]);
            // l_run * corr and the first pair's sum round once, as one fma: written out rather than left to the compiler's
            // contraction, which code between the multiply and the add (a branch) can prevent in one kernel and not another
            l_run[hh] = j == 0 ? fmaf(l_run[hh], corr[hh], e0 + e1) : l_run[hh] + (e0 + e1);
            sc[4 * j + 2 * hh] = e0;
            sc[4 * j + 2 * hh + 1] = e1;
        }
    }
}

// o *= corr, then P = p rounded to 16 bits as the A fragment of k16 step j / 2: a0 = (r, keys 0-7), a1 = (r + 8, keys 0-7),
// a2 / a3 = keys 8-15
template <bool kBF16>
__device__ __forceinline__ void rescale_and_pack(uint32_t (&pa)[16], float (&o)[32], const float (&sc)[32],
                                                 const float (&corr)[2]) {
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
}

// Dropout on P (rescale_and_pack's fragment), after the row sums took every probability: a dropped probability's 16 bits are
// cleared, which are the bits of a packed 0.  The keep bits of rows R[hh] (row r + 8 hh in the key's row numbering), in
// groups of 32 keys from key column col.
__device__ __forceinline__ void drop_probs(uint32_t (&pa)[16], const abdrop::Key& drop, const uint64_t (&R)[2], const int col,
                                           const uint32_t lane) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        uint32_t w[2][4];
#pragma unroll
        for (int gg = 0; gg < 2; ++gg)
            abdrop::attn_words(drop, R[hh], static_cast<uint32_t>((col + gg * 32) >> 5), lane & 3u, w[gg]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t word = w[j >> 2][j & 3];
            pa[4 * (j >> 1) + 2 * (j & 1) + hh] &=
                (abdrop::keep_lo(drop, word) ? 0x0000FFFFu : 0u) | (abdrop::keep_hi(drop, word) ? 0xFFFF0000u : 0u);
        }
    }
}

// a row's sum over the four threads of its quad
__device__ __forceinline__ float quad_sum(float x) {
    x += __shfl_xor_sync(0xffffffffu, x, 1);
    return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// The finished rows i = i0 and i0 + 8 below n_rows: the log-sum-exp (natural log) at lse[i] unless lse is null, and
// O * inv_keep / l rounded to 16 bits at out + i * ldo (out: this thread's first column in the segment's row 0).
template <bool kBF16>
__device__ __forceinline__ void write_rows(const float (&o)[32], const float (&m_run)[2], const float (&l_run)[2], const int i0,
                                           const int n_rows, uint16_t* out, const int64_t ldo, float* lse,
                                           const float inv_keep, const uint32_t lane) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const float l = quad_sum(l_run[hh]);
        const int i = i0 + 8 * hh;
        if (i >= n_rows) continue;
        const float inv = inv_keep / l;
        if (lse != nullptr && (lane & 3u) == 0u) lse[i] = m_run[hh] * (1.0f / LOG2E) + __logf(l);
        uint16_t* dst = out + i * ldo;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2<kBF16>(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
    }
}

// Shared-memory tables of attention_kernel and attention_long_kernel, both times log2e, written by nthreads threads: the key
// mask of segment b for keys 0 .. 64 nkb - 1 (-inf past Lk) and, if has_bias, entries d0 .. d0 + n_bias - 1 of head h's row
// of the [H, Lq + Lk - 1] bias table plus the causal value where j > i (entries past the table stay finite: 0).
__device__ __forceinline__ void stage_tables(float* s_mask, float* s_bias, const Params& p, const int b, const int h,
                                             const int nkb, const bool has_bias, const int d0, const int n_bias,
                                             const int nthreads) {
    for (int j = threadIdx.x; j < nkb * BK; j += nthreads)
        s_mask[j] = (j < p.Lk) ? (p.add_mask ? p.add_mask[static_cast<size_t>(b) * p.Lk + j] * LOG2E : 0.f) : -INFINITY;
    if (!has_bias) return;
    const int n_valid = p.Lq + p.Lk - 1;
    for (int t = threadIdx.x; t < n_bias; t += nthreads) {
        const int d = d0 + t;
        float v = 0.f;
        if (d < n_valid) {
            v = p.bias_delta ? p.bias_delta[static_cast<size_t>(h) * n_valid + d] : 0.f;
            if (p.causal_value != 0.f && d > p.Lq - 1) v += p.causal_value;   // j > i
        }
        s_bias[t] = v * LOG2E;
    }
}

// Per-row constants of attention_kernel and attention_long_kernel for rows r and r + 8: the staged bias row (s_bias holds the
// table from the offset of row bias_off to key 0) and the dropout row.  Rows past Lq, which are not stored, take row Lq - 1.
__device__ __forceinline__ void row_setup(const float* (&bias)[2], uint64_t (&R)[2], const float* s_bias, const int bias_off,
                                          const Params& p, const int b, const int h, const int i0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int i = min(i0 + 8 * hh, p.Lq - 1);
        bias[hh] = s_bias + bias_off - i;
        R[hh] = (static_cast<uint64_t>(b / p.q_div) * p.H + h) * p.Lq + i;
    }
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
    int q_row0 = (b / p.q_div) * p.Lq;
    int k_row0 = b * p.Lk;
    int o_row0 = b * p.Lq;
    int n_rows = p.Lq;            // rows of the segment that are stored
    int n_qload = 2;              // 64-row halves of the query tile loaded
    if (p.tile_off != nullptr) {
        q_row0 = k_row0 = o_row0 = BK * __ldg(p.tile_off + static_cast<size_t>(b) * nkb);
        n_rows = BK * __popc(live);
        if (qt * BQ >= n_rows) return;
        // a half past the segment's last kept tile is not loaded: its rows are neither stored nor allocated past the last
        // segment; the MMAs keep the rows of a tile apart
        n_qload = min(2, (n_rows - qt * BQ) / BK);
    }

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
        ab::mbar_arrive_expect_tx(&load_bar, static_cast<uint32_t>(n_qload * TILE_BYTES + 2 * nload * TILE_BYTES));
        for (int t = 0; t < n_qload; ++t)
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
    stage_tables(s_mask, s_bias, p, b, h, nkb, has_bias, 0, 2 * MAX_LK + BK, THREADS);
    __syncthreads();
    ab::mbar_wait(&load_bar, 0, 40);

    // ---- warpgroup g: query rows 64 g .. 64 g + 63 of the tile; this thread: rows r and r + 8, key pairs 8 j + 2 (lane % 4)
    const uint32_t g = warp >> 2, wl = warp & 3u;
    const int i0 = qt * BQ + static_cast<int>(g * 64u + wl * 16u + (lane >> 2));   // query index of row r (in the segment)
    const int cq = static_cast<int>(2u * (lane & 3u));
    const float scale2 = p.scale * LOG2E;
    const bool dropping = p.drop.thr16 != 0u;
    const float* bias[2];
    uint64_t R[2];
    row_setup(bias, R, s_bias, p.Lq - 1, p, b, h, i0);
    float o[32];
#pragma unroll
    for (int x = 0; x < 32; ++x) o[x] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    for (int kb = 0; kb < nkb; ++kb) {
        if (!((live >> kb) & 1u)) continue;
        float sc[32], corr[2];
        uint32_t pa[16];
        ab::wgmma_fence();
        issue_s<kBF16>(sc, sQ + g * 8192u, sK + kb * TILE_BYTES);
        ab::wgmma_wait<0>();
        block_softmax(sc, m_run, l_run, corr, s_mask, bias, has_bias, kb * BK + cq, scale2);
        rescale_and_pack<kBF16>(pa, o, sc, corr);
        if (dropping) drop_probs(pa, p.drop, R, (b % p.q_div) * p.Lk + kb * BK, lane);
        ab::wgmma_fence();
        issue_pv<kBF16>(o, pa, sV + kb * TILE_BYTES);
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(o);
    }

    // ---- output: normalised 16-bit rows, or split-KV partials (un-normalised fp32 O, row max and row sum)
    if (p.o_partial == nullptr) {
        write_rows<kBF16>(o, m_run, l_run, i0, n_rows, p.O + static_cast<size_t>(o_row0) * p.ldo + h * D + cq, p.ldo,
                          p.lse_out ? p.lse_out + (static_cast<size_t>(b) * p.H + h) * p.Lq : nullptr, p.drop.inv_keep, lane);
        return;
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const float l = quad_sum(l_run[hh]);
        const int i = i0 + 8 * hh;
        if (i >= p.Lq) continue;
        const size_t orow = static_cast<size_t>(o_row0) + i;
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
    }
}

// ---- attention_long_kernel: the same contract for Lk up to LONG_MAX_LK keys (no split-KV partials, no packed layout).  K and V
// stream through a LONG_STAGES-deep ring of 64-key tiles: one producer warp issues their TMA loads (full / empty mbarriers),
// the two consumer warpgroups of attention_kernel sweep the live blocks.  The CTA's slice of the bias table
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
    // last (clamped) row, bias_off, to key 0
    const bool has_bias = (p.bias_delta != nullptr) || (p.causal_value != 0.f);
    const int bias_off = min(qt * BQ + BQ - 1, p.Lq - 1);
    stage_tables(s_mask, s_bias, p, b, h, nkb, has_bias, (p.Lq - 1) - bias_off, nkb * BK + BQ - 1, LONG_THREADS);
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
    const float* bias[2];
    uint64_t R[2];
    row_setup(bias, R, s_bias, bias_off, p, b, h, i0);
    float o[32];
#pragma unroll
    for (int x = 0; x < 32; ++x) o[x] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    int n_used = 0;
    for (int kb = 0; kb < nkb; ++kb) {
        if (!all_live && !s_live[kb]) continue;
        const int s = n_used % LONG_STAGES;
        ab::mbar_wait(&full_bar[s], (n_used / LONG_STAGES) & 1, 52);
        float sc[32], corr[2];
        uint32_t pa[16];
        ab::wgmma_fence();
        issue_s<kBF16>(sc, sQ + g * 8192u, sK + s * TILE_BYTES);
        ab::wgmma_wait<0>();
        block_softmax(sc, m_run, l_run, corr, s_mask, bias, has_bias, kb * BK + cq, scale2);
        rescale_and_pack<kBF16>(pa, o, sc, corr);
        if (dropping) drop_probs(pa, p.drop, R, (b % p.q_div) * p.Lk + kb * BK, lane);
        ab::wgmma_fence();
        issue_pv<kBF16>(o, pa, sV + s * TILE_BYTES);
        ab::wgmma_wait<0>();
        ab::wgmma_reg_fence(o);
        __syncwarp();
        if (lane == 0) ab::mbar_arrive(&empty_bar[s]);     // this warp's MMAs on the slot have completed
        ++n_used;
    }

    write_rows<kBF16>(o, m_run, l_run, i0, p.Lq, p.O + static_cast<size_t>(b) * p.Lq * p.ldo + h * D + cq, p.ldo,
                      p.lse_out ? p.lse_out + (static_cast<size_t>(b) * p.H + h) * p.Lq : nullptr, p.drop.inv_keep, lane);
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
            const float* const bias[2] = {s_bias + (p.L - 1) - i0, s_bias + (p.L - 1) - (i0 + 8)};
            ab::mbar_wait_nocall(&full_q[s], (qi / PK_Q_STAGES) & 1);

            float o[32], sc[32], corr[2];
            uint32_t pa[16];
            float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll
            for (int x = 0; x < 32; ++x) o[x] = 0.f;
            ab::wgmma_fence();
            issue_s<kBF16>(sc, sQs, sK);
            ab::wgmma_wait<0>();
            block_softmax(sc, m_run, l_run, corr, mk, bias, has_bias, cq, scale2);
            rescale_and_pack<kBF16>(pa, o, sc, corr);
            for (int kb = 1; kb < n; ++kb) {
                // S_kb and O += P_{kb-1} V_{kb-1} in flight; the softmax of block kb runs under the P V
                ab::wgmma_fence();
                issue_s<kBF16>(sc, sQs, sK + kb * TILE_BYTES);
                issue_pv<kBF16>(o, pa, sV + (kb - 1) * TILE_BYTES);
                ab::wgmma_wait<1>();
                block_softmax(sc, m_run, l_run, corr, mk, bias, has_bias, kb * BK + cq, scale2);
                ab::wgmma_wait<0>();
                ab::wgmma_reg_fence(o);
#pragma unroll
                for (int x = 0; x < 16; ++x) asm volatile("" : "+r"(pa[x])::"memory");   // P_{kb-1} was read until here
                rescale_and_pack<kBF16>(pa, o, sc, corr);
            }
            ab::wgmma_fence();
            issue_pv<kBF16>(o, pa, sV + (n - 1) * TILE_BYTES);
            __syncwarp();
            if (lane == 0) ab::mbar_arrive(&empty_q[s]);     // every S of the query tile is complete
            ab::wgmma_wait<0>();
            ab::wgmma_reg_fence(o);
            write_rows<kBF16>(o, m_run, l_run, i0, n * BK, p.O + static_cast<size_t>(it.y) * p.ldo + h * D + cq, p.ldo, nullptr,
                              1.0f, lane);
        }
        q0 += n;
        __syncwarp();
        if (lane == 0) ab::mbar_arrive(&empty_kv[slot]);     // this warp's MMAs on the slot have completed
    }
}

static int make_tmaps(CUtensorMap& tq, CUtensorMap& tk, CUtensorMap& tv, const bool bf16, const void* q, int64_t ldq,
                      const void* k, int64_t ldk, const void* v, int64_t ldv, int q_rows, int k_rows, const Params& p) {
    int rc = abh::make_tmap_2d_16bit(&tq, q, static_cast<uint64_t>(q_rows), static_cast<uint64_t>(p.q_col0 + p.H * D),
                                     static_cast<uint64_t>(ldq), BK, D, bf16);
    if (rc) return rc;
    rc = abh::make_tmap_2d_16bit(&tk, k, static_cast<uint64_t>(k_rows), static_cast<uint64_t>(p.k_col0 + p.H * D),
                                 static_cast<uint64_t>(ldk), BK, D, bf16);
    if (rc) return rc;
    return abh::make_tmap_2d_16bit(&tv, v, static_cast<uint64_t>(k_rows), static_cast<uint64_t>(p.v_col0 + p.H * D),
                                   static_cast<uint64_t>(ldv), BK, D, bf16);
}

// One launch of kernel kF16 or kBF16 (by bf16) with kernel parameters kp, on the tensor maps of Q (q_rows rows) and K / V
// (k_rows rows) with the columns of tp's heads.  Each kernel's dynamic shared-memory limit is raised to max_smem on its
// first launch.
template <auto kF16, auto kBF16, typename KP>
static int launch(const bool bf16, const dim3 grid, const int threads, const size_t smem, const int max_smem, const void* q,
                  int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, int q_rows, int k_rows,
                  const Params& tp, const KP& kp, cudaStream_t s) {
    CUtensorMap tq, tk, tv;
    const int rc = make_tmaps(tq, tk, tv, bf16, q, ldq, k, ldk, v, ldv, q_rows, k_rows, tp);
    if (rc) return rc;
    const auto kernel = bf16 ? kBF16 : kF16;
    static bool attr_set[2] = {false, false};
    if (!attr_set[bf16]) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
        attr_set[bf16] = true;
    }
    kernel<<<grid, threads, smem, s>>>(tq, tk, tv, kp);
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
    p.tile_off = nullptr;
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

// Self-attention over the PACKED rows of the padding-compacted FiD encoder (atlas_b200_segment_tile_scan): segment b keeps the
// first popcount(keep[b, :]) of its L / 64 tiles, stored back to back from row 64 * tile_off[b * (L / 64)] of qkv / out.
// Without lse_out and dropout, L <= 384 runs on the persistent attention_packed_kernel; everything else (the training forward,
// 384 < L <= 576) on attention_kernel with packed-row addressing.
int atlas_b200_attention_packed(const void* qkv, int64_t ld, int32_t q_col0, int32_t k_col0, int32_t v_col0, void* out, int64_t ldo,
                                const float* add_mask, const float* bias_delta, const uint8_t* keep, const int32_t* tile_off,
                                int32_t B, int32_t H, int32_t L, float scale, float* lse_out, float dropout_p, uint64_t seed,
                                uint64_t offset, int32_t is_bf16, void* stream) {
    using namespace attn;
    AB_REQUIRE(B > 0 && H > 0 && L > 0 && L % 64 == 0 && L <= MAX_LK && keep != nullptr && tile_off != nullptr,
               "attention_packed: 0 < L <= %d, L %% 64 == 0 and the segment tables are required (got L=%d)", MAX_LK, L);
    AB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention_packed: need 0 <= dropout_p < 1 (got %f)", dropout_p);
    AB_REQUIRE(ld % 8 == 0 && ldo % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 && v_col0 % 8 == 0,
               "attention_packed: strides and column offsets must be multiples of 8 elements");
    AB_REQUIRE(static_cast<int64_t>(B) * L < (1ll << 31), "attention_packed: more than 2^31 rows");
    cudaStream_t ls = static_cast<cudaStream_t>(stream);
    Params tp = base_params(B, H, L, L, q_col0, k_col0, v_col0, out, ldo, add_mask, bias_delta, scale, 0.f);
    tp.drop = abdrop::make_key(dropout_p, seed, offset);
    // the packed rows of all segments: at most B * L (the tensor maps only bound the TMA boxes; no box reaches past the last
    // kept tile)
    const int rows = B * L;
    const int nb = L / BK;
    // the kernels' work: 4 * 64 FLOPs per (query, key) pair of the kept tiles, 64 x 64 pairs per (query tile, key tile)
    const double work_per_tile_pair = 4.0 * H * BK * BK * D;
    if (L > PK_MAX_TILES * BK || lse_out != nullptr || tp.drop.thr16 != 0u) {
        tp.lse_out = lse_out;
        tp.blk_live = keep;
        tp.tile_off = tile_off;
        abh::prof_begin(ls, abh::PROF_ATTENTION);
        const int lrc = launch<attention_kernel<false>, attention_kernel<true>>(
            is_bf16, dim3(tp.n_qt, H, B), THREADS, SMEM_BYTES, SMEM_BYTES, qkv, ld, qkv, ld, qkv, ld, rows, rows, tp, tp, ls);
        if (lrc) return lrc;
        abh::prof_end_tile_pairs(ls, abh::PROF_ATTENTION, work_per_tile_pair, keep, B, nb);
        abh::count_launch();
        return ATLAS_B200_OK;
    }
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
    abh::prof_begin(ls, abh::PROF_ATTENTION);
    const int lrc = launch<attention_packed_kernel<false>, attention_packed_kernel<true>>(
        is_bf16, dim3(p.G * p.H), PK_THREADS, packed_smem_bytes(L), static_cast<int>(packed_smem_bytes(PK_MAX_TILES * BK)), qkv,
        ld, qkv, ld, qkv, ld, rows, rows, tp, p, ls);
    if (lrc) return lrc;
    abh::prof_end_tile_pairs(ls, abh::PROF_ATTENTION, work_per_tile_pair, keep, B, nb);
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
    const int lrc = launch<attention_kernel<false>, attention_kernel<true>>(
        is_bf16, dim3(p.n_qt, H, B), THREADS, SMEM_BYTES, SMEM_BYTES, q, ldq, k, ldk, v, ldv, (B / q_div) * Lq, B * Lk, p, p, s);
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
    const int lrc = launch<attention_long_kernel<false>, attention_long_kernel<true>>(
        is_bf16, dim3(p.n_qt, H, B), LONG_THREADS, LONG_SMEM_BYTES, LONG_SMEM_BYTES, q, ldq, k, ldk, v, ldv, B * Lq, B * Lk, p, p,
        s);
    if (lrc) return lrc;
    abh::prof_end(s, abh::PROF_ATTENTION, 4.0 * B * H * static_cast<double>(Lq) * Lk * D);
    abh::count_launch();
    return ATLAS_B200_OK;
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
