// Backward of the fused attention (csrc/attention.cu), head_dim 64, any Lq / Lk:
//     S = scale * Q K^T + bias_delta[h, j - i + Lq - 1] + add_mask[b, j] (+ causal_value where j > i)
//     P = softmax_j(S)   (fp32),   O = P V
// given dO:   dV = P^T dO,   dP = dO V^T,   dS = P o (dP - D),  D_i = sum_d dO_id O_id,
//             dQ = scale * dS K,   dK = scale * dS^T Q,   dbias_delta[h, j - i + Lq - 1] += dS_ij.
// This is what autograd derives for `BertSelfAttention.forward` (src/modeling_bert.py:328-366), `T5Attention.forward`
// (src/modeling_t5.py:478-524) and FiD's `cross_attention_forward` (src/fid.py:298-349) in the reference's training
// step (train.py -> Atlas.forward -> loss.backward()); the [B, H, Lq, Lk] score / probability tensors the reference
// keeps alive for autograd are recomputed tile by tile instead (the forward saves only O).
//
// Warp-level `mma.sync.m16n8k16` tiles (64 queries x 64 keys per CTA step, 4 warps, operands through XOR-swizzled shared
// memory + ldmatrix), two kernels so that no output needs atomics:
//   attn_bwd_dq2_kernel   CTA = (b, h, 64-query block [, key chunk]): reads the row log-sum-exp the forward kernel wrote
//                         (atlas_b200_attention_train), writes D_i = sum_d dO O to `dsum`, accumulates dQ over the key blocks
//                         (cp.async double-buffered K / V tiles); dbias through a staged dS tile + diagonal sums.  A long
//                         few-query key range (FiD cross-attention) is split over key chunks with fp32 dQ atomics.
//   attn_bwd_dkv2_kernel  CTA = (b, h, 64-key block): the transposed problem, loops over the query blocks, accumulates dK, dV.
// atlas_b200_attention_packed_bwd runs the same two kernels on the packed rows of the padding-compacted encoder
// (Params::tile_off); the CTAs of a segment's dropped tiles return at once.
// Bound: tensor (warp-level mma.sync m16n8k16 fragments).
// FLOPs per call = 2 * B*H*Lq*Lk*64 * 7 (S + dP + dQ in the first kernel, S + dP + dV + dK in the second).
#include "common.cuh"
#include "dropout.cuh"
#include "host_common.h"

#include <math.h>

namespace attnb {

constexpr int D = 64;
constexpr int BM = 64;        // rows of the CTA's resident operand (queries in dq, keys in dkv)
constexpr int BN = 64;        // rows of the streamed operand tile
constexpr int THREADS = 128;  // 4 warps x 16 rows
constexpr int TILE_BYTES = 64 * 128;

struct Params {
    const uint16_t *q, *k, *v, *o, *dout;
    int64_t ldq, ldk, ldv, ldo, lddo;
    int q_col0, k_col0, v_col0;
    uint16_t *dq, *dk, *dv;
    int64_t lddq, lddk, lddv;
    int dq_col0, dk_col0, dv_col0;
    const float* add_mask;    // [B, Lk] or nullptr
    const float* bias_delta;  // [H, Lq + Lk - 1] or nullptr
    float* dbias;             // [H, Lq + Lk - 1] (+=, atomics) or nullptr
    float* lse;               // [B, H, Lq]  (input: written by the forward kernels)
    float* dsum;              // [B, H, Lq]
    float* dq_accum;          // [B*Lq, H*64] fp32 (+=, atomics) when the keys are split over `key_chunks` CTAs, else nullptr
    int key_chunks, pad_;     // pad_ keeps the fields below at 8-byte aligned offsets: without it ptxas allocates the
                              // kernels' registers differently (other spills) for the same source
    int B, H, Lq, Lk;
    float scale, causal_value;
    abdrop::Key drop;         // attention-probability dropout of the forward; thr16 == 0: off
    const uint8_t* blk_live;  // [B, ceil(Lk / 64)] or nullptr: 64-key blocks whose keys are all masked out (softmax weight exactly
                              // 0 in fp32, so dS = 0, dK = dV = 0 there): skipped
    // packed rows (atlas_b200_attention_packed_bwd, self-attention with Lq = Lk): segment b is its kept 64-row tiles, blk_live =
    // keep (a prefix of the segment), stored back to back from row 64 * tile_off[b * nkb] of every row operand; nullptr: the
    // padded layout.  Positions, mask, bias, dropout rows, lse and dsum stay those of the padded layout.
    const int32_t* tile_off;
};

// The rows of segment b: first row and number of rows of its queries and of its keys
struct SegRows {
    int64_t q0, k0;
    int nq, nk;
};
__device__ __forceinline__ SegRows segment_rows(const Params& p, const int b, const int nkb) {
    if (p.tile_off == nullptr)
        return {static_cast<int64_t>(b) * p.Lq, static_cast<int64_t>(b) * p.Lk, p.Lq, p.Lk};
    const int64_t row0 = 64ll * __ldg(p.tile_off + static_cast<int64_t>(b) * nkb);
    int n = 0;
    for (int t = 0; t < nkb; ++t) n += __ldg(p.blk_live + static_cast<int64_t>(b) * nkb + t) != 0;
    return {row0, row0, 64 * n, 64 * n};
}

// ---- shared-memory tiles: 64 rows x 128 bytes, 16-byte chunks XOR-swizzled by the row ------------------------------
__device__ __forceinline__ uint32_t tile_off(int row, int chunk) {
    return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}

// rows [r0, r0 + 64) of a [nrows, ld] matrix (columns col .. col + 63) -> tile; rows >= nrows are zero-filled
__device__ __forceinline__ void load_tile(uint8_t* tile, const uint16_t* base, int64_t ld, int col, int64_t row_base,
                                          int r0, int nrows) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int idx = it * THREADS + static_cast<int>(threadIdx.x);
        const int row = idx >> 3, chunk = idx & 7;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (r0 + row < nrows)
            v = __ldg(reinterpret_cast<const uint4*>(base + (row_base + r0 + row) * ld + col + chunk * 8));
        *reinterpret_cast<uint4*>(tile + tile_off(row, chunk)) = v;
    }
}

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

template <bool kBF16>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if constexpr (kBF16) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                     "{%0, %1, %2, %3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                     "{%0, %1, %2, %3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
}

// acc[nt][.] (16 x 64 over d) += P(16 x 64 over the tile rows, as accumulator-layout fp32 values) . T,
// T = tile of 64 rows x 64 d: B[k = tile row][n = d] (transposing ldmatrix)
template <bool kBF16>
__device__ __forceinline__ void mma_p_tile(float (&acc)[8][4], const float (&p)[8][4], uint32_t tile, int lane) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        uint32_t a[4];
        a[0] = ab::pack2_rn<kBF16>(p[2 * kk][0], p[2 * kk][1]);
        a[1] = ab::pack2_rn<kBF16>(p[2 * kk][2], p[2 * kk][3]);
        a[2] = ab::pack2_rn<kBF16>(p[2 * kk + 1][0], p[2 * kk + 1][1]);
        a[3] = ab::pack2_rn<kBF16>(p[2 * kk + 1][2], p[2 * kk + 1][3]);
#pragma unroll
        for (int dp = 0; dp < 4; ++dp) {
            uint32_t b[4];
            ldsm_x4_t(b, tile + tile_off(kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), dp * 2 + (lane >> 4)));
            mma16816<kBF16>(acc[2 * dp], a, b[0], b[1]);
            mma16816<kBF16>(acc[2 * dp + 1], a, b[2], b[3]);
        }
    }
}

template <bool kBF16>
__device__ __forceinline__ float to_f32(uint32_t h) {
    if constexpr (kBF16) return __bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(h)));
    return __half2float(__ushort_as_half(static_cast<unsigned short>(h)));
}

// 16 x 64 fp32 accumulator (rows g / g + 8 of the warp's 16) -> 16-bit global rows
template <bool kBF16>
__device__ __forceinline__ void store_acc(const float (&acc)[8][4], float mul, uint16_t* base, int64_t ld, int col,
                                          int64_t row_base, int r_lo, int nrows, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int r = r_lo + g + half * 8;
        if (r >= nrows) continue;
        uint16_t* row = base + (row_base + r) * ld + col;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
            *reinterpret_cast<uint32_t*>(row + nt * 8 + 2 * t) =
                ab::pack2_rn<kBF16>(acc[nt][2 * half] * mul, acc[nt][2 * half + 1] * mul);
    }
}

// ======================================================================================================================
// The kernels: the streamed tiles are double-buffered with cp.async (the next key / query block lands while this one is
// computed); the resident operand's A fragments are re-read from shared memory per k-step instead of living in 32 registers
// and the additive mask / bias come from (padded) shared-memory tables, so that three CTAs (12 warps) fit per SM.
// ======================================================================================================================
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// asynchronous version of load_tile (rows >= nrows are zero-filled through src-size 0)
__device__ __forceinline__ void load_tile_async(uint32_t tile, const uint16_t* base, int64_t ld, int col, int64_t row_base,
                                                int r0, int nrows) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int idx = it * THREADS + static_cast<int>(threadIdx.x);
        const int row = idx >> 3, chunk = idx & 7;
        const bool ok = r0 + row < nrows;
        const uint16_t* src = base + (row_base + (ok ? r0 + row : 0)) * ld + col + chunk * 8;
        cp_async16(tile + tile_off(row, chunk), src, ok ? 16 : 0);
    }
}

// acc (16 x 64) += A(rows row0.. of a_tile, 16 x 64 over d) . T^T with the A fragments read per k-step
template <bool kBF16>
__device__ __forceinline__ void mma_rows_tileT(float (&acc)[8][4], uint32_t a_tile, int row0, uint32_t b_tile, int lane) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        uint32_t a[4];
        ldsm_x4(a, a_tile + tile_off(row0 + (lane & 15), ks * 2 + (lane >> 4)));
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            uint32_t b[4];
            ldsm_x4(b, b_tile + tile_off(np * 16 + (lane & 7) + ((lane >> 4) << 3), ks * 2 + ((lane >> 3) & 1)));
            mma16816<kBF16>(acc[2 * np], a, b[0], b[1]);
            mma16816<kBF16>(acc[2 * np + 1], a, b[2], b[3]);
        }
    }
}

constexpr int BIAS_PAD = 64;   // zero entries on both sides of the shared bias table: offsets of padding rows / keys stay in range

template <bool kBF16>
__global__ void __launch_bounds__(THREADS, 3)
attn_bwd_dq2_kernel(const Params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int ntab = p.Lq + p.Lk - 1;
    // sQ | sdO | sK[2] | sV[2] | dS staging tile (dbias only) | mask_s[2][64] | bias (padded) | dbias
    uint32_t* stage = reinterpret_cast<uint32_t*>(smem + 6 * TILE_BYTES);                  // [64][32] packed 16-bit pairs
    float* mask_s = reinterpret_cast<float*>(smem + 7 * TILE_BYTES);                       // [2][64]
    float* bias_s = p.bias_delta ? mask_s + 2 * BN : nullptr;                              // [ntab + 2 * BIAS_PAD]
    float* dbias_s = p.dbias ? mask_s + 2 * BN + (p.bias_delta ? ntab + 2 * BIAS_PAD : 0) : nullptr;

    const int nqb = (p.Lq + BM - 1) / BM;
    const int chunk = static_cast<int>(blockIdx.x) % p.key_chunks;
    const int item = static_cast<int>(blockIdx.x) / p.key_chunks;
    const int qb = item % nqb;
    const int h = (item / nqb) % p.H;
    const int b = item / (nqb * p.H);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int q0 = qb * BM;
    const int nkb = (p.Lk + BN - 1) / BN;
    const SegRows seg = segment_rows(p, b, nkb);
    if (q0 >= seg.nq) return;                  // a dropped query tile of a packed segment
    const int64_t qrow_base = seg.q0, krow_base = seg.k0;
    const float* mask_row = p.add_mask ? p.add_mask + static_cast<int64_t>(b) * p.Lk : nullptr;

    if (bias_s)
        for (int x = threadIdx.x; x < ntab + 2 * BIAS_PAD; x += THREADS) {
            const int d = x - BIAS_PAD;
            bias_s[x] = (d >= 0 && d < ntab) ? __ldg(p.bias_delta + static_cast<int64_t>(h) * ntab + d) : 0.f;
        }
    if (dbias_s)
        for (int x = threadIdx.x; x < ntab; x += THREADS) dbias_s[x] = 0.f;
    const uint32_t smem_a = ab::smem_u32(smem);
    const uint32_t sQ_a = smem_a, sdO_a = smem_a + TILE_BYTES;
    load_tile(smem, p.q, p.ldq, p.q_col0 + h * D, qrow_base, q0, seg.nq);
    load_tile(smem + TILE_BYTES, p.dout, p.lddo, h * D, qrow_base, q0, seg.nq);

    float drow[2];
    {
        const int r = q0 + warp * 16 + (lane >> 1);
        float acc = 0.f;
        if (r < seg.nq) {
            const uint16_t* po = p.o + (qrow_base + r) * p.ldo + h * D + (lane & 1) * 32;
            const uint16_t* pd = p.dout + (qrow_base + r) * p.lddo + h * D + (lane & 1) * 32;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const uint4 a = __ldg(reinterpret_cast<const uint4*>(po) + c);
                const uint4 d = __ldg(reinterpret_cast<const uint4*>(pd) + c);
                const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    acc = fmaf(to_f32<kBF16>(aw[e] & 0xFFFFu), to_f32<kBF16>(dw[e] & 0xFFFFu), acc);
                    acc = fmaf(to_f32<kBF16>(aw[e] >> 16), to_f32<kBF16>(dw[e] >> 16), acc);
                }
            }
        }
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        drow[0] = __shfl_sync(0xffffffffu, acc, 2 * g);
        drow[1] = __shfl_sync(0xffffffffu, acc, 2 * (g + 8));
        if ((lane & 1) == 0 && r < seg.nq) p.dsum[(static_cast<int64_t>(b) * p.H + h) * p.Lq + r] = acc;
    }
    const int i_lo = q0 + warp * 16 + g;
    float lse[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int i = i_lo + r * 8;
        lse[r] = i < seg.nq ? __ldg(p.lse + (static_cast<int64_t>(b) * p.H + h) * p.Lq + i) : INFINITY;
    }
    const int per_chunk = (nkb + p.key_chunks - 1) / p.key_chunks;
    const int kb_begin = chunk * per_chunk;
    const int kb_end = min(nkb, kb_begin + per_chunk);

    auto prefetch = [&](int kb, int buf) {
        load_tile_async(smem_a + (2 + buf) * TILE_BYTES, p.k, p.ldk, p.k_col0 + h * D, krow_base, kb * BN, seg.nk);
        load_tile_async(smem_a + (4 + buf) * TILE_BYTES, p.v, p.ldv, p.v_col0 + h * D, krow_base, kb * BN, seg.nk);
        if (threadIdx.x < BN) {
            const int j = kb * BN + static_cast<int>(threadIdx.x);
            mask_s[buf * BN + threadIdx.x] = (mask_row != nullptr && j < p.Lk) ? __ldg(mask_row + j) : 0.f;
        }
        cp_async_commit();
    };
    // key blocks whose keys are all masked out contribute dS = 0 exactly: walk the live ones only
    const uint8_t* live_row = p.blk_live ? p.blk_live + static_cast<int64_t>(b) * nkb : nullptr;
    auto next_live = [&](int kb) {
        while (kb < kb_end && live_row != nullptr && __ldg(live_row + kb) == 0) ++kb;
        return kb;
    };
    int kb_cur = next_live(kb_begin);
    if (kb_cur < kb_end) prefetch(kb_cur, 0);

    float dqacc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) dqacc[nt][e] = 0.f;
    const float* bias_c = bias_s ? bias_s + BIAS_PAD : nullptr;
    for (int nblk = 0; kb_cur < kb_end; ++nblk) {
        const int kb = kb_cur;
        const int buf = nblk & 1;
        cp_async_wait_all();
        __syncthreads();                       // this block's tiles are visible; everyone is done with the other buffer
        kb_cur = next_live(kb + 1);
        if (kb_cur < kb_end) prefetch(kb_cur, buf ^ 1);
        const uint32_t sK_a = smem_a + (2 + buf) * TILE_BYTES, sV_a = smem_a + (4 + buf) * TILE_BYTES;
        float acc[8][4], dp[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                acc[nt][e] = 0.f;
                dp[nt][e] = 0.f;
            }
        mma_rows_tileT<kBF16>(acc, sQ_a, warp * 16, sK_a, lane);
        mma_rows_tileT<kBF16>(dp, sdO_a, warp * 16, sV_a, lane);
        const int base = kb * BN + 2 * t - i_lo + p.Lq - 1;      // table offset of (row i_lo, column 2t of this block)
        const float* mk = mask_s + buf * BN + 2 * t;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int half = e >> 1, e2 = e & 1;
                const int i = i_lo + half * 8, j = kb * BN + nt * 8 + 2 * t + e2;
                const int off = base + 8 * (nt - half) + e2;
                float sc = acc[nt][e] * p.scale + mk[nt * 8 + e2];
                if (bias_c != nullptr) sc += bias_c[off];
                if (p.causal_value != 0.f && j > min(i, p.Lq - 1)) sc += p.causal_value;
                if (j >= p.Lk) sc = -INFINITY;
                const float pr = __expf(sc - lse[half]);
                acc[nt][e] = pr;
            }
        if (p.drop.thr16 != 0u) {
            // dropout of the forward: dP reaches the softmax only through the kept probabilities, scaled by 1 / (1 - p).
            // One Philox call = this thread's eight elements of one row and 32-key group (csrc/dropout.cuh).
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const uint64_t R = (static_cast<uint64_t>(b) * p.H + h) * p.Lq + min(i_lo + half * 8, p.Lq - 1);
#pragma unroll
                for (int grp = 0; grp < 2; ++grp) {
                    uint32_t w[4];
                    abdrop::attn_words(p.drop, R, static_cast<uint32_t>(kb * 2 + grp), static_cast<uint32_t>(t), w);
#pragma unroll
                    for (int tw = 0; tw < 4; ++tw) {
                        const int nt = grp * 4 + tw;
                        dp[nt][2 * half] = abdrop::keep_lo(p.drop, w[tw]) ? dp[nt][2 * half] * p.drop.inv_keep : 0.f;
                        dp[nt][2 * half + 1] = abdrop::keep_hi(p.drop, w[tw]) ? dp[nt][2 * half + 1] * p.drop.inv_keep : 0.f;
                    }
                }
            }
        }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[nt][e] *= dp[nt][e] - drow[e >> 1];   // dS (0 for padding rows / keys: pr = 0)
        if (dbias_s != nullptr) {
            // dbias[h, j - i] += dS[i, j]: the 64 x 64 dS tile (16-bit, as the MMAs below consume it) goes through a
            // rotated shared tile, then thread d sums diagonal d - 63 and owns one table entry - no atomics.
            // word(r, c / 2) = r * 32 + ((c / 2 + 4 r) & 31): conflict-free for the fragment stores and the diagonal reads
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const int r = warp * 16 + g + half * 8;
                    stage[r * 32 + ((nt * 4 + t + 4 * r) & 31)] = ab::pack2_rn<kBF16>(acc[nt][2 * half], acc[nt][2 * half + 1]);
                }
            __syncthreads();
            const int dl = static_cast<int>(threadIdx.x) - 63;          // diagonal c - r in [-63, 63]
            if (dl <= 63) {
                float sum = 0.f;
                const int r_lo = dl < 0 ? -dl : 0, r_hi = dl > 0 ? 63 - dl : 63;
                for (int r = r_lo; r <= r_hi; ++r) {
                    const int c = r + dl;
                    const uint32_t w = stage[r * 32 + (((c >> 1) + 4 * r) & 31)];
                    sum += to_f32<kBF16>((c & 1) ? (w >> 16) : (w & 0xFFFFu));
                }
                const int idx = kb * BN - q0 + dl + p.Lq - 1;
                if (idx >= 0 && idx < ntab) dbias_s[idx] += sum;       // one owner per entry within a tile
            }
        }
        mma_p_tile<kBF16>(dqacc, acc, sK_a, lane);
    }
    if (p.dq_accum != nullptr) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int i = i_lo + half * 8;
            if (i >= p.Lq) continue;
            float* row = p.dq_accum + (qrow_base + i) * (static_cast<int64_t>(p.H) * D) + h * D;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                atomicAdd(row + nt * 8 + 2 * t, dqacc[nt][2 * half] * p.scale);
                atomicAdd(row + nt * 8 + 2 * t + 1, dqacc[nt][2 * half + 1] * p.scale);
            }
        }
    } else {
        store_acc<kBF16>(dqacc, p.scale, p.dq, p.lddq, p.dq_col0 + h * D, qrow_base, q0 + warp * 16, seg.nq, lane);
    }
    if (dbias_s != nullptr) {
        __syncthreads();
        for (int x = threadIdx.x; x < ntab; x += THREADS) {
            const float v = dbias_s[x];
            if (v != 0.f) atomicAdd(p.dbias + static_cast<int64_t>(h) * ntab + x, v);
        }
    }
}

template <bool kBF16>
__global__ void __launch_bounds__(THREADS, 3)
attn_bwd_dkv2_kernel(const Params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    // sK | sV | sQ[2] | sdO[2] | lse_s[2][64] | d_s[2][64] | bias (padded)
    const int ntab = p.Lq + p.Lk - 1;
    float* lse_s = reinterpret_cast<float*>(smem + 6 * TILE_BYTES);
    float* d_s = lse_s + 2 * BN;
    float* bias_s = p.bias_delta ? d_s + 2 * BN : nullptr;

    const int nkb = (p.Lk + BM - 1) / BM;
    const int kb = static_cast<int>(blockIdx.x) % nkb;
    const int h = (static_cast<int>(blockIdx.x) / nkb) % p.H;
    const int b = static_cast<int>(blockIdx.x) / (nkb * p.H);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int k0 = kb * BM;
    const SegRows seg = segment_rows(p, b, nkb);
    if (k0 >= seg.nk) return;                  // a dropped key tile of a packed segment
    const int64_t qrow_base = seg.q0, krow_base = seg.k0;
    const float* lse_g = p.lse + (static_cast<int64_t>(b) * p.H + h) * p.Lq;
    const float* d_g = p.dsum + (static_cast<int64_t>(b) * p.H + h) * p.Lq;

    if (p.blk_live != nullptr && __ldg(p.blk_live + static_cast<int64_t>(b) * nkb + kb) == 0) {
        // every key of this block is masked out: P = 0 exactly, so dK = dV = 0 (what the full computation would store)
        const int r = k0 + (static_cast<int>(threadIdx.x) >> 1), c0 = (static_cast<int>(threadIdx.x) & 1) * 32;
        if (r < p.Lk) {
            uint4* dkp = reinterpret_cast<uint4*>(p.dk + (krow_base + r) * p.lddk + p.dk_col0 + h * D + c0);
            uint4* dvp = reinterpret_cast<uint4*>(p.dv + (krow_base + r) * p.lddv + p.dv_col0 + h * D + c0);
#pragma unroll
            for (int v4 = 0; v4 < 4; ++v4) {
                dkp[v4] = make_uint4(0u, 0u, 0u, 0u);
                dvp[v4] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        return;
    }

    if (bias_s)
        for (int x = threadIdx.x; x < ntab + 2 * BIAS_PAD; x += THREADS) {
            const int d = x - BIAS_PAD;
            bias_s[x] = (d >= 0 && d < ntab) ? __ldg(p.bias_delta + static_cast<int64_t>(h) * ntab + d) : 0.f;
        }
    const uint32_t smem_a = ab::smem_u32(smem);
    const uint32_t sK_a = smem_a, sV_a = smem_a + TILE_BYTES;
    load_tile(smem, p.k, p.ldk, p.k_col0 + h * D, krow_base, k0, seg.nk);
    load_tile(smem + TILE_BYTES, p.v, p.ldv, p.v_col0 + h * D, krow_base, k0, seg.nk);

    const int j_lo = k0 + warp * 16 + g;
    float mk[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int j = j_lo + r * 8;
        mk[r] = (p.add_mask != nullptr && j < p.Lk) ? __ldg(p.add_mask + static_cast<int64_t>(b) * p.Lk + j) : 0.f;
    }
    const int nqb = (seg.nq + BN - 1) / BN;
    auto prefetch = [&](int qb, int buf) {
        load_tile_async(smem_a + (2 + buf) * TILE_BYTES, p.q, p.ldq, p.q_col0 + h * D, qrow_base, qb * BN, seg.nq);
        load_tile_async(smem_a + (4 + buf) * TILE_BYTES, p.dout, p.lddo, h * D, qrow_base, qb * BN, seg.nq);
        if (threadIdx.x < BN) {
            const int i = qb * BN + static_cast<int>(threadIdx.x);
            lse_s[buf * BN + threadIdx.x] = i < seg.nq ? __ldg(lse_g + i) : INFINITY;
            d_s[buf * BN + threadIdx.x] = i < seg.nq ? __ldg(d_g + i) : 0.f;
        }
        cp_async_commit();
    };
    prefetch(0, 0);

    float dkacc[8][4], dvacc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            dkacc[nt][e] = 0.f;
            dvacc[nt][e] = 0.f;
        }
    const float* bias_c = bias_s ? bias_s + BIAS_PAD : nullptr;
    for (int qb = 0; qb < nqb; ++qb) {
        const int buf = qb & 1;
        cp_async_wait_all();
        __syncthreads();
        if (qb + 1 < nqb) prefetch(qb + 1, buf ^ 1);
        const uint32_t sQ_a = smem_a + (2 + buf) * TILE_BYTES, sdO_a = smem_a + (4 + buf) * TILE_BYTES;
        float acc[8][4], dp[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                acc[nt][e] = 0.f;
                dp[nt][e] = 0.f;
            }
        mma_rows_tileT<kBF16>(acc, sK_a, warp * 16, sQ_a, lane);      // S^T  = K Q^T
        mma_rows_tileT<kBF16>(dp, sV_a, warp * 16, sdO_a, lane);      // dP^T = V dO^T
        const int base = j_lo - (qb * BN + 2 * t) + p.Lq - 1;         // table offset of (key j_lo, query column 2t)
        const float* ls = lse_s + buf * BN + 2 * t;
        const float* dd = d_s + buf * BN + 2 * t;
        const bool hi_word = ((j_lo & 31) >> 3) != 0;                 // j_lo % 32 in [0, 8) or [16, 24): words (0, 1) or (2, 3)
        const uint32_t jsh = static_cast<uint32_t>(j_lo & 1) * 16u;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            // the forward's dropout mask at (query i, key j): word (j % 32) / 8 of call (R(i), j / 32, (j % 8) / 2); the two
            // key rows of this thread (j_lo, j_lo + 8) share the call, the two query columns (e2) need one call each
            uint32_t u16[2][2] = {{0xFFFFu, 0xFFFFu}, {0xFFFFu, 0xFFFFu}};   // [half][e2]
            if (p.drop.thr16 != 0u) {
#pragma unroll
                for (int e2 = 0; e2 < 2; ++e2) {
                    const int i = qb * BN + nt * 8 + 2 * t + e2;
                    const uint64_t R = (static_cast<uint64_t>(b) * p.H + h) * p.Lq + min(i, p.Lq - 1);
                    uint32_t w[4];
                    abdrop::attn_words(p.drop, R, static_cast<uint32_t>(j_lo >> 5), static_cast<uint32_t>((j_lo & 7) >> 1), w);
                    u16[0][e2] = ((hi_word ? w[2] : w[0]) >> jsh) & 0xFFFFu;
                    u16[1][e2] = ((hi_word ? w[3] : w[1]) >> jsh) & 0xFFFFu;
                }
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int half = e >> 1, e2 = e & 1;
                const int j = j_lo + half * 8, i = qb * BN + nt * 8 + 2 * t + e2;
                float sc = acc[nt][e] * p.scale + mk[half];
                if (bias_c != nullptr) sc += bias_c[base + 8 * (half - nt) - e2];
                if (p.causal_value != 0.f && j > min(i, p.Lq - 1)) sc += p.causal_value;
                if (j >= p.Lk) sc = -INFINITY;
                const float pr = __expf(sc - ls[nt * 8 + e2]);
                const float km = (u16[half][e2] >= p.drop.thr16) ? p.drop.inv_keep : 0.f;   // thr16 == 0: always 1
                acc[nt][e] = pr * km;                              // dropped probabilities: dV = Pd^T dO
                dp[nt][e] = pr * (dp[nt][e] * km - dd[nt * 8 + e2]);
            }
        }
        mma_p_tile<kBF16>(dvacc, acc, sdO_a, lane);   // dV += P^T dO
        mma_p_tile<kBF16>(dkacc, dp, sQ_a, lane);     // dK += dS^T Q
    }
    store_acc<kBF16>(dkacc, p.scale, p.dk, p.lddk, p.dk_col0 + h * D, krow_base, k0 + warp * 16, seg.nk, lane);
    store_acc<kBF16>(dvacc, 1.0f, p.dv, p.lddv, p.dv_col0 + h * D, krow_base, k0 + warp * 16, seg.nk, lane);
}

// The two kernels of one backward on p (nq_ctas / nk_ctas CTAs), with their shared memory for its bias tables
static int launch_bwd(const Params& p, const int64_t nq_ctas, const int64_t nk_ctas, const int32_t is_bf16, cudaStream_t s) {
    const int64_t ntab = static_cast<int64_t>(p.Lq) + p.Lk - 1;
    const int smem_dq = 7 * TILE_BYTES + 2 * BN * 4 +
                        static_cast<int>(((p.bias_delta ? ntab + 2 * BIAS_PAD : 0) + (p.dbias ? ntab : 0)) * 4);
    const int smem_dkv = 6 * TILE_BYTES + 4 * BN * 4 + static_cast<int>((p.bias_delta ? ntab + 2 * BIAS_PAD : 0) * 4);
    constexpr int SMEM_MAX = 7 * TILE_BYTES + 4 * BN * 4 + 2 * (8192 + 2 * BIAS_PAD) * 4;
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dq2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
        AB_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dq2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
        AB_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dkv2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
        AB_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dkv2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
        attr_set = true;
    }
    if (is_bf16) {
        attn_bwd_dq2_kernel<true><<<static_cast<unsigned>(nq_ctas), THREADS, smem_dq, s>>>(p);
        attn_bwd_dkv2_kernel<true><<<static_cast<unsigned>(nk_ctas), THREADS, smem_dkv, s>>>(p);
    } else {
        attn_bwd_dq2_kernel<false><<<static_cast<unsigned>(nq_ctas), THREADS, smem_dq, s>>>(p);
        attn_bwd_dkv2_kernel<false><<<static_cast<unsigned>(nk_ctas), THREADS, smem_dkv, s>>>(p);
    }
    return ATLAS_B200_OK;
}

}  // namespace attnb


extern "C" {

int atlas_b200_attention_bwd_train(const void* q, int64_t ldq, int32_t q_col0, const void* k, int64_t ldk, int32_t k_col0,
                                   const void* v, int64_t ldv, int32_t v_col0, const void* out, int64_t ldo,
                                   const void* dout, int64_t lddo, void* dq, int64_t lddq, int32_t dq_col0, void* dk,
                                   int64_t lddk, int32_t dk_col0, void* dv, int64_t lddv, int32_t dv_col0,
                                   const float* add_mask, const float* bias_delta, float* dbias_delta, float* lse,
                                   float* dsum, float* dq_accum, int32_t B, int32_t H, int32_t Lq, int32_t Lk, float scale,
                                   float causal_value, float dropout_p, uint64_t seed, uint64_t offset,
                                   const uint8_t* key_block_live, int32_t is_bf16, void* stream) {
    using namespace attnb;
    AB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention_bwd: need 0 <= dropout_p < 1 (got %f)", dropout_p);
    const abdrop::Key drop = abdrop::make_key(dropout_p, seed, offset);
    AB_REQUIRE(dq_accum == nullptr || dbias_delta == nullptr,
               "attention_bwd: dq_accum (keys split over CTAs) cannot be combined with dbias_delta");
    AB_REQUIRE(B >= 0 && H > 0 && Lq > 0 && Lk > 0, "attention_bwd: bad shape B=%d H=%d Lq=%d Lk=%d", B, H, Lq, Lk);
    AB_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                   lddk % 8 == 0 && lddv % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 && v_col0 % 8 == 0 &&
                   dq_col0 % 8 == 0 && dk_col0 % 8 == 0 && dv_col0 % 8 == 0,
               "attention_bwd: strides and column offsets must be multiples of 8 elements");
    AB_REQUIRE(lse != nullptr && dsum != nullptr,
               "attention_bwd: lse (the forward's log-sum-exp) and dsum ([B, H, Lq] fp32 each) are required");
    AB_REQUIRE(dbias_delta == nullptr || bias_delta != nullptr, "attention_bwd: dbias_delta without bias_delta");
    const int64_t ntab = static_cast<int64_t>(Lq) + Lk - 1;
    AB_REQUIRE(bias_delta == nullptr || ntab <= 8192, "attention_bwd: Lq + Lk - 1 = %lld exceeds the bias table (8192)",
               static_cast<long long>(ntab));
    if (B == 0) return ATLAS_B200_OK;
    // split the keys of a long, few-query attention (FiD cross-attention: 32 queries x 15 360 keys) over enough CTAs to
    // fill the GPU; each CTA keeps >= 4 key blocks so the atomics stay a small part of its work
    int key_chunks = 1;
    if (dq_accum != nullptr) {
        const int nkb = (Lk + BN - 1) / BN;
        const int64_t base = static_cast<int64_t>(B) * H * ((Lq + BM - 1) / BM);
        const int64_t want = (2ll * abh::num_sms() + base - 1) / base;
        key_chunks = static_cast<int>(want < 1 ? 1 : (want > (nkb + 3) / 4 ? (nkb + 3) / 4 : want));
        if (key_chunks < 1) key_chunks = 1;
    }
    const int64_t nq_ctas = static_cast<int64_t>(B) * H * ((Lq + BM - 1) / BM) * key_chunks;
    const int64_t nk_ctas = static_cast<int64_t>(B) * H * ((Lk + BM - 1) / BM);
    AB_REQUIRE(nq_ctas < (1ll << 31) && nk_ctas < (1ll << 31), "attention_bwd: grid too large");
    Params p;
    p.q = static_cast<const uint16_t*>(q);
    p.k = static_cast<const uint16_t*>(k);
    p.v = static_cast<const uint16_t*>(v);
    p.o = static_cast<const uint16_t*>(out);
    p.dout = static_cast<const uint16_t*>(dout);
    p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo; p.lddo = lddo;
    p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
    p.dq = static_cast<uint16_t*>(dq);
    p.dk = static_cast<uint16_t*>(dk);
    p.dv = static_cast<uint16_t*>(dv);
    p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
    p.dq_col0 = dq_col0; p.dk_col0 = dk_col0; p.dv_col0 = dv_col0;
    p.add_mask = add_mask;
    p.bias_delta = bias_delta;
    p.dbias = dbias_delta;
    p.lse = lse;
    p.dsum = dsum;
    p.dq_accum = dq_accum;
    p.key_chunks = key_chunks;
    p.B = B; p.H = H; p.Lq = Lq; p.Lk = Lk;
    p.scale = scale;
    p.causal_value = causal_value;
    p.drop = drop;
    p.blk_live = key_block_live;
    p.tile_off = nullptr;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    abh::prof_begin(s, abh::PROF_ATTENTION_BWD);
    const int lrc = launch_bwd(p, nq_ctas, nk_ctas, is_bf16, s);
    if (lrc) return lrc;
    abh::prof_end(s, abh::PROF_ATTENTION_BWD, 16.0 * B * H * static_cast<double>(Lq) * Lk * D);
    abh::count_launch(2);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

// Backward of atlas_b200_attention_packed with lse_out (self-attention on the packed rows of the padding-compacted encoder):
// qkv / dqkv hold q | k | v and dq | dk | dv at columns 0, 64 H and 128 H of [rows, >= 192 H] buffers; out / dout [rows, 64 H].
// lse and dsum are [B, H, L] in the padded layout; dbias_delta [H, 2L - 1] is incremented.
int atlas_b200_attention_packed_bwd(const void* qkv, int64_t ld, const void* out, int64_t ldo, const void* dout, int64_t lddo,
                                    void* dqkv, int64_t ldd, const float* add_mask, const float* bias_delta, float* dbias_delta,
                                    const float* lse, float* dsum, const uint8_t* keep, const int32_t* tile_off, int32_t B,
                                    int32_t H, int32_t L, float scale, float dropout_p, uint64_t seed, uint64_t offset,
                                    int32_t is_bf16, void* stream) {
    using namespace attnb;
    AB_REQUIRE(B > 0 && H > 0 && L > 0 && L % 64 == 0 && L <= 576 && keep != nullptr && tile_off != nullptr,
               "attention_packed_bwd: 0 < L <= 576, L %% 64 == 0 and the segment tables are required (got L=%d)", L);
    AB_REQUIRE(lse != nullptr && dsum != nullptr,
               "attention_packed_bwd: lse (the forward's log-sum-exp) and dsum ([B, H, L] fp32 each) are required");
    AB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention_packed_bwd: need 0 <= dropout_p < 1 (got %f)", dropout_p);
    AB_REQUIRE(ld % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && ldd % 8 == 0,
               "attention_packed_bwd: strides must be multiples of 8 elements");
    AB_REQUIRE(dbias_delta == nullptr || bias_delta != nullptr, "attention_packed_bwd: dbias_delta without bias_delta");
    AB_REQUIRE(static_cast<int64_t>(B) * L < (1ll << 31) && static_cast<int64_t>(B) * H * (L / 64) < (1ll << 31),
               "attention_packed_bwd: more than 2^31 rows");
    const int nb = L / 64;
    Params p;
    p.q = p.k = p.v = static_cast<const uint16_t*>(qkv);
    p.o = static_cast<const uint16_t*>(out);
    p.dout = static_cast<const uint16_t*>(dout);
    p.ldq = p.ldk = p.ldv = ld;
    p.ldo = ldo;
    p.lddo = lddo;
    p.q_col0 = 0, p.k_col0 = H * D, p.v_col0 = 2 * H * D;
    p.dq = p.dk = p.dv = static_cast<uint16_t*>(dqkv);
    p.lddq = p.lddk = p.lddv = ldd;
    p.dq_col0 = 0, p.dk_col0 = H * D, p.dv_col0 = 2 * H * D;
    p.add_mask = add_mask;
    p.bias_delta = bias_delta;
    p.dbias = dbias_delta;
    p.lse = const_cast<float*>(lse);
    p.dsum = dsum;
    p.dq_accum = nullptr;
    p.key_chunks = 1;
    p.B = B, p.H = H, p.Lq = L, p.Lk = L;
    p.scale = scale;
    p.causal_value = 0.f;
    p.drop = abdrop::make_key(dropout_p, seed, offset);
    p.blk_live = keep;
    p.tile_off = tile_off;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int64_t ctas = static_cast<int64_t>(B) * H * nb;     // per kernel; the CTAs of dropped tiles return at once
    abh::prof_begin(s, abh::PROF_ATTENTION_BWD);
    const int lrc = launch_bwd(p, ctas, ctas, is_bf16, s);
    if (lrc) return lrc;
    abh::prof_end_tile_pairs(s, abh::PROF_ATTENTION_BWD, 16.0 * H * 64.0 * 64.0 * D, keep, B, nb);
    abh::count_launch(2);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
