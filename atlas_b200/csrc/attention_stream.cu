// cross_stream_kernel: FiD decoder cross-attention in the teacher-forced / training forward - FEW queries (Lq <= 64: the target
// tokens) against the n_docs x text_maxlength concatenated encoder keys of one batch element (15 360 at BASELINE
// configs[3]); replaces `cross_attention_forward` (src/fid.py:298-349) for that shape, same math as the split-KV path of
// csrc/attention.cu:   partial_c = (un-normalised P_c V_c, row max m_c, row sum l_c) over key chunk c, merged by
// combine_splits_kernel.
//
// Why a second kernel: the operation is a pure K / V STREAM (377 MB per layer and 8 queries, 12 GFLOP: 32 FLOP/B, far left of
// the ridge).  A one-CTA-per-segment kernel treats every 384-key segment as a serial load -> S -> softmax -> P.V chain on a
// 128-row tile of which 32 rows are real: the chain, not the load, sets the segment time.  Here: small CTAs (128 threads,
// 40 KB of shared memory -> 5 per SM), each streaming its key chunk through a
// cp.async double buffer of 64-key K / V tiles, flash-attention style online softmax on warp-level mma.sync fragments (the
// arithmetic is 1 / 6 of what the HBM time allows, so the legacy tensor-core path is the right tool: many
// independent CTAs per SM hide each other's latencies).
// Bound: HBM.  Algorithmic bytes per launch = B x Lk x 2 x H x 64 x 2 (K and V once) + the fp32 partials.
//
// <kFP8> (beam-search decode over the e4m3 cross K|V cache of csrc/kv_fp8.cu): the 64 x 64-byte code tiles stream through the
// same cp.async double buffer, are converted to the run's 16-bit type WITHOUT their scales (every e4m3 value is exact in fp16
// and bf16) into one 16-bit K / V tile pair, and the mma.sync path is unchanged: kscale multiplies each column of S, vscale
// is folded into P before P is rounded to 16 bits (fp16: times 256, undone on the fp32 output, so that small p * vscale do
// not fall into fp16's subnormal range).  0.53x the K|V bytes.
#include "common.cuh"
#include "host_common.h"
#include "kv_fp8.cuh"

#include <math.h>

namespace xs {

constexpr int D = 64;
constexpr int BQ = 64;         // query rows per CTA (>= Lq; 4 warps x 16 rows)
constexpr int BN = 64;         // keys per streamed tile
constexpr int THREADS = 128;
constexpr int TILE_BYTES = 64 * 128;
constexpr int SMEM_BYTES = 5 * TILE_BYTES + 2 * BN * 4;      // Q | K[2] | V[2] | mask[2][64]
// e4m3: Q | K | V (16-bit) | (K8 | V8)[2] codes (4 KB each) | mask[2][64] | kscale[2][64] | vscale[2][64]
constexpr int TILE8_BYTES = 64 * 64;
constexpr int SMEM8_BYTES = 3 * TILE_BYTES + 4 * TILE8_BYTES + 6 * BN * 4;
constexpr float LOG2E = 1.4426950408889634f;

struct Params {
    const uint16_t *q, *kv;
    int64_t ldq, ldkv;
    int q_col0, k_col0, v_col0;
    const float* add_mask;     // [B, Lk] or nullptr
    const uint8_t* tile_live;  // [B, ceil(Lk / 64)] or nullptr: 0 = every key of the 64-key tile is masked out (its
                               // probabilities are exactly 0 in fp32: exp(-10000 + s - max) underflows) -> neither loaded nor
                               // computed.  FiD passages are padded to text_maxlength: ~45 % of the keys at BASELINE configs[3]
    const int32_t* tile_row;   // [B, Lk / 64] or nullptr: kv holds only the LIVE 64-key tiles, compacted; tile t of batch b
                               // starts at row 64 * tile_row[b * (Lk / 64) + t] of kv (atlas_b200_compact_live_tiles)
    float* o_partial;          // [(B * chunks + c) * Lq + i, H * 64] fp32, un-normalised
    float* ml_partial;         // [(B * chunks + c) * Lq + i, H, 2]: (row max, natural log units; row sum)
    int H, Lq, Lk, chunk;
    float scale;
};

__device__ __forceinline__ uint32_t tile_off(int row, int chunk) {
    return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// rows [r0, r0 + 64) of a row-major matrix (columns col .. col + 63) -> swizzled tile; rows >= nrows zero-filled
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
// e4m3: rows [r0, r0 + 64) x 64 code bytes -> plain row-major 64 x 64 B staging tile; rows >= nrows zero-filled
__device__ __forceinline__ void load_tile8_async(uint32_t tile, const uint8_t* base, int64_t ld, int col, int64_t row_base,
                                                 int r0, int nrows) {
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const int idx = it * THREADS + static_cast<int>(threadIdx.x);
        const int row = idx >> 2, chunk = idx & 3;
        const bool ok = r0 + row < nrows;
        const uint8_t* src = base + (row_base + (ok ? r0 + row : 0)) * ld + col + chunk * 16;
        cp_async16(tile + row * 64 + chunk * 16, src, ok ? 16 : 0);
    }
}
// e4m3: staging tile of codes -> the swizzled 16-bit tile the ldmatrix path reads (values unscaled, exact)
template <bool kBF16>
__device__ __forceinline__ void convert_tile8(const uint8_t* stage, uint8_t* tile16) {
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const int idx = it * THREADS + static_cast<int>(threadIdx.x);
        const int row = idx >> 2, chunk = idx & 3;
        const uint4 w = *reinterpret_cast<const uint4*>(stage + row * 64 + chunk * 16);
        const uint32_t u[4] = {w.x, w.y, w.z, w.w};
        uint32_t h[8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const uint32_t h2 = kv8::e4m3x2_to_f16x2(static_cast<uint16_t>(u[i] >> (16 * k)));
                if constexpr (kBF16) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h2));
                    h[2 * i + k] = ab::pack2_rn<true>(f.x, f.y);
                } else {
                    h[2 * i + k] = h2;
                }
            }
        *reinterpret_cast<uint4*>(tile16 + tile_off(row, 2 * chunk)) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(tile16 + tile_off(row, 2 * chunk + 1)) = make_uint4(h[4], h[5], h[6], h[7]);
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
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// grid = (chunks, H, B); CTA = keys [c * chunk, min(Lk, (c + 1) * chunk)) of batch b, head h, all Lq <= 64 queries.
// kFP8: kv8 holds e4m3 codes in place of p.kv (same columns) and kv_scale [B * Lk, ld_scale] their scales (key row j: column
// block k_col0 / 64 + h for K, v_col0 / 64 + h for V); p.tile_row is not supported.  3 CTAs per SM: the scale folds need
// registers past the 128 that 4 allow.
template <bool kBF16, bool kFP8 = false>
__global__ void __launch_bounds__(THREADS, kFP8 ? 3 : 4)
cross_stream_kernel(const Params p, const uint8_t* __restrict__ kv8 = nullptr, const float* __restrict__ kv_scale = nullptr,
                    int64_t ld_scale = 0) {
    extern __shared__ __align__(128) uint8_t smem[];
    float* mask_s = reinterpret_cast<float*>(smem + 5 * TILE_BYTES);        // [2][64], log2 units
    float* ks_s = mask_s + 2 * BN;              // kFP8: [2][64] kscale * scale * log2(e)
    float* vs_s = mask_s + 4 * BN;              // kFP8: [2][64] vscale * PV_BOOST
    constexpr float PV_BOOST = kBF16 ? 1.f : 256.f;
    constexpr int STAGE = 3 * TILE_BYTES;       // kFP8: code staging buffers (K8 | V8) x 2
    const int c = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int chunks = gridDim.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const uint32_t smem_a = ab::smem_u32(smem);
    const uint32_t sQ = smem_a;
    const int64_t qrow_base = static_cast<int64_t>(b) * p.Lq, krow_base = static_cast<int64_t>(b) * p.Lk;
    const int j_begin = c * p.chunk, j_end = min(p.Lk, (c + 1) * p.chunk);
    const int n_all = (j_end - j_begin + BN - 1) / BN;
    const float* mask_row = p.add_mask ? p.add_mask + static_cast<int64_t>(b) * p.Lk : nullptr;
    // the live 64-key tiles of this chunk (uniform over the CTA; chunk <= 64 tiles)
    uint64_t live = n_all >= 64 ? ~0ull : ((1ull << n_all) - 1ull);
    if (p.tile_live != nullptr) {
        const uint8_t* fl = p.tile_live + static_cast<int64_t>(b) * ((p.Lk + BN - 1) / BN) + j_begin / BN;
        uint64_t m = 0;
        for (int i = 0; i < n_all; ++i) m |= static_cast<uint64_t>(__ldg(fl + i) != 0) << i;
        live = m;
    }
    const int n_tiles = __popcll(live);
    // ordinal -> tile index of the chunk
    auto tile_at = [&](int ord) {
        uint64_t m = live;
        for (int i = 0; i < ord; ++i) m &= m - 1;
        return __ffsll(static_cast<long long>(m)) - 1;
    };

    auto prefetch = [&](int ord, int buf) {
        const int j0 = j_begin + tile_at(ord) * BN;
        if constexpr (kFP8) {
            load_tile8_async(smem_a + STAGE + buf * 2 * TILE8_BYTES, kv8, p.ldkv, p.k_col0 + h * D, krow_base, j0, j_end);
            load_tile8_async(smem_a + STAGE + buf * 2 * TILE8_BYTES + TILE8_BYTES, kv8, p.ldkv, p.v_col0 + h * D, krow_base, j0,
                             j_end);
            if (threadIdx.x < BN) {         // a key past the chunk weighs 0 whatever its (possibly NaN) scale
                const int j = j0 + static_cast<int>(threadIdx.x);
                const bool in = j < j_end;
                const float* sr = kv_scale + (krow_base + (in ? j : j_begin)) * ld_scale + p.k_col0 / D + h;
                ks_s[buf * BN + threadIdx.x] = in ? __ldg(sr) * (p.scale * LOG2E) : 0.f;
                vs_s[buf * BN + threadIdx.x] = in ? __ldg(sr + (p.v_col0 - p.k_col0) / D) * PV_BOOST : 0.f;
            }
        } else if (p.tile_row != nullptr) {      // compacted K | V: whole 64-row tiles, addressed through the table
            const int64_t r0 = static_cast<int64_t>(__ldg(p.tile_row + static_cast<int64_t>(b) * (p.Lk / BN) + j0 / BN)) * BN;
            load_tile_async(smem_a + (1 + buf) * TILE_BYTES, p.kv, p.ldkv, p.k_col0 + h * D, r0, 0, BN);
            load_tile_async(smem_a + (3 + buf) * TILE_BYTES, p.kv, p.ldkv, p.v_col0 + h * D, r0, 0, BN);
        } else {
            load_tile_async(smem_a + (1 + buf) * TILE_BYTES, p.kv, p.ldkv, p.k_col0 + h * D, krow_base, j0, j_end);
            load_tile_async(smem_a + (3 + buf) * TILE_BYTES, p.kv, p.ldkv, p.v_col0 + h * D, krow_base, j0, j_end);
        }
        if (threadIdx.x < BN) {
            const int j = j0 + static_cast<int>(threadIdx.x);
            mask_s[buf * BN + threadIdx.x] = j < j_end ? (mask_row ? __ldg(mask_row + j) * LOG2E : 0.f) : -INFINITY;
        }
        cp_async_commit();
    };
    // Q rows (zero-filled past Lq) ride in the first cp.async group together with tile 0
    load_tile_async(sQ, p.q, p.ldq, p.q_col0 + h * D, qrow_base, 0, p.Lq);
    if (n_tiles > 0) prefetch(0, 0);        // a chunk without a live tile writes (0, -inf, 0): weight 0 in the merge
    else cp_async_commit();

    const bool active = warp * 16 < p.Lq;                 // warps whose 16 rows are all padding only help with the loads
    const float scale2 = p.scale * LOG2E;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;

    for (int kt = 0; kt < n_tiles; ++kt) {
        const int buf = kt & 1;
        cp_async_wait_all();
        __syncthreads();                                   // tile kt is visible; everyone is done with the other buffer
        if (kt + 1 < n_tiles) prefetch(kt + 1, buf ^ 1);
        if constexpr (kFP8) {       // codes of tile kt -> the single 16-bit K / V tile pair (free since the barrier above)
            convert_tile8<kBF16>(smem + STAGE + buf * 2 * TILE8_BYTES, smem + TILE_BYTES);
            convert_tile8<kBF16>(smem + STAGE + buf * 2 * TILE8_BYTES + TILE8_BYTES, smem + 2 * TILE_BYTES);
            __syncthreads();
        }
        if (!active) continue;
        const uint32_t sK = smem_a + (kFP8 ? 1 : 1 + buf) * TILE_BYTES, sV = smem_a + (kFP8 ? 2 : 3 + buf) * TILE_BYTES;
        // ---- S = Q K^T (16 x 64 per warp) ----
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) s[nt][e] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            uint32_t a[4];
            ldsm_x4(a, sQ + tile_off(warp * 16 + (lane & 15), ks * 2 + (lane >> 4)));
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t bfr[4];
                ldsm_x4(bfr, sK + tile_off(np * 16 + (lane & 7) + ((lane >> 4) << 3), ks * 2 + ((lane >> 3) & 1)));
                mma16816<kBF16>(s[2 * np], a, bfr[0], bfr[1]);
                mma16816<kBF16>(s[2 * np + 1], a, bfr[2], bfr[3]);
            }
        }
        // ---- online softmax in the log2 domain ----
        const float* mk = mask_s + buf * BN + 2 * t;
        const float* ksp = ks_s + buf * BN + 2 * t;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float v = fmaf(s[nt][e], kFP8 ? ksp[nt * 8 + (e & 1)] : scale2, mk[nt * 8 + (e & 1)]);
                s[nt][e] = v;
                mx[e >> 1] = fmaxf(mx[e >> 1], v);
            }
        float corr[2];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 1));
            mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 2));
            const float m_new = fmaxf(m[hf], mx[hf]);
            corr[hf] = m_new > -INFINITY ? ex2_approx(m[hf] - m_new) : 1.f;
            m[hf] = m_new;
        }
        float rs[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int hf = e >> 1;
                const float pv = m[hf] > -INFINITY ? ex2_approx(s[nt][e] - m[hf]) : 0.f;
                s[nt][e] = pv;
                rs[hf] += pv;
            }
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) l[hf] = l[hf] * corr[hf] + rs[hf];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            o[nt][0] *= corr[0];
            o[nt][1] *= corr[0];
            o[nt][2] *= corr[1];
            o[nt][3] *= corr[1];
        }
        // ---- O += P V: P (accumulator layout) as the A operand, V rows through transposing ldmatrix ----
        const float* vsp = vs_s + buf * BN + 2 * t;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            uint32_t a[4];
            if constexpr (kFP8) {   // P's columns 16 kk + 2t (+1) and 16 kk + 8 + 2t (+1) carry their keys' vscale
                const float v0 = vsp[kk * 16], v1 = vsp[kk * 16 + 1], v8 = vsp[kk * 16 + 8], v9 = vsp[kk * 16 + 9];
                a[0] = ab::pack2_rn<kBF16>(s[2 * kk][0] * v0, s[2 * kk][1] * v1);
                a[1] = ab::pack2_rn<kBF16>(s[2 * kk][2] * v0, s[2 * kk][3] * v1);
                a[2] = ab::pack2_rn<kBF16>(s[2 * kk + 1][0] * v8, s[2 * kk + 1][1] * v9);
                a[3] = ab::pack2_rn<kBF16>(s[2 * kk + 1][2] * v8, s[2 * kk + 1][3] * v9);
            } else {
                a[0] = ab::pack2_rn<kBF16>(s[2 * kk][0], s[2 * kk][1]);
                a[1] = ab::pack2_rn<kBF16>(s[2 * kk][2], s[2 * kk][3]);
                a[2] = ab::pack2_rn<kBF16>(s[2 * kk + 1][0], s[2 * kk + 1][1]);
                a[3] = ab::pack2_rn<kBF16>(s[2 * kk + 1][2], s[2 * kk + 1][3]);
            }
#pragma unroll
            for (int dp = 0; dp < 4; ++dp) {
                uint32_t bfr[4];
                ldsm_x4_t(bfr, sV + tile_off(kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), dp * 2 + (lane >> 4)));
                mma16816<kBF16>(o[2 * dp], a, bfr[0], bfr[1]);
                mma16816<kBF16>(o[2 * dp + 1], a, bfr[2], bfr[3]);
            }
        }
    }
    if (!active) return;
    // ---- partial results of this chunk: un-normalised O, (max, sum) ----
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        l[hf] += __shfl_xor_sync(0xffffffffu, l[hf], 1);
        l[hf] += __shfl_xor_sync(0xffffffffu, l[hf], 2);
        const int i = warp * 16 + g + hf * 8;
        if (i >= p.Lq) continue;
        const int64_t prow = (static_cast<int64_t>(b) * chunks + c) * p.Lq + i;
        float* orow = p.o_partial + prow * (static_cast<int64_t>(p.H) * D) + h * D;
        constexpr float unboost = 1.f / PV_BOOST;   // exact (power of two); 1 outside kFP8
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            if constexpr (kFP8)
                *reinterpret_cast<float2*>(orow + nt * 8 + 2 * t) = make_float2(o[nt][2 * hf] * unboost,
                                                                                o[nt][2 * hf + 1] * unboost);
            else
                *reinterpret_cast<float2*>(orow + nt * 8 + 2 * t) = make_float2(o[nt][2 * hf], o[nt][2 * hf + 1]);
        }
        if (t == 0) {
            float* ml = p.ml_partial + (prow * p.H + h) * 2;
            ml[0] = m[hf] * (1.0f / LOG2E);
            ml[1] = l[hf];
        }
    }
}

}  // namespace xs

extern "C" {

int atlas_b200_cross_attention_stream(const void* q, int64_t ldq, int32_t q_col0, const void* kv, int64_t ldkv, int32_t k_col0,
                                      int32_t v_col0, const float* add_mask, const uint8_t* tile_live, int32_t B, int32_t H,
                                      int32_t Lq, int32_t Lk, int32_t chunk, float scale, float* o_partial, float* ml_partial,
                                      int32_t is_bf16, void* stream) {
    return atlas_b200_cross_attention_stream_compact(q, ldq, q_col0, kv, ldkv, k_col0, v_col0, add_mask, tile_live, nullptr, B, H,
                                                     Lq, Lk, chunk, scale, o_partial, ml_partial, is_bf16, stream);
}

int atlas_b200_cross_attention_stream_compact(const void* q, int64_t ldq, int32_t q_col0, const void* kv, int64_t ldkv,
                                              int32_t k_col0, int32_t v_col0, const float* add_mask, const uint8_t* tile_live,
                                              const int32_t* tile_row, int32_t B, int32_t H, int32_t Lq, int32_t Lk,
                                              int32_t chunk, float scale, float* o_partial, float* ml_partial, int32_t is_bf16,
                                              void* stream) {
    using namespace xs;
    AB_REQUIRE(tile_row == nullptr || (tile_live != nullptr && Lk % BN == 0),
               "cross_attention_stream: compacted K | V needs the live-tile flags and Lk %% 64 == 0");
    AB_REQUIRE(B >= 0 && H > 0 && Lq > 0 && Lq <= BQ && Lk > 0 && chunk > 0 && chunk % BN == 0 && chunk <= 64 * BN,
               "cross_attention_stream: need Lq <= %d and a chunk that is a multiple of %d, <= %d (Lq=%d chunk=%d)", BQ, BN,
               64 * BN, Lq, chunk);
    AB_REQUIRE(ldq % 8 == 0 && ldkv % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 && v_col0 % 8 == 0,
               "cross_attention_stream: strides and column offsets must be multiples of 8 elements");
    AB_REQUIRE(o_partial != nullptr && ml_partial != nullptr, "cross_attention_stream: partial buffers required");
    if (B == 0) return ATLAS_B200_OK;
    const int chunks = (Lk + chunk - 1) / chunk;
    AB_REQUIRE(chunks <= 65535 && H <= 65535 && B <= 65535, "cross_attention_stream: grid too large");
    Params p;
    p.q = static_cast<const uint16_t*>(q);
    p.kv = static_cast<const uint16_t*>(kv);
    p.ldq = ldq, p.ldkv = ldkv;
    p.q_col0 = q_col0, p.k_col0 = k_col0, p.v_col0 = v_col0;
    p.add_mask = add_mask;
    p.tile_live = tile_live;
    p.tile_row = tile_row;
    p.o_partial = o_partial, p.ml_partial = ml_partial;
    p.H = H, p.Lq = Lq, p.Lk = Lk, p.chunk = chunk;
    p.scale = scale;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(cross_stream_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        AB_CUDA_CHECK(cudaFuncSetAttribute(cross_stream_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set = true;
    }
    dim3 grid(chunks, H, B);
    abh::prof_begin(s, abh::PROF_ATTENTION);
    if (is_bf16) cross_stream_kernel<true><<<grid, THREADS, SMEM_BYTES, s>>>(p);
    else cross_stream_kernel<false><<<grid, THREADS, SMEM_BYTES, s>>>(p);
    abh::prof_end(s, abh::PROF_ATTENTION, 4.0 * B * H * static_cast<double>(Lq) * Lk * D);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_cross_attention_stream_e4m3(const void* q, int64_t ldq, int32_t q_col0, const uint8_t* kv8, int64_t ldkv,
                                           const float* kv_scale, int64_t ld_scale, int32_t k_col0, int32_t v_col0,
                                           const float* add_mask, const uint8_t* tile_live, int32_t B, int32_t H, int32_t Lq,
                                           int32_t Lk, int32_t chunk, float scale, float* o_partial, float* ml_partial,
                                           int32_t is_bf16, void* stream) {
    using namespace xs;
    AB_REQUIRE(B >= 0 && H > 0 && Lq > 0 && Lq <= BQ && Lk > 0 && chunk > 0 && chunk % BN == 0 && chunk <= 64 * BN,
               "cross_attention_stream_e4m3: need Lq <= %d and a chunk that is a multiple of %d, <= %d (Lq=%d chunk=%d)", BQ,
               BN, 64 * BN, Lq, chunk);
    AB_REQUIRE(ldq % 8 == 0 && q_col0 % 8 == 0 && ldkv % 16 == 0 && k_col0 % 64 == 0 && v_col0 % 64 == 0 && ld_scale > 0,
               "cross_attention_stream_e4m3: ldq and q_col0 must be multiples of 8 elements, ldkv of 16 bytes, the K and V "
               "column offsets multiples of 64");
    AB_REQUIRE(kv8 != nullptr && kv_scale != nullptr && o_partial != nullptr && ml_partial != nullptr,
               "cross_attention_stream_e4m3: null buffer");
    AB_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(kv8) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(kv_scale) & 3) == 0,
               "cross_attention_stream_e4m3: q and kv8 must be 16-byte aligned (16-byte cp.async)");
    if (B == 0) return ATLAS_B200_OK;
    const int chunks = (Lk + chunk - 1) / chunk;
    AB_REQUIRE(chunks <= 65535 && H <= 65535 && B <= 65535, "cross_attention_stream_e4m3: grid too large");
    Params p;
    p.q = static_cast<const uint16_t*>(q);
    p.kv = nullptr;
    p.ldq = ldq, p.ldkv = ldkv;
    p.q_col0 = q_col0, p.k_col0 = k_col0, p.v_col0 = v_col0;
    p.add_mask = add_mask;
    p.tile_live = tile_live;
    p.tile_row = nullptr;
    p.o_partial = o_partial, p.ml_partial = ml_partial;
    p.H = H, p.Lq = Lq, p.Lk = Lk, p.chunk = chunk;
    p.scale = scale;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(cross_stream_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SMEM8_BYTES));
        AB_CUDA_CHECK(cudaFuncSetAttribute(cross_stream_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SMEM8_BYTES));
        attr_set = true;
    }
    dim3 grid(chunks, H, B);
    abh::prof_begin(s, abh::PROF_ATTENTION);
    if (is_bf16) cross_stream_kernel<true, true><<<grid, THREADS, SMEM8_BYTES, s>>>(p, kv8, kv_scale, ld_scale);
    else cross_stream_kernel<false, true><<<grid, THREADS, SMEM8_BYTES, s>>>(p, kv8, kv_scale, ld_scale);
    abh::prof_end(s, abh::PROF_ATTENTION, 4.0 * B * H * static_cast<double>(Lq) * Lk * D);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
