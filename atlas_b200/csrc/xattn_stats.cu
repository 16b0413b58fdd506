// Cross-attention statistics of the FiD decoder for retriever distillation (`cross_attention_forward`,
// src/fid.py:333-343): per decoder layer, with S = Q K^T + mask and P = softmax_j(S) over the n_ctx * L keys,
//     score_storage            = mean over heads of S                       [B, T, n*L]
//     prob_storage             = mean over heads of P
//     normalized_score_storage = mean over heads of ||V[b, j, h, :]||_2 * P
// The reference materialises S and P ([B, H, T, n*L] each) to take these means; here one pass over the K / V rows
// recomputes the logits against the (tiny) query block, normalises with the log-sum-exp the attention kernel already
// produced, and reduces over heads in registers.  HBM-bound: K and V are read once (2 * B * n*L * H*64 * 2 bytes), the
// three [B, T, n*L] fp32 maps are written once.
//
// Block = 32 consecutive keys of one batch element, 8 warps x 4 keys; lane = query position (t = lane + 32 c).
//
// Precision: S and the given lse are fp32, so a key's S carries the rounding of its mask term (up to |mask| * 2^-24).  In a row
// whose keys are ALL masked with -1e9 that rounding (32) swallows the logits, and the fp32 lse loses log(Lk) the same way, so
// P = exp(S - lse) comes out near 1 per key instead of the reference's uniform 1 / Lk.  FiD never builds such a row (every
// passage holds the question tokens); at -1e4 (fp16) a fully masked row keeps about 3 significant digits.
#include "common.cuh"
#include "host_common.h"

#include <math.h>

namespace xs {

constexpr int KEYS = 32;
constexpr int MAXC = 4;   // T <= 128

template <bool kBF16>
__device__ __forceinline__ float f32(uint32_t h) {
    if constexpr (kBF16) return __bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(h & 0xFFFFu)));
    return __half2float(__ushort_as_half(static_cast<unsigned short>(h & 0xFFFFu)));
}

template <bool kBF16>
__global__ void __launch_bounds__(256)
xattn_stats_kernel(const uint16_t* __restrict__ q, int64_t ldq, int q_col0, const uint16_t* __restrict__ kv, int64_t ldkv,
                   int k_col0, int v_col0, const float* __restrict__ add_mask, const float* __restrict__ lse,
                   float* __restrict__ out_s, float* __restrict__ out_p, float* __restrict__ out_n, int H, int T, int Lk,
                   float scale) {
    __shared__ float ks[KEYS][64];
    __shared__ float vnorm[KEYS];
    const int b = blockIdx.y, j0 = blockIdx.x * KEYS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nc = (T + 31) / 32;
    float acc_s[MAXC][4], acc_p[MAXC][4], acc_n[MAXC][4];
#pragma unroll
    for (int c = 0; c < MAXC; ++c)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) acc_s[c][kk] = acc_p[c][kk] = acc_n[c][kk] = 0.f;
    float mk[4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const int j = j0 + warp * 4 + kk;
        mk[kk] = (add_mask != nullptr && j < Lk) ? add_mask[static_cast<int64_t>(b) * Lk + j] : 0.f;
    }
    for (int h = 0; h < H; ++h) {
        __syncthreads();
        {   // K tile -> fp32 smem, ||V row||: thread = (key, 8-element chunk)
            const int key = threadIdx.x >> 3, chunk = threadIdx.x & 7;
            const int j = j0 + key;
            uint4 kq = make_uint4(0, 0, 0, 0), vq = make_uint4(0, 0, 0, 0);
            if (j < Lk) {
                const uint16_t* row = kv + (static_cast<int64_t>(b) * Lk + j) * ldkv + h * 64 + chunk * 8;
                kq = __ldg(reinterpret_cast<const uint4*>(row + k_col0));
                vq = __ldg(reinterpret_cast<const uint4*>(row + v_col0));
            }
            const uint32_t kw[4] = {kq.x, kq.y, kq.z, kq.w}, vw[4] = {vq.x, vq.y, vq.z, vq.w};
            float ss = 0.f;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                ks[key][chunk * 8 + 2 * e] = f32<kBF16>(kw[e]);
                ks[key][chunk * 8 + 2 * e + 1] = f32<kBF16>(kw[e] >> 16);
                const float a = f32<kBF16>(vw[e]), c2 = f32<kBF16>(vw[e] >> 16);
                ss = fmaf(a, a, fmaf(c2, c2, ss));
            }
            ss += __shfl_xor_sync(0xffffffffu, ss, 1);
            ss += __shfl_xor_sync(0xffffffffu, ss, 2);
            ss += __shfl_xor_sync(0xffffffffu, ss, 4);
            if (chunk == 0) vnorm[key] = sqrtf(ss);
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {
            if (c >= nc) break;
            const int t = c * 32 + lane;
            if (t >= T) continue;
            const uint16_t* qrow = q + (static_cast<int64_t>(b) * T + t) * ldq + q_col0 + h * 64;
            float dot[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ch = 0; ch < 8; ++ch) {
                const uint4 qq = __ldg(reinterpret_cast<const uint4*>(qrow) + ch);
                const uint32_t qw[4] = {qq.x, qq.y, qq.z, qq.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float q0 = f32<kBF16>(qw[e]), q1 = f32<kBF16>(qw[e] >> 16);
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)
                        dot[kk] = fmaf(q0, ks[warp * 4 + kk][ch * 8 + 2 * e], fmaf(q1, ks[warp * 4 + kk][ch * 8 + 2 * e + 1], dot[kk]));
                }
            }
            const float l = __ldg(lse + (static_cast<int64_t>(b) * H + h) * T + t);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float s = dot[kk] * scale + mk[kk];
                const float p = __expf(s - l);
                acc_s[c][kk] += s;
                acc_p[c][kk] += p;
                acc_n[c][kk] = fmaf(p, vnorm[warp * 4 + kk], acc_n[c][kk]);
            }
        }
    }
    const float inv = 1.0f / static_cast<float>(H);
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
        if (c >= nc) break;
        const int t = c * 32 + lane;
        if (t >= T) continue;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const int j = j0 + warp * 4 + kk;
            if (j >= Lk) continue;
            const int64_t o = (static_cast<int64_t>(b) * T + t) * Lk + j;
            out_s[o] = acc_s[c][kk] * inv;
            out_p[o] = acc_p[c][kk] * inv;
            out_n[o] = acc_n[c][kk] * inv;
        }
    }
}

}  // namespace xs

extern "C" {

int atlas_b200_cross_attention_stats(const void* q, int64_t ldq, int32_t q_col0, const void* kv, int64_t ldkv,
                                     int32_t k_col0, int32_t v_col0, const float* add_mask, const float* lse,
                                     float* out_scores, float* out_probs, float* out_norms, int32_t B, int32_t H, int32_t T,
                                     int32_t Lk, float scale, int32_t is_bf16, void* stream) {
    AB_REQUIRE(B >= 0 && H > 0 && T > 0 && T <= 32 * xs::MAXC && Lk > 0, "cross_attention_stats: need 0 < T <= %d (T=%d)",
               32 * xs::MAXC, T);
    AB_REQUIRE(ldq % 8 == 0 && ldkv % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 && v_col0 % 8 == 0,
               "cross_attention_stats: strides and column offsets must be multiples of 8 elements");
    AB_REQUIRE(lse != nullptr && out_scores && out_probs && out_norms, "cross_attention_stats: lse and outputs required");
    if (B == 0) return ATLAS_B200_OK;
    AB_REQUIRE(B <= 65535, "cross_attention_stats: batch too large");
    dim3 grid((Lk + xs::KEYS - 1) / xs::KEYS, B);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16)
        xs::xattn_stats_kernel<true><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(q), ldq, q_col0,
                                                          static_cast<const uint16_t*>(kv), ldkv, k_col0, v_col0, add_mask,
                                                          lse, out_scores, out_probs, out_norms, H, T, Lk, scale);
    else
        xs::xattn_stats_kernel<false><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(q), ldq, q_col0,
                                                           static_cast<const uint16_t*>(kv), ldkv, k_col0, v_col0, add_mask,
                                                           lse, out_scores, out_probs, out_norms, H, T, Lk, scale);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
