// Single-token decode attention for `FiD.generate` (reference: src/atlas.py:592-619 -> transformers 4.18 `generate` with
// `use_cache`, T5Attention.forward with past_key_value, src/modeling_t5.py:418-531; FiD cross-attention src/fid.py:298-349).
// One new decoder token per sequence: GEMV-shaped, every K / V byte is used exactly once -> HBM-bound byte work on the
// CUDA cores (no tensor-core tile can help a 1-row query); 16-byte coalesced row reads, fp32 online softmax, warp shuffles.
//
//   decode_cross_attention_kernel   q [B, H*64] against the cached cross K|V rows [B*Lk, 2*H*64] (projected once per
//                                   generation): block = (key chunk, head, batch); emits un-normalised fp32 partials +
//                                   (max, sum) that attn::combine_splits_kernel merges (same identity as the split-KV
//                                   forward).  Algorithmic bytes per (query, layer, step) = Lk * 2 * H*64 * 2 B
//                                   (FiD-base, Lk = 15 360: 47 MB).
//                                   <kFP8>: the same over the e4m3 cross K|V cache of csrc/kv_fp8.cu (0.53x the bytes).
//   decode_self_attention_kernel    appends the new token's K | V to the per-layer cache row t (t read from DEVICE memory so
//                                   the whole step can be replayed from one CUDA graph) and attends over keys 0..t with
//                                   T5's relative-position bias.
#include "common.cuh"
#include "host_common.h"
#include "kv_fp8.cuh"

#include <math.h>

#include <type_traits>

namespace dec {

constexpr int D = 64;
constexpr int CROSS_THREADS = 128;      // 4 warps; a warp reads 4 key rows (4 x 128 B) per instruction
constexpr float LOG2E = 1.4426950408889634f;

template <bool kBF16>
__device__ __forceinline__ void unpack8(const uint4& w, float (&f)[8]) {
    const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if constexpr (kBF16) {
            f[2 * i] = __uint_as_float(u[i] << 16);
            f[2 * i + 1] = __uint_as_float(u[i] & 0xFFFF0000u);
        } else {
            const __half2 h = *reinterpret_cast<const __half2*>(&u[i]);
            const float2 v = __half22float2(h);
            f[2 * i] = v.x;
            f[2 * i + 1] = v.y;
        }
    }
}

// grid = (chunks, H, B); block = 128.  Keys [c*chunk, min(Lk, (c+1)*chunk)) of batch b, head h.
// kFP8: kv holds e4m3 codes (uint8, csrc/kv_fp8.cu) and kv_scale one fp32 scale per (key row, 64-column block): the score
// is kscale_j * (q . k8_j), the value weight p_j * vscale_j.  A lane then reads 16 codes (16 bytes) of a row, 4 lanes per
// row; a warp still covers 16 keys per iteration, so its key group never straddles a 64-key tile either.
template <bool kBF16, bool kFP8 = false>
__global__ void __launch_bounds__(CROSS_THREADS)
decode_cross_attention_kernel(const uint16_t* __restrict__ q, int64_t ldq,
                              const std::conditional_t<kFP8, uint8_t, uint16_t>* __restrict__ kv, int64_t ldkv,
                              int k_col0, int v_col0, const float* __restrict__ add_mask, const uint8_t* __restrict__ tile_live,
                              int Lk, int chunk, float scale, float* __restrict__ o_partial, float* __restrict__ ml_partial,
                              int H, const float* __restrict__ kv_scale = nullptr, int64_t ld_scale = 0) {
    using T = std::conditional_t<kFP8, uint8_t, uint16_t>;
    constexpr int RL = kFP8 ? 4 : 8;    // lanes per key row (16 bytes of K and 16 of V each)
    constexpr int DL = D / RL;          // head dims per lane
    constexpr int ROWS = 32 / RL;       // key rows per warp instruction
    const int c = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int chunks = gridDim.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / RL;          // which of the ROWS key rows of this warp instruction
    const int seg = lane % RL;          // which DL of the 64 head dims
    __shared__ float s_o[CROSS_THREADS / 32][D];
    __shared__ float s_m[CROSS_THREADS / 32], s_l[CROSS_THREADS / 32];

    float qf[DL];
    if constexpr (kFP8) {
#pragma unroll
        for (int i = 0; i < DL / 8; ++i) {
            float f8[8];
            unpack8<kBF16>(*reinterpret_cast<const uint4*>(q + static_cast<int64_t>(b) * ldq + h * D + seg * DL + i * 8), f8);
#pragma unroll
            for (int e = 0; e < 8; ++e) qf[i * 8 + e] = f8[e] * (scale * LOG2E);   // scores in the log2 domain
        }
    } else {
        const uint4 qw = *reinterpret_cast<const uint4*>(q + static_cast<int64_t>(b) * ldq + h * D + seg * 8);
        unpack8<kBF16>(qw, *reinterpret_cast<float(*)[8]>(qf));
#pragma unroll
        for (int e = 0; e < 8; ++e) qf[e] *= scale * LOG2E;          // scores in the log2 domain
    }
    const int j_begin = c * chunk, j_end = min(Lk, (c + 1) * chunk);
    const T* base = kv + (static_cast<int64_t>(b) * Lk) * ldkv + h * D + seg * DL;
    const float* mrow = add_mask ? add_mask + static_cast<int64_t>(b) * Lk : nullptr;
    // kFP8: scale of key row j = sbase[j * ld_scale] (K), sbase[j * ld_scale + (v_col0 - k_col0) / 64] (V)
    const float* sbase = kFP8 ? kv_scale + (static_cast<int64_t>(b) * Lk) * ld_scale + k_col0 / D + h : nullptr;
    const int vs_off = (v_col0 - k_col0) / D;
    // 64-key tiles whose keys are all masked out weigh exactly 0 in the softmax (see atlas_b200_cross_attention_stream): skipped.
    // A warp's 16-key group never straddles a tile (chunk and the group offsets are multiples of 16, tiles of 64).
    const uint8_t* live_row = tile_live ? tile_live + static_cast<int64_t>(b) * ((Lk + 63) / 64) : nullptr;

    float m = -INFINITY, l = 0.f, acc[DL];
#pragma unroll
    for (int e = 0; e < DL; ++e) acc[e] = 0.f;
    constexpr int UNROLL = 16 / ROWS;                                // UNROLL x (K row + V row) 16-byte loads in flight per lane
    for (int j0 = j_begin + warp * ROWS * UNROLL; j0 < j_end; j0 += (CROSS_THREADS / 32) * ROWS * UNROLL) {
        if (live_row != nullptr && __ldg(live_row + (j0 >> 6)) == 0) continue;
        uint4 kw[UNROLL], vw[UNROLL];
        float madd[UNROLL], ksc[UNROLL], vsc[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int j = j0 + u * ROWS + sub;
            const bool ok = j < j_end;
            const T* row = base + static_cast<int64_t>(ok ? j : j_begin) * ldkv;
            kw[u] = *reinterpret_cast<const uint4*>(row + k_col0);
            vw[u] = *reinterpret_cast<const uint4*>(row + v_col0);
            madd[u] = ok ? (mrow ? mrow[j] * LOG2E : 0.f) : -INFINITY;
            if constexpr (kFP8) {           // a key past the chunk weighs 0 whatever its (possibly NaN) scale
                const float* srow = sbase + static_cast<int64_t>(ok ? j : j_begin) * ld_scale;
                ksc[u] = ok ? __ldg(srow) : 0.f;
                vsc[u] = ok ? __ldg(srow + vs_off) : 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            float kf[DL], vf[DL];
            if constexpr (kFP8) {
                kv8::unpack16(kw[u], kf);
                kv8::unpack16(vw[u], vf);
            } else {
                unpack8<kBF16>(kw[u], kf);
                unpack8<kBF16>(vw[u], vf);
            }
            float s = 0.f;
#pragma unroll
            for (int e = 0; e < DL; ++e) s = fmaf(qf[e], kf[e], s);
#pragma unroll
            for (int off = 1; off < RL; off <<= 1) s += __shfl_xor_sync(0xffffffffu, s, off);   // all RL lanes of the row
            if constexpr (kFP8) s *= ksc[u];
            s += madd[u];
            const float m_new = fmaxf(m, s);
            if (m_new > -INFINITY) {
                const float corr = exp2f(m - m_new), p = exp2f(s - m_new);
                l = l * corr + p;
                const float pv = kFP8 ? p * vsc[u] : p;
#pragma unroll
                for (int e = 0; e < DL; ++e) acc[e] = fmaf(acc[e], corr, pv * vf[e]);
                m = m_new;
            }
        }
    }
    // merge the ROWS key rows of the warp (lanes seg, seg+RL, ...), then the warps
#pragma unroll
    for (int off = RL; off < 32; off <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, off), l2 = __shfl_xor_sync(0xffffffffu, l, off);
        const float mn = fmaxf(m, m2);
        const float c1 = mn > -INFINITY ? exp2f(m - mn) : 0.f, c2 = mn > -INFINITY ? exp2f(m2 - mn) : 0.f;
#pragma unroll
        for (int e = 0; e < DL; ++e) {
            const float a2 = __shfl_xor_sync(0xffffffffu, acc[e], off);
            acc[e] = acc[e] * c1 + a2 * c2;
        }
        l = l * c1 + l2 * c2;
        m = mn;
    }
    if (lane < RL) {
#pragma unroll
        for (int e = 0; e < DL; ++e) s_o[warp][lane * DL + e] = acc[e];
        if (lane == 0) s_m[warp] = m, s_l[warp] = l;
    }
    __syncthreads();
    if (threadIdx.x < D) {
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < CROSS_THREADS / 32; ++w) M = fmaxf(M, s_m[w]);
        float o = 0.f, L = 0.f;
#pragma unroll
        for (int w = 0; w < CROSS_THREADS / 32; ++w) {
            const float cw = M > -INFINITY ? exp2f(s_m[w] - M) : 0.f;
            o += cw * s_o[w][threadIdx.x];
            L += cw * s_l[w];
        }
        const int64_t prow = static_cast<int64_t>(b) * chunks + c;
        o_partial[prow * (static_cast<int64_t>(H) * D) + h * D + threadIdx.x] = o;
        if (threadIdx.x == 0) {
            ml_partial[(prow * H + h) * 2] = M * (1.0f / LOG2E);     // natural-log units, as combine_splits_kernel expects
            ml_partial[(prow * H + h) * 2 + 1] = L;
        }
    }
}

// grid = (H, B); block = 64 (thread = head dim).  qkv [B, 3*H*64] = (q | k | v) of the NEW token; cache [B, Tmax, 2*H*64]
// (k | v); step t is read from device memory.  bias_delta [H, 2*Tmax - 1]: entry (j - i) + (Tmax - 1) (nullptr = none).
// kAnc (beam search): anc [2, B, Tmax], buffer (t & 1): key / value j of row b is cache row (anc[b, j], j) instead of (b, j);
// the new token still lands in (b, t) (anc[b, t] == b).  Same arithmetic in the same order as without kAnc.
template <bool kBF16, bool kAnc = false>
__global__ void __launch_bounds__(D)
decode_self_attention_kernel(const uint16_t* __restrict__ qkv, int64_t ldqkv, uint16_t* __restrict__ cache, int Tmax,
                             const int32_t* __restrict__ t_dev, const float* __restrict__ bias_delta, float scale,
                             uint16_t* __restrict__ out, int64_t ldo, int H, const int32_t* __restrict__ anc = nullptr) {
    const int h = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
    const int t = min(max(*t_dev, 0), Tmax - 1);
    const int64_t ldc = static_cast<int64_t>(2) * H * D;
    uint16_t* crow = cache + (static_cast<int64_t>(b) * Tmax) * ldc;
    const int32_t* arow = kAnc ? anc + (static_cast<int64_t>(t & 1) * gridDim.y + b) * Tmax : nullptr;
    auto key_row = [&](int j) -> const uint16_t* {
        if constexpr (kAnc) return cache + (static_cast<int64_t>(__ldg(arow + j)) * Tmax + j) * ldc;
        return crow + static_cast<int64_t>(j) * ldc;
    };
    const uint16_t* tok = qkv + static_cast<int64_t>(b) * ldqkv;
    // append this token's K | V (the reference concatenates past_key_value with the new states, modeling_t5.py:459-470)
    crow[static_cast<int64_t>(t) * ldc + h * D + d] = tok[H * D + h * D + d];
    crow[static_cast<int64_t>(t) * ldc + H * D + h * D + d] = tok[2 * H * D + h * D + d];
    auto ld16 = [](uint16_t v) -> float {
        if constexpr (kBF16) return __uint_as_float(static_cast<uint32_t>(v) << 16);
        return __half2float(__ushort_as_half(v));
    };
    const float qd = ld16(tok[h * D + d]) * scale;
    __shared__ float s_part[2];
    float m = -INFINITY, l = 0.f, acc = 0.f;
    __syncthreads();     // the appended row is visible to the block
    for (int j = 0; j <= t; ++j) {
        const uint16_t* kvrow = key_row(j);
        float s = qd * ld16(kvrow[h * D + d]);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if ((d & 31) == 0) s_part[d >> 5] = s;
        __syncthreads();
        s = s_part[0] + s_part[1];
        __syncthreads();
        if (bias_delta) s += bias_delta[static_cast<int64_t>(h) * (2 * Tmax - 1) + (j - t) + (Tmax - 1)];
        const float m_new = fmaxf(m, s);
        const float corr = __expf(m - m_new), p = __expf(s - m_new);
        l = l * corr + p;
        acc = acc * corr + p * ld16(kvrow[H * D + h * D + d]);
        m = m_new;
    }
    const float o = acc / l;
    uint16_t r;
    if constexpr (kBF16) r = __bfloat16_as_ushort(__float2bfloat16_rn(o));
    else r = __half_as_ushort(__float2half_rn(o));
    out[static_cast<int64_t>(b) * ldo + h * D + d] = r;
}

// (x, i) ranks above (y, j) in torch.argmax's order: NaN above every number, then the larger value; among equal values or
// among NaNs the lower index.  Plain `x > y` would skip NaNs, and an all-NaN row would keep the "no index" sentinel.
__device__ __forceinline__ bool argmax_better(float x, int i, float y, int j) {
    const bool xn = isnan(x), yn = isnan(y);
    if (xn != yn) return xn;
    return x > y || ((xn || x == y) && i < j);
}

// next[b] = done[b] ? pad : argmax_v(logits[b, v] + (v == eos && t + 1 < min_length ? -inf : 0)); seq[b, t + 1] = next;
// done |= next == eos; tok_in[b] = next (the next step's decoder input); t += 1 (thread 0 of block 0).
// grid = B, block = 256.  Same pick as torch.argmax: the first NaN if any, else the lowest index of the maximum.
template <bool kBF16>
__global__ void __launch_bounds__(256)
decode_argmax_kernel(const uint16_t* __restrict__ logits, int64_t ld, int V, int64_t* __restrict__ seq, int64_t ld_seq,
                     int64_t* __restrict__ tok_in, uint8_t* __restrict__ done, int32_t* __restrict__ t_dev, int eos, int pad,
                     int min_length, int B) {
    const int b = blockIdx.x;
    const int t = *t_dev;
    auto ld16 = [](uint16_t v) -> float {
        if constexpr (kBF16) return __uint_as_float(static_cast<uint32_t>(v) << 16);
        return __half2float(__ushort_as_half(v));
    };
    float best = -INFINITY;
    int idx = 0x7fffffff;
    const bool ban_eos = (t + 1) < min_length;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        float x = ld16(logits[static_cast<int64_t>(b) * ld + v]);
        if (ban_eos && v == eos) x = -INFINITY;
        if (argmax_better(x, v, best, idx)) best = x, idx = v;
    }
    __shared__ float s_b[256];
    __shared__ int s_i[256];
    s_b[threadIdx.x] = best;
    s_i[threadIdx.x] = idx;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            const float ob = s_b[threadIdx.x + s];
            const int oi = s_i[threadIdx.x + s];
            if (argmax_better(ob, oi, s_b[threadIdx.x], s_i[threadIdx.x])) s_b[threadIdx.x] = ob, s_i[threadIdx.x] = oi;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int nxt = done[b] ? pad : s_i[0];
        seq[static_cast<int64_t>(b) * ld_seq + t + 1] = nxt;
        tok_in[b] = nxt;
        if (nxt == eos) done[b] = 1;
    }
    // every block read t before any block can have advanced it?  No: blocks are independent - advance in a second kernel
    (void)B;
}

__global__ void advance_step_kernel(int32_t* t_dev) { *t_dev += 1; }

}  // namespace dec

extern "C" {

int atlas_b200_decode_cross_attention_live(const void* q, int64_t ldq, const void* kv, int64_t ldkv, int32_t k_col0,
                                           int32_t v_col0, const float* add_mask, const uint8_t* tile_live, int32_t B,
                                           int32_t H, int32_t Lk, int32_t chunk, float scale, float* o_partial,
                                           float* ml_partial, int32_t is_bf16, void* stream) {
    AB_REQUIRE(B >= 0 && H > 0 && Lk > 0 && chunk > 0 && chunk % 16 == 0, "decode_cross_attention: bad shape");
    AB_REQUIRE(ldq % 8 == 0 && ldkv % 8 == 0 && k_col0 % 8 == 0 && v_col0 % 8 == 0,
               "decode_cross_attention: strides and column offsets must be multiples of 8 elements");
    if (B == 0) return ATLAS_B200_OK;
    const int chunks = (Lk + chunk - 1) / chunk;
    AB_REQUIRE(chunks <= 65535 && H <= 65535 && B <= 65535, "decode_cross_attention: grid too large");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid(chunks, H, B);
    abh::prof_begin(s, abh::PROF_DECODE_CROSS);
    if (is_bf16)
        dec::decode_cross_attention_kernel<true><<<grid, dec::CROSS_THREADS, 0, s>>>(
            static_cast<const uint16_t*>(q), ldq, static_cast<const uint16_t*>(kv), ldkv, k_col0, v_col0, add_mask, tile_live, Lk,
            chunk, scale, o_partial, ml_partial, H);
    else
        dec::decode_cross_attention_kernel<false><<<grid, dec::CROSS_THREADS, 0, s>>>(
            static_cast<const uint16_t*>(q), ldq, static_cast<const uint16_t*>(kv), ldkv, k_col0, v_col0, add_mask, tile_live, Lk,
            chunk, scale, o_partial, ml_partial, H);
    abh::prof_end(s, abh::PROF_DECODE_CROSS, 4.0 * B * H * static_cast<double>(Lk) * dec::D);   // = K | V bytes read
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_decode_cross_attention_e4m3(const void* q, int64_t ldq, const uint8_t* kv8, int64_t ldkv, const float* kv_scale,
                                           int64_t ld_scale, int32_t k_col0, int32_t v_col0, const float* add_mask,
                                           const uint8_t* tile_live, int32_t B, int32_t H, int32_t Lk, int32_t chunk, float scale,
                                           float* o_partial, float* ml_partial, int32_t is_bf16, void* stream) {
    AB_REQUIRE(B >= 0 && H > 0 && Lk > 0 && chunk > 0 && chunk % 16 == 0, "decode_cross_attention_e4m3: bad shape");
    AB_REQUIRE(ldq % 8 == 0 && ldkv % 16 == 0 && k_col0 % 64 == 0 && v_col0 % 64 == 0 && ld_scale > 0,
               "decode_cross_attention_e4m3: ldq must be a multiple of 8 elements, ldkv of 16 bytes, the K and V column "
               "offsets multiples of 64");
    AB_REQUIRE(kv8 != nullptr && kv_scale != nullptr, "decode_cross_attention_e4m3: null K|V codes or scales");
    AB_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(kv8) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(kv_scale) & 3) == 0,
               "decode_cross_attention_e4m3: q and kv8 must be 16-byte aligned (16-byte loads)");
    if (B == 0) return ATLAS_B200_OK;
    const int chunks = (Lk + chunk - 1) / chunk;
    AB_REQUIRE(chunks <= 65535 && H <= 65535 && B <= 65535, "decode_cross_attention_e4m3: grid too large");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid(chunks, H, B);
    abh::prof_begin(s, abh::PROF_DECODE_CROSS);
    if (is_bf16)
        dec::decode_cross_attention_kernel<true, true><<<grid, dec::CROSS_THREADS, 0, s>>>(
            static_cast<const uint16_t*>(q), ldq, kv8, ldkv, k_col0, v_col0, add_mask, tile_live, Lk, chunk, scale, o_partial,
            ml_partial, H, kv_scale, ld_scale);
    else
        dec::decode_cross_attention_kernel<false, true><<<grid, dec::CROSS_THREADS, 0, s>>>(
            static_cast<const uint16_t*>(q), ldq, kv8, ldkv, k_col0, v_col0, add_mask, tile_live, Lk, chunk, scale, o_partial,
            ml_partial, H, kv_scale, ld_scale);
    // = K | V codes + their two scales read
    abh::prof_end(s, abh::PROF_DECODE_CROSS, 2.0 * B * H * static_cast<double>(Lk) * (dec::D + 4));
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_decode_self_attention(const void* qkv, int64_t ldqkv, void* cache, int32_t Tmax, const int32_t* t_dev,
                                     const float* bias_delta, float scale, void* out, int64_t ldo, int32_t B, int32_t H,
                                     int32_t is_bf16, void* stream) {
    AB_REQUIRE(B >= 0 && H > 0 && Tmax > 0 && t_dev != nullptr, "decode_self_attention: bad shape");
    if (B == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid(H, B);
    if (is_bf16)
        dec::decode_self_attention_kernel<true><<<grid, dec::D, 0, s>>>(static_cast<const uint16_t*>(qkv), ldqkv,
                                                                        static_cast<uint16_t*>(cache), Tmax, t_dev, bias_delta,
                                                                        scale, static_cast<uint16_t*>(out), ldo, H);
    else
        dec::decode_self_attention_kernel<false><<<grid, dec::D, 0, s>>>(static_cast<const uint16_t*>(qkv), ldqkv,
                                                                         static_cast<uint16_t*>(cache), Tmax, t_dev, bias_delta,
                                                                         scale, static_cast<uint16_t*>(out), ldo, H);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_decode_self_attention_beam(const void* qkv, int64_t ldqkv, void* cache, int32_t Tmax, const int32_t* t_dev,
                                          const int32_t* anc, const float* bias_delta, float scale, void* out, int64_t ldo,
                                          int32_t R, int32_t H, int32_t is_bf16, void* stream) {
    AB_REQUIRE(R >= 0 && H > 0 && Tmax > 0 && t_dev != nullptr && anc != nullptr, "decode_self_attention_beam: bad shape");
    AB_REQUIRE(R <= 65535 && H <= 65535, "decode_self_attention_beam: grid too large");
    if (R == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid(H, R);
    if (is_bf16)
        dec::decode_self_attention_kernel<true, true><<<grid, dec::D, 0, s>>>(
            static_cast<const uint16_t*>(qkv), ldqkv, static_cast<uint16_t*>(cache), Tmax, t_dev, bias_delta, scale,
            static_cast<uint16_t*>(out), ldo, H, anc);
    else
        dec::decode_self_attention_kernel<false, true><<<grid, dec::D, 0, s>>>(
            static_cast<const uint16_t*>(qkv), ldqkv, static_cast<uint16_t*>(cache), Tmax, t_dev, bias_delta, scale,
            static_cast<uint16_t*>(out), ldo, H, anc);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_decode_argmax(const void* logits, int64_t ld, int32_t V, int64_t* seq, int64_t ld_seq, int64_t* tok_in,
                             uint8_t* done, int32_t* t_dev, int32_t eos_id, int32_t pad_id, int32_t min_length, int32_t B,
                             int32_t is_bf16, void* stream) {
    AB_REQUIRE(B >= 0 && V > 0 && t_dev != nullptr, "decode_argmax: bad shape");
    if (B == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16)
        dec::decode_argmax_kernel<true><<<B, 256, 0, s>>>(static_cast<const uint16_t*>(logits), ld, V, seq, ld_seq, tok_in, done,
                                                          t_dev, eos_id, pad_id, min_length, B);
    else
        dec::decode_argmax_kernel<false><<<B, 256, 0, s>>>(static_cast<const uint16_t*>(logits), ld, V, seq, ld_seq, tok_in,
                                                           done, t_dev, eos_id, pad_id, min_length, B);
    dec::advance_step_kernel<<<1, 1, 0, s>>>(t_dev);
    abh::count_launch(2);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
