// HBM-bound kernels of the training step (train.py -> Atlas.forward -> loss.backward() in the reference): what autograd
// derives for the row-wise / elementwise pieces of Contriever (src/modeling_bert.py) and FiD's T5 (src/modeling_t5.py),
// plus the layout helpers the weight-gradient GEMMs need.  One pass over the rows each, 16-bit activations, fp32 math.
//
//   transpose_16bit     [R, C] -> [C, Rpad] (zero padded): dY^T and X^T for dW = dY^T X on the K-major wgmma GEMM
//   colsum_f32          bias gradient: db[n] = sum_m dY[m, n]
//   norm_bwd            BertLayerNorm (uncentred 2nd moment, modeling_bert.py:104-114) / T5 RMSNorm (modeling_t5.py:244-253)
//   gated_gelu fwd/bwd  T5DenseGatedGeluDense (modeling_t5.py:281-285) on the interleaved (wi_0 | wi_1) projection
//   gelu_erf fwd/bwd    BertIntermediate (modeling_bert.py:444)
//   relu_bwd            T5DenseReluDense (modeling_t5.py:263-265, T5 v1.0) from the saved ReLU output
//   bert_embed_sum      word + token_type + position (modeling_bert.py:236-243) without the LayerNorm (training keeps the sum)
//   scatter_add_rows    embedding gradients (fp32 accumulation by row index)
//   masked_mean_pool_bwd  Contriever pooling (src/retrievers.py:50-53)
//   cross_entropy fwd/bwd CrossEntropyLoss(ignore_index=-100) over the LM-head logits (modeling_t5.py:1650-1652)
#include "common.cuh"
#include "host_common.h"

#include <math.h>

namespace bw {

template <bool kBF16>
__device__ __forceinline__ float f32(uint32_t h) {
    if constexpr (kBF16) return __bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(h & 0xFFFFu)));
    return __half2float(__ushort_as_half(static_cast<unsigned short>(h & 0xFFFFu)));
}
template <bool kBF16>
__device__ __forceinline__ uint16_t r16(float v) {
    if constexpr (kBF16) return __bfloat16_as_ushort(__float2bfloat16_rn(v));
    return __half_as_ushort(__float2half_rn(v));
}
template <bool kBF16>
__device__ __forceinline__ float rf(float v) {
    return f32<kBF16>(r16<kBF16>(v));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- transpose ------------------------------------------------------------------------------------------------------
// dst[c, r] = src[r, c] for r < R, 0 for R <= r < Rpad.  64 x 64 tiles through shared memory.
__global__ void __launch_bounds__(256)
transpose_kernel(const uint16_t* __restrict__ src, int64_t lds, uint16_t* __restrict__ dst, int64_t ldd, int R, int C,
                 int Rpad) {
    __shared__ uint16_t tile[64][66];
    const int r0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 lanes x 8 warps
    for (int rr = ty; rr < 64; rr += 8) {
        const int r = r0 + rr, c = c0 + 2 * tx;
        uint32_t v = 0;
        if (r < R && c < C) v = *reinterpret_cast<const uint32_t*>(src + static_cast<int64_t>(r) * lds + c);  // C even
        tile[rr][2 * tx] = static_cast<uint16_t>(v & 0xFFFFu);
        tile[rr][2 * tx + 1] = static_cast<uint16_t>(v >> 16);
    }
    __syncthreads();
    for (int cc = ty; cc < 64; cc += 8) {
        const int c = c0 + cc, r = r0 + 2 * tx;
        if (c < C && r < Rpad) {   // Rpad even, r even
            const uint32_t v = static_cast<uint32_t>(tile[2 * tx][cc]) | (static_cast<uint32_t>(tile[2 * tx + 1][cc]) << 16);
            *reinterpret_cast<uint32_t*>(dst + static_cast<int64_t>(c) * ldd + r) = v;
        }
    }
}

// ---- column sums ----------------------------------------------------------------------------------------------------
template <bool kBF16>
__global__ void __launch_bounds__(256)
colsum_kernel(const uint16_t* __restrict__ x, int64_t ld, float* __restrict__ out, int M, int N, int rows_per_block) {
    const int c = (blockIdx.x * 256 + threadIdx.x) * 2;
    if (c >= N) return;
    const int m0 = blockIdx.y * rows_per_block;
    const int m1 = min(M, m0 + rows_per_block);
    float a = 0.f, b = 0.f;
    for (int m = m0; m < m1; ++m) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(x + static_cast<int64_t>(m) * ld + c));
        a += f32<kBF16>(v);
        b += f32<kBF16>(v >> 16);
    }
    atomicAdd(out + c, a);
    atomicAdd(out + c + 1, b);
}

// ---- LayerNorm / RMSNorm backward ------------------------------------------------------------------------------------
// forward: xn = (x - mean) * rs, rs = rsqrt(mean(x^2) + eps) [mean only for kCentre], y = w * r16(xn) (+ b)
// backward (dxn = dy * w):  dx = rs * (dxn - mean(dxn) [kCentre]) - rs^2 * x * mean(dxn * xn)  (+ dres)
//                           dw += dy * r16(xn),  db += dy
// One warp per row (grid-stride over rows); dw / db accumulate in shared memory, flushed once per block.
constexpr int MAXV = 8;
// NV = 16-byte vectors per lane (H <= NV * 256).  kRegAcc: dw / db partial sums live in registers across the rows a warp
// processes and reach shared memory once per warp (NV <= 4: H <= 1024); otherwise one shared atomic per element and row.
template <bool kBF16, bool kCentre, int NV, bool kRegAcc>
__global__ void __launch_bounds__(256)
norm_bwd_kernel(const uint16_t* __restrict__ x, int64_t ldx, const uint16_t* __restrict__ dy, int64_t lddy,
                const uint16_t* __restrict__ w, const uint16_t* __restrict__ dres, int64_t lddres,
                uint16_t* __restrict__ dx, int64_t lddx, float* __restrict__ dw, float* __restrict__ db, int rows, int H,
                float eps) {
    extern __shared__ float acc_s[];   // [2][H]
    float* dw_s = acc_s;
    float* db_s = acc_s + H;
    for (int i = threadIdx.x; i < 2 * H; i += blockDim.x) acc_s[i] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    const int nvec = H >> 3;
    float wv[NV][8];                              // the norm weight of this lane's columns
    float rdw[kRegAcc ? NV : 1][8], rdb[kRegAcc ? NV : 1][8];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int vec = lane + 32 * i;
        uint4 ww = make_uint4(0, 0, 0, 0);
        if (vec < nvec) ww = __ldg(reinterpret_cast<const uint4*>(w) + vec);
        const uint32_t w4[4] = {ww.x, ww.y, ww.z, ww.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            wv[i][e] = f32<kBF16>(w4[e >> 1] >> ((e & 1) * 16));
            if (kRegAcc) rdw[i][e] = rdb[i][e] = 0.f;
        }
    }
    for (int row = blockIdx.x * nwarp + warp; row < rows; row += gridDim.x * nwarp) {
        float xv[NV][8], gv[NV][8];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int vec = lane + 32 * i;
            if (vec < nvec) {
                const uint4 a = __ldg(reinterpret_cast<const uint4*>(x + row * ldx) + vec);
                const uint4 d = __ldg(reinterpret_cast<const uint4*>(dy + row * lddy) + vec);
                const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, dw4[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    xv[i][2 * e] = f32<kBF16>(aw[e]);
                    xv[i][2 * e + 1] = f32<kBF16>(aw[e] >> 16);
                    gv[i][2 * e] = f32<kBF16>(dw4[e]);          // dy for now; the weight is applied below
                    gv[i][2 * e + 1] = f32<kBF16>(dw4[e] >> 16);
                    s1 += xv[i][2 * e] + xv[i][2 * e + 1];
                    s2 += xv[i][2 * e] * xv[i][2 * e] + xv[i][2 * e + 1] * xv[i][2 * e + 1];
                }
            }
        }
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        const float mean = kCentre ? s1 / static_cast<float>(H) : 0.f;
        const float rs = rsqrtf(s2 / static_cast<float>(H) + eps);
        float m1 = 0.f, m2 = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int vec = lane + 32 * i;
            if (vec < nvec) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float xn = (xv[i][e] - mean) * rs;
                    const float dyv = gv[i][e];
                    if (kRegAcc) {
                        rdw[i][e] = fmaf(dyv, rf<kBF16>(xn), rdw[i][e]);
                        rdb[i][e] += dyv;
                    } else {
                        atomicAdd(&dw_s[vec * 8 + e], dyv * rf<kBF16>(xn));
                        if (db != nullptr) atomicAdd(&db_s[vec * 8 + e], dyv);
                    }
                    const float dxn = dyv * wv[i][e];
                    gv[i][e] = dxn;
                    m1 += dxn;
                    m2 += dxn * xn;
                }
            }
        }
        m1 = kCentre ? warp_sum(m1) / static_cast<float>(H) : 0.f;
        m2 = warp_sum(m2) / static_cast<float>(H);
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int vec = lane + 32 * i;
            if (vec < nvec) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = rs * (gv[i][e] - m1) - rs * rs * xv[i][e] * m2;
                if (dres != nullptr) {
                    const uint4 r = __ldg(reinterpret_cast<const uint4*>(dres + row * lddres) + vec);
                    const uint32_t r4[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
                    for (int e = 0; e < 8; ++e) o[e] += f32<kBF16>(r4[e >> 1] >> ((e & 1) * 16));
                }
                uint4 out;
                out.x = ab::pack2_rn<kBF16>(o[0], o[1]);
                out.y = ab::pack2_rn<kBF16>(o[2], o[3]);
                out.z = ab::pack2_rn<kBF16>(o[4], o[5]);
                out.w = ab::pack2_rn<kBF16>(o[6], o[7]);
                reinterpret_cast<uint4*>(dx + row * lddx)[vec] = out;
            }
        }
    }
    if (kRegAcc) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int vec = lane + 32 * i;
            if (vec < nvec) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    atomicAdd(&dw_s[vec * 8 + e], rdw[i][e]);
                    if (db != nullptr) atomicAdd(&db_s[vec * 8 + e], rdb[i][e]);
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        atomicAdd(dw + i, dw_s[i]);
        if (db != nullptr) atomicAdd(db + i, db_s[i]);
    }
}

// ---- activations ----------------------------------------------------------------------------------------------------
// transformers' gelu_new and its derivative: gelu(x) = x * sig(2u), u = c (x + 0.044715 x^3), c = sqrt(2 / pi)
__device__ __forceinline__ void gelu_new_and_grad(float x, float& y, float& dydx) {
    const float c = 0.7978845608028654f, a = 0.044715f;
    const float u = c * (x + a * x * x * x);
    const float t = tanhf(u);
    y = 0.5f * x * (1.0f + t);
    dydx = 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * c * (1.0f + 3.0f * a * x * x);
}

// u [M, 2F] with columns (2j, 2j + 1) = (x.wi_0[j], x.wi_1[j]);  g[m, j] = r16(r16(gelu_new(u0)) * u1)
// (gelu evaluated in fp32 and cast, then the 16-bit product: modeling_t5.py:281-285)
template <bool kBF16>
__global__ void __launch_bounds__(256)
gated_fwd_kernel(const uint16_t* __restrict__ u, int64_t ldu, uint16_t* __restrict__ g, int64_t ldg, int64_t M, int F) {
    const int64_t pairs = M * (F / 2);
    for (int64_t idx = blockIdx.x * 256ll + threadIdx.x; idx < pairs; idx += gridDim.x * 256ll) {
        const int64_t m = idx / (F / 2);
        const int j2 = static_cast<int>(idx % (F / 2)) * 2;      // output columns j2, j2 + 1
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(u + m * ldu + 2 * j2));
        float y0, y1, d;
        gelu_new_and_grad(f32<kBF16>(v.x), y0, d);
        gelu_new_and_grad(f32<kBF16>(v.y), y1, d);
        const float o0 = rf<kBF16>(y0) * f32<kBF16>(v.x >> 16), o1 = rf<kBF16>(y1) * f32<kBF16>(v.y >> 16);
        *reinterpret_cast<uint32_t*>(g + m * ldg + j2) = ab::pack2_rn<kBF16>(o0, o1);
    }
}

// du[m, 2j] = dg * u1 * gelu_new'(u0),  du[m, 2j + 1] = dg * gelu_new(u0)
template <bool kBF16>
__global__ void __launch_bounds__(256)
gated_bwd_kernel(const uint16_t* __restrict__ u, int64_t ldu, const uint16_t* __restrict__ dg, int64_t lddg,
                 uint16_t* __restrict__ du, int64_t lddu, int64_t M, int F) {
    const int64_t pairs = M * (F / 2);
    for (int64_t idx = blockIdx.x * 256ll + threadIdx.x; idx < pairs; idx += gridDim.x * 256ll) {
        const int64_t m = idx / (F / 2);
        const int j2 = static_cast<int>(idx % (F / 2)) * 2;
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(u + m * ldu + 2 * j2));
        const uint32_t d2 = __ldg(reinterpret_cast<const uint32_t*>(dg + m * lddg + j2));
        float y0, y1, g0, g1;
        gelu_new_and_grad(f32<kBF16>(v.x), y0, g0);
        gelu_new_and_grad(f32<kBF16>(v.y), y1, g1);
        const float d0 = f32<kBF16>(d2), d1 = f32<kBF16>(d2 >> 16);
        uint2 o;
        o.x = ab::pack2_rn<kBF16>(d0 * f32<kBF16>(v.x >> 16) * g0, d0 * y0);
        o.y = ab::pack2_rn<kBF16>(d1 * f32<kBF16>(v.y >> 16) * g1, d1 * y1);
        *reinterpret_cast<uint2*>(du + m * lddu + 2 * j2) = o;
    }
}

// erf GELU: y = 0.5 z (1 + erf(z / sqrt 2));  dz = dy * (Phi(z) + z phi(z)).  `dy == nullptr`: forward.
template <bool kBF16>
__global__ void __launch_bounds__(256)
gelu_erf_kernel(const uint16_t* __restrict__ z, int64_t ldz, const uint16_t* __restrict__ dy, int64_t lddy,
                uint16_t* __restrict__ out, int64_t ldo, int64_t M, int N) {
    const int64_t pairs = M * (N / 2);
    for (int64_t idx = blockIdx.x * 256ll + threadIdx.x; idx < pairs; idx += gridDim.x * 256ll) {
        const int64_t m = idx / (N / 2);
        const int c = static_cast<int>(idx % (N / 2)) * 2;
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(z + m * ldz + c));
        const float z0 = f32<kBF16>(v), z1 = f32<kBF16>(v >> 16);
        const float p0 = 0.5f * (1.0f + erff(z0 * 0.70710678118654752f)), p1 = 0.5f * (1.0f + erff(z1 * 0.70710678118654752f));
        float o0, o1;
        if (dy == nullptr) {
            o0 = z0 * p0;
            o1 = z1 * p1;
        } else {
            const uint32_t d = __ldg(reinterpret_cast<const uint32_t*>(dy + m * lddy + c));
            o0 = f32<kBF16>(d) * (p0 + z0 * 0.3989422804014327f * __expf(-0.5f * z0 * z0));
            o1 = f32<kBF16>(d >> 16) * (p1 + z1 * 0.3989422804014327f * __expf(-0.5f * z1 * z1));
        }
        *reinterpret_cast<uint32_t*>(out + m * ldo + c) = ab::pack2_rn<kBF16>(o0, o1);
    }
}

// dU = dG * [G > 0] from the saved forward output G = relu(U) (the ReLU's own output decides, as torch's
// threshold_backward does): a pure select of 16-bit values, eight columns per thread
template <bool kBF16>
__global__ void __launch_bounds__(256)
relu_bwd_kernel(const uint16_t* __restrict__ g, int64_t ldg, const uint16_t* __restrict__ dg, int64_t lddg,
                uint16_t* __restrict__ du, int64_t lddu, int64_t M, int N) {
    const int64_t vecs = M * (N / 8);
    for (int64_t idx = blockIdx.x * 256ll + threadIdx.x; idx < vecs; idx += gridDim.x * 256ll) {
        const int64_t m = idx / (N / 8);
        const int c = static_cast<int>(idx % (N / 8)) * 8;
        const uint4 gv = __ldg(reinterpret_cast<const uint4*>(g + m * ldg + c));
        const uint4 dv = __ldg(reinterpret_cast<const uint4*>(dg + m * lddg + c));
        const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w}, dw[4] = {dv.x, dv.y, dv.z, dv.w};
        uint32_t o[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint32_t lo = f32<kBF16>(gw[q]) > 0.f ? 0x0000FFFFu : 0u;
            const uint32_t hi = f32<kBF16>(gw[q] >> 16) > 0.f ? 0xFFFF0000u : 0u;
            o[q] = dw[q] & (lo | hi);
        }
        *reinterpret_cast<uint4*>(du + m * lddu + c) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// ---- embeddings -----------------------------------------------------------------------------------------------------
// y[row] = r16(r16(word[id] + type[tt]) + pos[row % L])   (16-bit adds in the reference's order)
template <bool kBF16>
__global__ void __launch_bounds__(256)
bert_embed_sum_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ tts, const uint16_t* __restrict__ word,
                      const uint16_t* __restrict__ type, const uint16_t* __restrict__ pos, uint16_t* __restrict__ y,
                      int64_t rows, int L, int H) {
    const int hp = H / 2;
    for (int64_t idx = blockIdx.x * 256ll + threadIdx.x; idx < rows * hp; idx += gridDim.x * 256ll) {
        const int64_t row = idx / hp;
        const int c = static_cast<int>(idx % hp) * 2;
        const int64_t tok = ids[row], tt = tts ? tts[row] : 0;
        const uint32_t a = __ldg(reinterpret_cast<const uint32_t*>(word + tok * H + c));
        const uint32_t b = __ldg(reinterpret_cast<const uint32_t*>(type + tt * H + c));
        const uint32_t d = __ldg(reinterpret_cast<const uint32_t*>(pos + (row % L) * H + c));
        const float o0 = rf<kBF16>(f32<kBF16>(a) + f32<kBF16>(b)) + f32<kBF16>(d);
        const float o1 = rf<kBF16>(f32<kBF16>(a >> 16) + f32<kBF16>(b >> 16)) + f32<kBF16>(d >> 16);
        *reinterpret_cast<uint32_t*>(y + row * H + c) = ab::pack2_rn<kBF16>(o0, o1);
    }
}

// dst[idx[row] (or row % modulo when idx == nullptr), :] += src[row, :]   (fp32 atomics; rows with idx == skip are dropped)
template <bool kBF16>
__global__ void __launch_bounds__(256)
scatter_add_rows_kernel(const int64_t* __restrict__ idx, int modulo, const uint16_t* __restrict__ src, int64_t lds,
                        float* __restrict__ dst, int64_t rows, int H, int64_t skip, int64_t table_rows) {
    const int hp = H / 2;
    for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < rows * hp; i += gridDim.x * 256ll) {
        const int64_t row = i / hp;
        const int c = static_cast<int>(i % hp) * 2;
        const int64_t r = idx ? idx[row] : row % modulo;
        if (r == skip || r < 0 || r >= table_rows) continue;
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(src + row * lds + c));
        atomicAdd(dst + r * H + c, f32<kBF16>(v));
        atomicAdd(dst + r * H + c + 1, f32<kBF16>(v >> 16));
    }
}

// dx[b, l, :] = mask[b, l] ? demb[b, :] / count[b] : 0
template <bool kBF16>
__global__ void __launch_bounds__(256)
pool_bwd_kernel(const uint16_t* __restrict__ demb, int64_t ldd, const int64_t* __restrict__ mask, uint16_t* __restrict__ dx,
                int L, int H) {
    const int b = blockIdx.x;
    __shared__ int cnt_s;
    if (threadIdx.x == 0) cnt_s = 0;
    __syncthreads();
    int c = 0;
    for (int l = threadIdx.x; l < L; l += blockDim.x) c += mask[static_cast<int64_t>(b) * L + l] != 0;
    atomicAdd(&cnt_s, c);
    __syncthreads();
    const float inv = 1.0f / static_cast<float>(cnt_s);
    const int hp = H / 2;
    for (int i = threadIdx.x; i < L * hp; i += blockDim.x) {
        const int l = i / hp, col = (i % hp) * 2;
        uint32_t o = 0;
        if (mask[static_cast<int64_t>(b) * L + l] != 0) {
            const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(demb + b * ldd + col));
            o = ab::pack2_rn<kBF16>(f32<kBF16>(v) * inv, f32<kBF16>(v >> 16) * inv);
        }
        *reinterpret_cast<uint32_t*>(dx + (static_cast<int64_t>(b) * L + l) * H + col) = o;
    }
}

// ---- cross entropy --------------------------------------------------------------------------------------------------
// one block per row: lse[row] = logsumexp(logits[row]) (fp32), loss[row] = lse - logits[row, label] (0 when label == -100)
template <bool kBF16>
__global__ void __launch_bounds__(256)
ce_fwd_kernel(const uint16_t* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels, float* __restrict__ lse,
              float* __restrict__ loss, int V) {
    __shared__ float red[8];
    __shared__ float bcast;
    const int row = blockIdx.x;
    const uint16_t* x = logits + row * ld;
    float mx = -INFINITY;
    for (int c = threadIdx.x; c < V; c += 256) mx = fmaxf(mx, f32<kBF16>(x[c]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = red[0];
        for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
        bcast = m;
    }
    __syncthreads();
    mx = bcast;
    float s = 0.f;
    for (int c = threadIdx.x; c < V; c += 256) s += expf(f32<kBF16>(x[c]) - mx);
    s = warp_sum(s);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        const float l = mx + logf(t);
        lse[row] = l;
        const int64_t y = labels[row];
        loss[row] = (y >= 0 && y < V) ? l - f32<kBF16>(x[y]) : 0.f;
    }
}

// dlogits[row, c] = (exp(logits - lse) - [c == label]) * gscale[0]   (0 for ignored rows)
template <bool kBF16>
__global__ void __launch_bounds__(256)
ce_bwd_kernel(const uint16_t* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels,
              const float* __restrict__ lse, const float* __restrict__ gscale, uint16_t* __restrict__ dlogits, int64_t ldd,
              int V) {
    const int row = blockIdx.y;
    const int c = (blockIdx.x * 256 + threadIdx.x) * 2;
    if (c >= V) return;
    const int64_t y = labels[row];
    uint32_t o = 0;
    if (y >= 0 && y < V) {
        const float gs = __ldg(gscale), l = lse[row];
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(logits + row * ld + c));
        float p0 = expf(f32<kBF16>(v) - l), p1 = expf(f32<kBF16>(v >> 16) - l);
        if (c == y) p0 -= 1.0f;
        if (c + 1 == y) p1 -= 1.0f;
        o = ab::pack2_rn<kBF16>(p0 * gs, p1 * gs);
    }
    *reinterpret_cast<uint32_t*>(dlogits + row * ldd + c) = o;
}

inline int grid_for(int64_t work_items) {
    const int64_t blocks = (work_items + 255) / 256;
    const int64_t cap = static_cast<int64_t>(abh::num_sms()) * 16;
    return static_cast<int>(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

}  // namespace bw

extern "C" {

int atlas_b200_transpose(const void* src, int64_t lds, void* dst, int64_t ldd, int32_t R, int32_t C, int32_t Rpad,
                         void* stream) {
    AB_REQUIRE(R >= 0 && C > 0 && C % 2 == 0 && lds % 2 == 0 && ldd % 2 == 0 && Rpad >= R && Rpad % 2 == 0 && ldd >= Rpad,
               "transpose: need even C / strides / Rpad and ldd >= Rpad >= R (R=%d C=%d Rpad=%d)", R, C, Rpad);
    if (Rpad == 0) return ATLAS_B200_OK;
    dim3 grid((Rpad + 63) / 64, (C + 63) / 64);
    AB_REQUIRE(grid.y <= 65535, "transpose: too many columns");
    bw::transpose_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint16_t*>(src), lds, static_cast<uint16_t*>(dst), ldd, R, C, Rpad);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_colsum(const void* x, int64_t ld, float* out, int32_t M, int32_t N, int32_t is_bf16, void* stream) {
    AB_REQUIRE(M >= 0 && N > 0 && N % 2 == 0 && ld % 2 == 0, "colsum: N and ld must be even");
    if (M == 0) return ATLAS_B200_OK;
    const int rows_per_block = 256;
    dim3 grid((N / 2 + 255) / 256, (M + rows_per_block - 1) / rows_per_block);
    AB_REQUIRE(grid.y <= 65535, "colsum: too many rows");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16) bw::colsum_kernel<true><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(x), ld, out, M, N, rows_per_block);
    else bw::colsum_kernel<false><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(x), ld, out, M, N, rows_per_block);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_layernorm_bwd(const void* x, int64_t ldx, const void* dy, int64_t lddy, const void* weight,
                             const void* dres, int64_t lddres, void* dx, int64_t lddx, float* dweight, float* dbias,
                             int32_t rows, int32_t H, float eps, int32_t kind, int32_t is_bf16, void* stream) {
    AB_REQUIRE(rows >= 0 && H > 0 && H % 8 == 0 && H <= bw::MAXV * 256, "layernorm_bwd: H=%d must be a multiple of 8, <= %d",
               H, bw::MAXV * 256);
    AB_REQUIRE(ldx % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0 && (dres == nullptr || lddres % 8 == 0),
               "layernorm_bwd: row strides must be multiples of 8");
    AB_REQUIRE(kind == 0 || kind == 1, "layernorm_bwd: kind must be 0 (BertLayerNorm) or 1 (T5 RMSNorm)");
    AB_REQUIRE(dweight != nullptr && (kind == 1 || dbias != nullptr), "layernorm_bwd: dweight (and dbias for kind 0) required");
    if (rows == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int blocks_needed = (rows + 7) / 8;
    const int cap = abh::num_sms() * 4;
    const int grid = blocks_needed < cap ? blocks_needed : cap;
    const size_t smem = 2 * static_cast<size_t>(H) * sizeof(float);
    const uint16_t *xp = static_cast<const uint16_t*>(x), *dyp = static_cast<const uint16_t*>(dy),
                   *wp = static_cast<const uint16_t*>(weight), *rp = static_cast<const uint16_t*>(dres);
    uint16_t* dxp = static_cast<uint16_t*>(dx);
    float* dbp = kind == 0 ? dbias : nullptr;
    auto go = [&](auto kern) { kern<<<grid, 256, smem, s>>>(xp, ldx, dyp, lddy, wp, rp, lddres, dxp, lddx, dweight, dbp, rows, H, eps); };
#define AB_NORM_BWD(NV, REG)                                                                      \
    do {                                                                                          \
        if (kind == 0) {                                                                          \
            if (is_bf16) go(bw::norm_bwd_kernel<true, true, NV, REG>);                            \
            else go(bw::norm_bwd_kernel<false, true, NV, REG>);                                   \
        } else {                                                                                  \
            if (is_bf16) go(bw::norm_bwd_kernel<true, false, NV, REG>);                           \
            else go(bw::norm_bwd_kernel<false, false, NV, REG>);                                  \
        }                                                                                         \
    } while (0)
    if (H <= 768) AB_NORM_BWD(3, true);
    else if (H <= 1024) AB_NORM_BWD(4, true);
    else AB_NORM_BWD(8, false);
#undef AB_NORM_BWD
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_gated_gelu(const void* u, int64_t ldu, const void* dg, int64_t lddg, void* out, int64_t ldo, int64_t M,
                          int32_t F, int32_t is_bf16, void* stream) {
    AB_REQUIRE(M >= 0 && F > 0 && F % 2 == 0 && ldu % 4 == 0 && ldo % 2 == 0 && (dg == nullptr || (lddg % 2 == 0 && ldo % 4 == 0)),
               "gated_gelu: F must be even and the strides 8-byte aligned");
    if (M == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = bw::grid_for(M * (F / 2));
    const uint16_t *up = static_cast<const uint16_t*>(u), *dp = static_cast<const uint16_t*>(dg);
    uint16_t* op = static_cast<uint16_t*>(out);
    if (dg == nullptr) {
        if (is_bf16) bw::gated_fwd_kernel<true><<<grid, 256, 0, s>>>(up, ldu, op, ldo, M, F);
        else bw::gated_fwd_kernel<false><<<grid, 256, 0, s>>>(up, ldu, op, ldo, M, F);
    } else {
        if (is_bf16) bw::gated_bwd_kernel<true><<<grid, 256, 0, s>>>(up, ldu, dp, lddg, op, ldo, M, F);
        else bw::gated_bwd_kernel<false><<<grid, 256, 0, s>>>(up, ldu, dp, lddg, op, ldo, M, F);
    }
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_gelu_erf(const void* z, int64_t ldz, const void* dy, int64_t lddy, void* out, int64_t ldo, int64_t M,
                        int32_t N, int32_t is_bf16, void* stream) {
    AB_REQUIRE(M >= 0 && N > 0 && N % 2 == 0 && ldz % 2 == 0 && ldo % 2 == 0 && (dy == nullptr || lddy % 2 == 0),
               "gelu_erf: N and the strides must be even");
    if (M == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = bw::grid_for(M * (N / 2));
    if (is_bf16)
        bw::gelu_erf_kernel<true><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(z), ldz, static_cast<const uint16_t*>(dy),
                                                        lddy, static_cast<uint16_t*>(out), ldo, M, N);
    else
        bw::gelu_erf_kernel<false><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(z), ldz, static_cast<const uint16_t*>(dy),
                                                         lddy, static_cast<uint16_t*>(out), ldo, M, N);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_relu_bwd(const void* g, int64_t ldg, const void* dg, int64_t lddg, void* du, int64_t lddu, int64_t M, int32_t N,
                        int32_t is_bf16, void* stream) {
    AB_REQUIRE(M >= 0 && N > 0 && N % 8 == 0 && ldg % 8 == 0 && lddg % 8 == 0 && lddu % 8 == 0,
               "relu_bwd: N and the strides must be multiples of 8");
    AB_REQUIRE(((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(dg) | reinterpret_cast<uintptr_t>(du)) & 15u) == 0,
               "relu_bwd: g, dg and du must be 16-byte aligned");
    if (M == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = bw::grid_for(M * (N / 8));
    const uint16_t *gp = static_cast<const uint16_t*>(g), *dp = static_cast<const uint16_t*>(dg);
    uint16_t* op = static_cast<uint16_t*>(du);
    if (is_bf16) bw::relu_bwd_kernel<true><<<grid, 256, 0, s>>>(gp, ldg, dp, lddg, op, lddu, M, N);
    else bw::relu_bwd_kernel<false><<<grid, 256, 0, s>>>(gp, ldg, dp, lddg, op, lddu, M, N);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_bert_embed_sum(const int64_t* input_ids, const int64_t* token_type_ids, const void* word_emb,
                              const void* type_emb, const void* pos_emb, void* y, int32_t batch, int32_t L, int32_t H,
                              int32_t is_bf16, void* stream) {
    AB_REQUIRE(batch >= 0 && L > 0 && H > 0 && H % 2 == 0, "bert_embed_sum: bad shape");
    AB_REQUIRE(abh::aligned(word_emb, 4) && abh::aligned(type_emb, 4) && abh::aligned(pos_emb, 4) && abh::aligned(y, 4),
               "bert_embed_sum: the tables and y must be 4-byte aligned");
    const int64_t rows = static_cast<int64_t>(batch) * L;
    if (rows == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = bw::grid_for(rows * (H / 2));
    const uint16_t *we = static_cast<const uint16_t*>(word_emb), *te = static_cast<const uint16_t*>(type_emb),
                   *pe = static_cast<const uint16_t*>(pos_emb);
    if (is_bf16) bw::bert_embed_sum_kernel<true><<<grid, 256, 0, s>>>(input_ids, token_type_ids, we, te, pe, static_cast<uint16_t*>(y), rows, L, H);
    else bw::bert_embed_sum_kernel<false><<<grid, 256, 0, s>>>(input_ids, token_type_ids, we, te, pe, static_cast<uint16_t*>(y), rows, L, H);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_scatter_add_rows(const int64_t* index, int32_t modulo, const void* src, int64_t lds, float* dst,
                                int64_t rows, int32_t H, int64_t skip_index, int64_t table_rows, int32_t is_bf16,
                                void* stream) {
    AB_REQUIRE(rows >= 0 && H > 0 && H % 2 == 0 && lds % 2 == 0 && (index != nullptr || modulo > 0) && table_rows > 0,
               "scatter_add_rows: bad arguments");
    if (rows == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = bw::grid_for(rows * (H / 2));
    if (is_bf16) bw::scatter_add_rows_kernel<true><<<grid, 256, 0, s>>>(index, modulo, static_cast<const uint16_t*>(src), lds, dst, rows, H, skip_index, table_rows);
    else bw::scatter_add_rows_kernel<false><<<grid, 256, 0, s>>>(index, modulo, static_cast<const uint16_t*>(src), lds, dst, rows, H, skip_index, table_rows);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_masked_mean_pool_bwd(const void* demb, int64_t ld_demb, const int64_t* mask, void* dx, int32_t batch,
                                    int32_t L, int32_t H, int32_t is_bf16, void* stream) {
    AB_REQUIRE(batch >= 0 && L > 0 && H > 0 && H % 2 == 0 && ld_demb % 2 == 0, "masked_mean_pool_bwd: bad shape");
    if (batch == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16) bw::pool_bwd_kernel<true><<<batch, 256, 0, s>>>(static_cast<const uint16_t*>(demb), ld_demb, mask, static_cast<uint16_t*>(dx), L, H);
    else bw::pool_bwd_kernel<false><<<batch, 256, 0, s>>>(static_cast<const uint16_t*>(demb), ld_demb, mask, static_cast<uint16_t*>(dx), L, H);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_cross_entropy_fwd(const void* logits, int64_t ld, const int64_t* labels, float* lse, float* loss,
                                 int32_t rows, int32_t V, int32_t is_bf16, void* stream) {
    AB_REQUIRE(rows >= 0 && V > 0, "cross_entropy_fwd: bad shape");
    if (rows == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16) bw::ce_fwd_kernel<true><<<rows, 256, 0, s>>>(static_cast<const uint16_t*>(logits), ld, labels, lse, loss, V);
    else bw::ce_fwd_kernel<false><<<rows, 256, 0, s>>>(static_cast<const uint16_t*>(logits), ld, labels, lse, loss, V);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_cross_entropy_bwd(const void* logits, int64_t ld, const int64_t* labels, const float* lse,
                                 const float* gscale, void* dlogits, int64_t ldd, int32_t rows, int32_t V, int32_t is_bf16,
                                 void* stream) {
    AB_REQUIRE(rows >= 0 && V > 0 && V % 2 == 0 && ld % 2 == 0 && ldd % 2 == 0, "cross_entropy_bwd: V and strides must be even");
    if (rows == 0) return ATLAS_B200_OK;
    AB_REQUIRE(rows <= 65535, "cross_entropy_bwd: too many rows");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid((V / 2 + 255) / 256, rows);
    if (is_bf16) bw::ce_bwd_kernel<true><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(logits), ld, labels, lse, gscale, static_cast<uint16_t*>(dlogits), ldd, V);
    else bw::ce_bwd_kernel<false><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(logits), ld, labels, lse, gscale, static_cast<uint16_t*>(dlogits), ldd, V);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
