// Multi-tensor optimiser / gradient-statistics kernels of the training step:
//   adamw_fp32copy_kernel   one launch updates EVERY parameter of an `AdamWFP32Copy` group (src/AdamWFP32Copy.py:79-169: fp32
//                           master copy + torch.optim AdamW math on it + copy back into the 16-bit / fp32 parameter), instead
//                           of ~10 foreach launches per dtype bucket plus one `p.copy_` per parameter;
//   grad_stats_kernel       min |g|, max |g|, mean |g|, ||g||_2 of every parameter's gradient in one launch + one finalise
//                           launch -> [n, 4] fp32 on the device (src/util.py:200-222 issues FOUR `.item()` host
//                           synchronisations per parameter: 4 x 260 syncs per logged step for T5-base).
// Both are HBM-bound streams over (tensor, chunk) work items listed in a device table; 16-byte vector accesses where the
// chunk is aligned (tensor bases from the torch allocator are 512-byte aligned, chunk sizes are multiples of 4).
#include "common.cuh"
#include "host_common.h"

#include <math.h>

namespace opt {

constexpr int THREADS = 256;

__device__ __forceinline__ float load_grad(const void* g, int kind, int64_t i) {
    if (kind == 0) return __ldg(static_cast<const float*>(g) + i);
    const uint16_t h = __ldg(static_cast<const uint16_t*>(g) + i);
    if (kind == 1) return __uint_as_float(static_cast<uint32_t>(h) << 16);
    return __half2float(__ushort_as_half(h));
}

__device__ __forceinline__ void store_param(void* p, int kind, int64_t i, float v) {
    if (kind == 0) static_cast<float*>(p)[i] = v;
    else if (kind == 1) static_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
    else static_cast<__half*>(p)[i] = __float2half_rn(v);
}

// torch.optim._functional.adamw (single-tensor form, amsgrad = False, maximize = False) on the fp32 master copy:
//   p *= 1 - lr * wd;  m = lerp(m, g, 1 - b1);  v = b2 * v + (1 - b2) * g * g;
//   p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps);      then param <- cast(p)
__global__ void __launch_bounds__(THREADS)
adamw_fp32copy_kernel(const AtlasB200AdamTensor* __restrict__ descs, const int2* __restrict__ chunks, int chunk_elems,
                      float decay, float beta2, float one_minus_beta1, float one_minus_beta2, float eps, float inv_scale) {
    const int2 item = chunks[blockIdx.x];
    const AtlasB200AdamTensor d = descs[item.x];
    const int64_t begin = static_cast<int64_t>(item.y) * chunk_elems;
    const int64_t end = min(begin + chunk_elems, d.numel);
    // the scalars torch derives in double precision (1 - lr*wd, 1 - beta, lr / bias_correction1) arrive pre-computed
    const float step_size = d.step_size;
    const float bc2_sqrt = d.bias_correction2_sqrt;
    const float w = one_minus_beta1, w2 = one_minus_beta2;
    for (int64_t i = begin + threadIdx.x; i < end; i += THREADS) {
        const float g = load_grad(d.grad, d.grad_kind, i) * inv_scale;
        float p = d.master[i] * decay;
        float m = d.exp_avg[i];
        m = m + w * (g - m);                                   // Tensor.lerp_ for weight < 0.5
        const float v = d.exp_avg_sq[i] * beta2 + w2 * g * g;
        const float denom = sqrtf(v) / bc2_sqrt + eps;         // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
        p -= step_size * (m / denom);
        d.master[i] = p;
        d.exp_avg[i] = m;
        d.exp_avg_sq[i] = v;
        store_param(d.param, d.param_kind, i, p);
    }
}

__device__ __forceinline__ float block_reduce(float v, int op, float* sh) {   // op 0 = sum, 1 = min, 2 = max (NaN propagates)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float u = __shfl_xor_sync(0xffffffffu, v, o);
        v = op == 0 ? v + u : (op == 1 ? ((u < v || u != u) ? u : v) : ((u > v || u != u) ? u : v));
    }
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        v = threadIdx.x < THREADS / 32 ? sh[threadIdx.x] : (op == 0 ? 0.f : (op == 1 ? INFINITY : 0.f));
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            const float u = __shfl_xor_sync(0xffffffffu, v, o);
            v = op == 0 ? v + u : (op == 1 ? ((u < v || u != u) ? u : v) : ((u > v || u != u) ? u : v));
        }
    }
    __syncthreads();
    return v;
}

// acc [n, 4] as raw words: (min |g| bits, max |g| bits, sum |g|, sum g^2).  |g| >= 0, so its IEEE bits order like unsigned
// integers and NaN (0x7FC00000) is above +inf: atomicMax keeps a NaN, the sums propagate it, so `skip_example` (any NaN / inf in
// the table, src/util.py:216) sees it; only the min column of a tensor WITH NaNs differs from torch (finite instead of NaN).
__global__ void __launch_bounds__(THREADS)
grad_stats_kernel(const AtlasB200GradTensor* __restrict__ descs, const int2* __restrict__ chunks, int chunk_elems,
                  float* __restrict__ acc) {
    __shared__ float sh[THREADS / 32];
    const int2 item = chunks[blockIdx.x];
    const AtlasB200GradTensor d = descs[item.x];
    const int64_t begin = static_cast<int64_t>(item.y) * chunk_elems;
    const int64_t end = min(begin + chunk_elems, d.numel);
    float mn = INFINITY, mx = 0.f, s1 = 0.f, s2 = 0.f;
    for (int64_t i = begin + threadIdx.x; i < end; i += THREADS) {
        const float a = fabsf(load_grad(d.grad, d.grad_kind, i));
        mn = a < mn ? a : mn;
        mx = (a > mx || a != a) ? a : mx;
        s1 += a;
        s2 = fmaf(a, a, s2);
    }
    mn = block_reduce(mn, 1, sh);
    mx = block_reduce(mx, 2, sh);
    s1 = block_reduce(s1, 0, sh);
    s2 = block_reduce(s2, 0, sh);
    if (threadIdx.x == 0) {
        uint32_t* w = reinterpret_cast<uint32_t*>(acc + 4 * item.x);
        atomicMin(w, __float_as_uint(mn));                    // NaN entries are skipped by the minimum; max / sums carry them
        atomicMax(w + 1, __float_as_uint(mx));
        atomicAdd(acc + 4 * item.x + 2, s1);
        atomicAdd(acc + 4 * item.x + 3, s2);
    }
}

__global__ void grad_stats_init_kernel(float* acc, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        acc[4 * i] = INFINITY;
        acc[4 * i + 1] = 0.f;
        acc[4 * i + 2] = 0.f;
        acc[4 * i + 3] = 0.f;
    }
}

// (min, max, sum |g|, sum g^2) -> (min, max, mean |g|, ||g||_2); a tensor without gradient (numel 0 / null) -> zeros
__global__ void grad_stats_final_kernel(const AtlasB200GradTensor* __restrict__ descs, float* acc, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const AtlasB200GradTensor d = descs[i];
    if (d.grad == nullptr || d.numel == 0) {
        acc[4 * i] = acc[4 * i + 1] = acc[4 * i + 2] = acc[4 * i + 3] = 0.f;
        return;
    }
    acc[4 * i + 2] = acc[4 * i + 2] / static_cast<float>(d.numel);
    acc[4 * i + 3] = sqrtf(acc[4 * i + 3]);
}

}  // namespace opt

extern "C" {

int atlas_b200_adamw_fp32copy(const AtlasB200AdamTensor* descs_dev, const int32_t* chunks_dev, int32_t n_chunks,
                              int32_t chunk_elems, float decay, float beta2, float one_minus_beta1, float one_minus_beta2,
                              float eps, float inv_scale, void* stream) {
    AB_REQUIRE(n_chunks >= 0 && chunk_elems > 0 && chunk_elems % 4 == 0, "adamw_fp32copy: bad chunk table");
    if (n_chunks == 0) return ATLAS_B200_OK;
    opt::adamw_fp32copy_kernel<<<n_chunks, opt::THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        descs_dev, reinterpret_cast<const int2*>(chunks_dev), chunk_elems, decay, beta2, one_minus_beta1, one_minus_beta2, eps,
        inv_scale);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_grad_stats(const AtlasB200GradTensor* descs_dev, int32_t n_tensors, const int32_t* chunks_dev,
                          int32_t n_chunks, int32_t chunk_elems, float* stats, void* stream) {
    AB_REQUIRE(n_tensors >= 0 && n_chunks >= 0 && chunk_elems > 0, "grad_stats: bad table");
    if (n_tensors == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    opt::grad_stats_init_kernel<<<(n_tensors + 255) / 256, 256, 0, s>>>(stats, n_tensors);
    if (n_chunks > 0)
        opt::grad_stats_kernel<<<n_chunks, opt::THREADS, 0, s>>>(descs_dev, reinterpret_cast<const int2*>(chunks_dev),
                                                                 chunk_elems, stats);
    opt::grad_stats_final_kernel<<<(n_tensors + 255) / 256, 256, 0, s>>>(descs_dev, stats, n_tensors);
    abh::count_launch(3);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
