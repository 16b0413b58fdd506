// FP8 (e4m3) cross-attention K|V cache of KV-cached generation (FiD.generate(cross_kv_dtype="fp8")): the per-layer 16-bit
// cross K|V projection [rows, 2*H*64] is quantized once per generation into codes kv8 uint8 [rows, 2*H*64] plus one fp32
// scale per (key row, 64-column block) kv_scale [rows, 2*H] - the block index is that of the 16-bit layout (K of head h =
// block h, V of head h = block H + h).  64 + 4 bytes per 64 values instead of 128: the decode steps, which stream the whole
// cache once per step (csrc/decode.cu, csrc/attention_stream.cu), read 0.53x the bytes.
//
// Rule per 64-value group x (exactly these fp32 operations, so a CPU oracle reproduces codes and scales bit for bit):
//   amax = max |x|;  inv = 448 / amax (RN);  code = e4m3_rn_satfinite(x * inv (RN));  scale = amax / 448 (RN)
//   amax == 0              -> scale 0, every code 0
//   a non-finite x in the group -> scale NaN, every code 0 (attention over that key then yields NaN, as in 16 bits)
// The dequantized value is float(e4m3(code)) * scale.
//
// One 8-lane group per 64 values (16-byte loads, 8-byte stores), 32 groups per 256-thread block.  Runs once per generation
// and layer: not on the per-step path.
#include "common.cuh"
#include "host_common.h"
#include "kv_fp8.cuh"

#include <float.h>

namespace kv8 {

constexpr int THREADS = 256;

template <bool kBF16>
__global__ void __launch_bounds__(THREADS)
quantize_kernel(const uint16_t* __restrict__ x, int64_t ldx, uint8_t* __restrict__ q, int64_t ldq, float* __restrict__ scale,
                int64_t lds, int64_t groups, int C) {
    const int64_t gi = static_cast<int64_t>(blockIdx.x) * (THREADS / 8) + (threadIdx.x >> 3);
    const int seg = threadIdx.x & 7;
    const bool ok = gi < groups;                  // no early exit: the 8-lane shuffles need the whole warp
    const int64_t g = ok ? gi : 0;
    const int64_t row = g / C;
    const int c = static_cast<int>(g - row * C);
    const uint4 w = *reinterpret_cast<const uint4*>(x + row * ldx + c * 64 + seg * 8);
    const uint32_t u[4] = {w.x, w.y, w.z, w.w};
    float f[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if constexpr (kBF16) {
            f[2 * i] = __uint_as_float(u[i] << 16);
            f[2 * i + 1] = __uint_as_float(u[i] & 0xFFFF0000u);
        } else {
            const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&u[i]));
            f[2 * i] = v.x;
            f[2 * i + 1] = v.y;
        }
    }
    float amax = 0.f;
    int bad = 0;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const float a = fabsf(f[e]);
        bad |= !(a <= FLT_MAX);                   // NaN or inf
        amax = fmaxf(amax, a);
    }
#pragma unroll
    for (int off = 1; off < 8; off <<= 1) {
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
        bad |= __shfl_xor_sync(0xffffffffu, bad, off);
    }
    uint2 codes = make_uint2(0u, 0u);
    float sc;
    if (bad) {
        sc = __int_as_float(0x7fc00000);
    } else if (amax == 0.f) {
        sc = 0.f;
    } else {
        const float inv = __fdiv_rn(E4M3_MAX, amax);
        uint32_t p[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
            p[i] = f32x2_to_e4m3x2(__fmul_rn(f[2 * i], inv), __fmul_rn(f[2 * i + 1], inv));
        codes = make_uint2(p[0] | (p[1] << 16), p[2] | (p[3] << 16));
        sc = __fdiv_rn(amax, E4M3_MAX);
    }
    if (!ok) return;
    *reinterpret_cast<uint2*>(q + row * ldq + c * 64 + seg * 8) = codes;
    if (seg == 0) scale[row * lds + c] = sc;
}

}  // namespace kv8

extern "C" {

int atlas_b200_quantize_kv_e4m3(const void* x, int64_t ldx, int64_t rows, int32_t n_blocks, uint8_t* kv8, int64_t ldkv8,
                                float* kv_scale, int64_t ld_scale, int32_t is_bf16, void* stream) {
    AB_REQUIRE(rows >= 0 && n_blocks > 0, "quantize_kv_e4m3: bad shape (rows=%lld n_blocks=%d)", (long long)rows, n_blocks);
    AB_REQUIRE(ldx % 8 == 0 && ldx >= 64LL * n_blocks && ldkv8 % 8 == 0 && ldkv8 >= 64LL * n_blocks && ld_scale >= n_blocks,
               "quantize_kv_e4m3: row strides must cover the row (ldx, ldkv8 multiples of 8 elements)");
    AB_REQUIRE(x != nullptr && kv8 != nullptr && kv_scale != nullptr, "quantize_kv_e4m3: null buffer");
    AB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(kv8) & 7) == 0 &&
                   (reinterpret_cast<uintptr_t>(kv_scale) & 3) == 0,
               "quantize_kv_e4m3: x must be 16-byte aligned (16-byte loads), kv8 8-byte aligned (8-byte stores)");
    if (rows == 0) return ATLAS_B200_OK;
    const int64_t groups = rows * n_blocks;
    const int64_t blocks = (groups + kv8::THREADS / 8 - 1) / (kv8::THREADS / 8);
    AB_REQUIRE(blocks <= 0x7fffffffLL, "quantize_kv_e4m3: too many rows");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (is_bf16)
        kv8::quantize_kernel<true><<<static_cast<unsigned>(blocks), kv8::THREADS, 0, s>>>(
            static_cast<const uint16_t*>(x), ldx, kv8, ldkv8, kv_scale, ld_scale, groups, n_blocks);
    else
        kv8::quantize_kernel<false><<<static_cast<unsigned>(blocks), kv8::THREADS, 0, s>>>(
            static_cast<const uint16_t*>(x), ldx, kv8, ldkv8, kv_scale, ld_scale, groups, n_blocks);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
