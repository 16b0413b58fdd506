// e4m3 (OCP "fn": no inf, max 448) conversions shared by the FP8 cross K|V cache kernels (csrc/kv_fp8.cu, the fp8 paths of
// csrc/decode.cu and csrc/attention_stream.cu).  sm_89+ conversion instructions; every e4m3 value is exact in fp16 and bf16.
#pragma once

#include <cuda_fp16.h>
#include <stdint.h>

namespace kv8 {

constexpr float E4M3_MAX = 448.f;

// two e4m3 codes (low byte = element 0) -> f16x2 (low half = element 0), exact
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint16_t v) {
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(v));
    return r;
}

// (a, b) -> two e4m3 codes, a in the low byte; round to nearest even, saturating to +-448
__device__ __forceinline__ uint16_t f32x2_to_e4m3x2(float a, float b) {
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
    return r;
}

// 16 e4m3 codes (one 16-byte load) -> 16 floats
__device__ __forceinline__ void unpack16(const uint4& w, float (&f)[16]) {
    const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint32_t h2 = e4m3x2_to_f16x2(static_cast<uint16_t>(u[i] >> (16 * k)));
            const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&h2));
            f[4 * i + 2 * k] = v.x;
            f[4 * i + 2 * k + 1] = v.y;
        }
    }
}

}  // namespace kv8
