// Elementwise dropout of 16-bit rows (+ optional residual add) and the mask-export kernels the tests use.
//   out[m, n] = (residual[m, n] +) r16( keep(m, n) ? x[m, n] * inv_keep : 0 )
// replaces nn.Dropout on hidden states in the TRAINING path (src/modeling_t5.py:266,286,310,561 and the T5Stack input /
// output dropouts :960,1070; src/modeling_bert.py:222,378,459).  The backward of y = dropout(x) is the same kernel on dy
// with the same (seed, offset): masks are re-derived, never stored (csrc/dropout.cuh for the generator and the layout).
// HBM-bound: one read of x (+ residual) and one write, 16-byte vectors, one Philox call per vector.
#include "common.cuh"
#include "dropout.cuh"
#include "host_common.h"

namespace dr {

template <bool kBF16>
__device__ __forceinline__ float f32(uint32_t h) {
    if constexpr (kBF16) return __uint_as_float(h << 16);
    else return __half2float(__ushort_as_half(static_cast<unsigned short>(h & 0xFFFFu)));
}

template <bool kBF16>
__global__ void __launch_bounds__(256)
dropout_kernel(const uint16_t* __restrict__ x, int64_t ldx, const uint16_t* __restrict__ res, int64_t ldr,
               uint16_t* __restrict__ out, int64_t ldo, int64_t M, int N, const int32_t* __restrict__ row_tiles,
               abdrop::Key key) {
    const int vec_per_row = N / 8;
    const int64_t nvec = M * vec_per_row;
    for (int64_t v = blockIdx.x * 256ll + threadIdx.x; v < nvec; v += gridDim.x * 256ll) {
        const int64_t m = v / vec_per_row;
        const int c = static_cast<int>(v % vec_per_row) * 8;
        const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + m * ldx + c));
        // the mask of row m, or of padded row 64 row_tiles[m / 64] + m % 64 on the packed rows of the compacted encoder
        const int64_t mk = row_tiles != nullptr ? 64ll * __ldg(row_tiles + m / 64) + m % 64 : m;
        uint32_t w[4];
        abdrop::elem_words(key, static_cast<uint64_t>(mk * vec_per_row + c / 8), w);
        const uint32_t xs[4] = {xv.x, xv.y, xv.z, xv.w};
        uint32_t o[4];
        uint4 rv = make_uint4(0, 0, 0, 0);
        if (res != nullptr) rv = __ldg(reinterpret_cast<const uint4*>(res + m * ldr + c));
        const uint32_t rs[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float a = abdrop::keep_lo(key, w[k]) ? f32<kBF16>(xs[k]) * key.inv_keep : 0.f;
            float b = abdrop::keep_hi(key, w[k]) ? f32<kBF16>(xs[k] >> 16) * key.inv_keep : 0.f;
            if (res != nullptr) {
                // nn.Dropout rounds its result to the activation dtype before the residual add (separate torch ops)
                const uint32_t d = ab::pack2_rn<kBF16>(a, b);
                a = f32<kBF16>(d) + f32<kBF16>(rs[k]);
                b = f32<kBF16>(d >> 16) + f32<kBF16>(rs[k] >> 16);
            }
            o[k] = ab::pack2_rn<kBF16>(a, b);
        }
        *reinterpret_cast<uint4*>(out + m * ldo + c) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

__global__ void __launch_bounds__(256) mask_elem_kernel(uint8_t* __restrict__ out, int64_t M, int N, abdrop::Key key) {
    const int64_t nvec = M * (N / 8);
    for (int64_t v = blockIdx.x * 256ll + threadIdx.x; v < nvec; v += gridDim.x * 256ll) {
        uint32_t w[4];
        abdrop::elem_words(key, static_cast<uint64_t>(v), w);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            out[v * 8 + 2 * k] = abdrop::keep_lo(key, w[k]) ? 1 : 0;
            out[v * 8 + 2 * k + 1] = abdrop::keep_hi(key, w[k]) ? 1 : 0;
        }
    }
}

// keep mask of attention probabilities: out [rows, Lk] (rows = B * H * Lq), csrc/dropout.cuh's attention layout
__global__ void __launch_bounds__(256) mask_attn_kernel(uint8_t* __restrict__ out, int64_t rows, int Lk, abdrop::Key key) {
    const int calls_per_row = ((Lk + 31) / 32) * 4;
    const int64_t ncalls = rows * calls_per_row;
    for (int64_t idx = blockIdx.x * 256ll + threadIdx.x; idx < ncalls; idx += gridDim.x * 256ll) {
        const int64_t R = idx / calls_per_row;
        const int gq = static_cast<int>(idx % calls_per_row);
        const uint32_t G = gq >> 2, q = gq & 3;
        uint32_t w[4];
        abdrop::attn_words(key, static_cast<uint64_t>(R), G, q, w);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int j = 32 * G + 8 * t + 2 * q;
            if (j < Lk) out[R * Lk + j] = abdrop::keep_lo(key, w[t]) ? 1 : 0;
            if (j + 1 < Lk) out[R * Lk + j + 1] = abdrop::keep_hi(key, w[t]) ? 1 : 0;
        }
    }
}

inline int grid_for(int64_t work) {
    const int64_t blocks = (work + 255) / 256;
    const int64_t cap = static_cast<int64_t>(abh::num_sms()) * 16;
    return static_cast<int>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace dr

extern "C" {

int atlas_b200_dropout(const void* x, int64_t ldx, const void* residual, int64_t ldr, void* out, int64_t ldo, int64_t M,
                       int32_t N, float p, uint64_t seed, uint64_t offset, const int32_t* row_tiles, int32_t is_bf16,
                       void* stream) {
    AB_REQUIRE(M >= 0 && N > 0 && N % 8 == 0 && ldx % 8 == 0 && ldo % 8 == 0 && (residual == nullptr || ldr % 8 == 0),
               "dropout: N and the strides must be multiples of 8 elements");
    AB_REQUIRE(row_tiles == nullptr || M % 64 == 0, "dropout: row_tiles needs whole 64-row tiles (got M=%lld)",
               static_cast<long long>(M));
    AB_REQUIRE(p >= 0.f && p < 1.f, "dropout: need 0 <= p < 1 (got %f)", p);
    if (M == 0) return ATLAS_B200_OK;
    const abdrop::Key key = abdrop::make_key(p, seed, offset);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = dr::grid_for(M * (N / 8));
    const uint16_t *xp = static_cast<const uint16_t*>(x), *rp = static_cast<const uint16_t*>(residual);
    uint16_t* op = static_cast<uint16_t*>(out);
    if (is_bf16) dr::dropout_kernel<true><<<grid, 256, 0, s>>>(xp, ldx, rp, ldr, op, ldo, M, N, row_tiles, key);
    else dr::dropout_kernel<false><<<grid, 256, 0, s>>>(xp, ldx, rp, ldr, op, ldo, M, N, row_tiles, key);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_dropout_mask(uint8_t* out, int64_t M, int32_t N, float p, uint64_t seed, uint64_t offset, void* stream) {
    AB_REQUIRE(M >= 0 && N > 0 && N % 8 == 0, "dropout_mask: N must be a multiple of 8");
    if (M == 0) return ATLAS_B200_OK;
    dr::mask_elem_kernel<<<dr::grid_for(M * (N / 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        out, M, N, abdrop::make_key(p, seed, offset));
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_attention_dropout_mask(uint8_t* out, int64_t rows, int32_t Lk, float p, uint64_t seed, uint64_t offset,
                                      void* stream) {
    AB_REQUIRE(rows >= 0 && Lk > 0, "attention_dropout_mask: bad shape");
    if (rows == 0) return ATLAS_B200_OK;
    dr::mask_attn_kernel<<<dr::grid_for(rows * ((Lk + 31) / 32) * 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        out, rows, Lk, abdrop::make_key(p, seed, offset));
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
