// Counter-based dropout masks shared by the elementwise dropout kernel and the attention kernels (forward and backward
// re-derive the SAME keep decisions from (seed, offset, element position); nothing is stored).
//
// Reference: nn.Dropout in the training path - hidden states `src/modeling_t5.py:266,286,310,561`, attention
// probabilities `src/modeling_t5.py:515-516`, `src/modeling_bert.py:354` (BertSelfAttention.dropout), embeddings /
// BertSelfOutput / BertOutput `src/modeling_bert.py:222,378,459`.  torch's own Philox stream cannot be reproduced element
// for element by a fused kernel, so parity is defined on the distribution (keep rate, 1 / (1 - p) scaling) and on exact
// forward <-> backward consistency against torch fed the mask these kernels export (tests/test_dropout_gpu.py).
//
// Generator: Philox4x32 with 7 rounds (Salmon et al., SC'11: the smallest round count of Philox4x32 that passes BigCrush),
// key = (seed_lo, seed_hi ^ offset_hi), one call -> 4 x 32 bits = EIGHT 16-bit uniforms; an element is kept iff its
// uniform >= thr16 = round(p * 65536), so the realised drop probability is thr16 / 65536 (0.1 -> 0.100006) and the kept
// values are scaled by 65536 / (65536 - thr16).
//   * elementwise ([M, N] rows, N % 8 == 0): call v = (row * N + col) / 8, counter (v_lo, v_hi, offset_lo, 0x9E3779B9);
//     element k = col % 8 uses bits [16 (k & 1), +16) of word k >> 1.
//   * attention probabilities P[R, j], R = (b * H + h) * Lq + i, j = key index: call (G = j / 32, q = (j % 8) / 2),
//     counter (4 G + q, R_lo, R_hi, offset_lo); element j uses bits [16 (j & 1), +16) of word t = (j % 32) / 8.
//     One call therefore covers the columns {32 G + 8 t + 2 q + {0, 1} : t = 0..3} of one row: exactly the eight
//     elements one thread of an mma.sync accumulator fragment holds per row and 32-column group (backward kernels), and
//     four calls cover a 32-key group of the two rows a thread of a wgmma accumulator holds (forward kernel) - no call is shared or wasted.
#pragma once

#include <stdint.h>

namespace abdrop {

struct Key {
    uint32_t k0, k1;       // Philox key
    uint32_t off;          // low 32 bits of the offset (goes into the counter)
    uint32_t thr16;        // drop iff u16 < thr16; 0 = dropout off
    float inv_keep;        // 65536 / (65536 - thr16)
};

__host__ __device__ inline uint32_t threshold16(float p) {
    if (!(p > 0.f)) return 0u;
    float t = p * 65536.0f + 0.5f;
    if (t > 65535.0f) t = 65535.0f;
    return static_cast<uint32_t>(t);
}

__host__ __device__ inline Key make_key(float p, uint64_t seed, uint64_t offset) {
    Key k;
    k.k0 = static_cast<uint32_t>(seed);
    k.k1 = static_cast<uint32_t>(seed >> 32) ^ static_cast<uint32_t>(offset >> 32);
    k.off = static_cast<uint32_t>(offset);
    k.thr16 = threshold16(p);
    k.inv_keep = 65536.0f / static_cast<float>(65536u - k.thr16);
    return k;
}

#ifdef __CUDACC__
__device__ __forceinline__ void philox4x32_7(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                             uint32_t (&out)[4]) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 7; ++r) {
        const uint64_t p0 = static_cast<uint64_t>(M0) * c0;
        const uint64_t p1 = static_cast<uint64_t>(M1) * c2;
        const uint32_t n0 = static_cast<uint32_t>(p1 >> 32) ^ c1 ^ k0;
        const uint32_t n2 = static_cast<uint32_t>(p0 >> 32) ^ c3 ^ k1;
        c1 = static_cast<uint32_t>(p1);
        c3 = static_cast<uint32_t>(p0);
        c0 = n0;
        c2 = n2;
        k0 += W0;
        k1 += W1;
    }
    out[0] = c0, out[1] = c1, out[2] = c2, out[3] = c3;
}

// the four mask words of attention row R, column group G = j / 32, pair slot q = (j % 8) / 2
__device__ __forceinline__ void attn_words(const Key& k, uint64_t R, uint32_t G, uint32_t q, uint32_t (&w)[4]) {
    philox4x32_7(4u * G + q, static_cast<uint32_t>(R), static_cast<uint32_t>(R >> 32), k.off, k.k0, k.k1, w);
}
// keep flags of the element pair (j, j + 1), j even, out of word t = (j % 32) / 8 of attn_words(.., q = (j % 8) / 2)
__device__ __forceinline__ bool keep_lo(const Key& k, uint32_t word) { return (word & 0xFFFFu) >= k.thr16; }
__device__ __forceinline__ bool keep_hi(const Key& k, uint32_t word) { return (word >> 16) >= k.thr16; }

// the four mask words of elementwise vector v (8 consecutive elements)
__device__ __forceinline__ void elem_words(const Key& k, uint64_t v, uint32_t (&w)[4]) {
    philox4x32_7(static_cast<uint32_t>(v), static_cast<uint32_t>(v >> 32), k.off, 0x9E3779B9u, k.k0, k.k1, w);
}
#endif

}  // namespace abdrop
