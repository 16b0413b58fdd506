// Pieces of the exact top-k machinery shared by the flat MIPS scan (mips.cu) and the product-quantized scan (pq.cu):
// the order-preserving 16-bit score keys, the packed (score key, id) candidate format, the lower bound that turns a k-th
// score into a scan threshold, the per-query radix select over candidate lists and the candidate-list capacity.
#pragma once

#include "common.cuh"
#include "host_common.h"

#include <math.h>

namespace mips {

// ---------------------------------------------------------------------------------------------
// 16-bit float <-> order-preserving integer key (larger key = larger score; -0 canonicalised)
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t bits_to_key(uint32_t h) {
    h &= 0xFFFFu;
    if (h == 0x8000u) h = 0;
    return (h & 0x8000u) ? (~h & 0xFFFFu) : (h | 0x8000u);
}
__host__ __device__ __forceinline__ uint32_t key_to_bits(uint32_t key) {
    return (key & 0x8000u) ? (key & 0x7FFFu) : (~key & 0xFFFFu);
}

template <bool kBF16>
__device__ __forceinline__ uint32_t round_to_bits(float v) {
    if constexpr (kBF16) {
        return static_cast<uint32_t>(__bfloat16_as_ushort(__float2bfloat16_rn(v)));
    } else {
        return static_cast<uint32_t>(__half_as_ushort(__float2half_rn(v)));
    }
}
template <bool kBF16>
__device__ __forceinline__ float bits_to_float(uint32_t h) {
    if constexpr (kBF16) {
        return __bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(h)));
    } else {
        return __half2float(__ushort_as_half(static_cast<unsigned short>(h)));
    }
}

__device__ __forceinline__ uint64_t pack_candidate(uint32_t key16, uint32_t id) {
    return (static_cast<uint64_t>(key16) << 32) | static_cast<uint64_t>(0xFFFFFFFFu - id);
}

// Smallest fp32 x whose round-to-nearest-even 16-bit value is >= the value with sortable key `key16`.
template <bool kBF16>
__device__ float lower_bound_for_key(uint32_t key16) {
    const uint32_t hb = key_to_bits(key16);
    const float t = bits_to_float<kBF16>(hb);
    if (t != t) return -INFINITY;            // NaN threshold: keep everything
    if (t == -INFINITY) return -INFINITY;
    const float big = kBF16 ? 3.4028236692e38f : 65536.0f;  // first magnitude that rounds to inf
    // previous representable value (in value order, skipping the -0/+0 duplicate)
    uint32_t kp = key16 - 1;
    if (key_to_bits(kp) == 0x8000u) kp -= 1;
    float p = bits_to_float<kBF16>(key_to_bits(kp));
    if (p == -INFINITY || p != p) p = -big;
    float tt = (t == INFINITY) ? big : t;
    if (kBF16 && (fabsf(p) > 1e38f || fabsf(tt) > 1e38f)) {
        // avoid fp32 overflow of p + tt at the extreme end of the bf16 range
        return fminf(p, tt);
    }
    const float mid = 0.5f * (p + tt);  // exact: neighbours differ in one ulp of the 16-bit format
    const float r = bits_to_float<kBF16>(round_to_bits<kBF16>(mid));
    return (r >= t) ? mid : nextafterf(mid, INFINITY);
}

// ---------------------------------------------------------------------------------------------
// select: exact top-k of one query's candidate list (radix select on the 48-bit composite key,
// then a bitonic sort of the k winners).  One CTA per query.
// ---------------------------------------------------------------------------------------------
constexpr int SEL_THREADS = 256;
constexpr int SEL_WRITE_BOUND = 1;  // bound[q] = lower bound of the k-th key, count[q] = 0
constexpr int SEL_EMIT = 2;         // write out_scores / out_ids
constexpr int SEL_CARRY = 4;        // cand[q][0..k) = winners, count[q] = k

template <bool kBF16>
__global__ void __launch_bounds__(SEL_THREADS)
mips_select_kernel(uint64_t* __restrict__ cand, uint32_t* __restrict__ count, uint32_t capq, int k, int mode,
                   float* __restrict__ bound, uint16_t* __restrict__ out_scores, int64_t* __restrict__ out_ids,
                   int64_t id_base, int64_t id_stride, int32_t* __restrict__ status) {
    __shared__ uint32_t hist[256];
    __shared__ uint64_t s_prefix;
    __shared__ uint32_t s_krem;
    __shared__ uint32_t s_nwin;
    __shared__ uint64_t win[ATLAS_B200_MAX_TOPK];

    const int q = blockIdx.x;
    const int t = threadIdx.x;
    uint32_t n = count[q];
    if (n > capq) {
        if (t == 0 && status) atomicExch(status, 1);
        n = capq;
    }
    uint64_t* c = cand + static_cast<size_t>(q) * capq;
    const uint32_t kk = min(static_cast<uint32_t>(k), n);
    int P = 1;
    while (P < static_cast<int>(kk)) P <<= 1;

    if (t == 0) {
        s_prefix = 0;
        s_krem = kk;
        s_nwin = 0;
    }
    for (int i = t; i < P; i += SEL_THREADS) win[i] = 0;
    __syncthreads();

    // A bound-only pass (no winners needed) stops after the two score bytes of the 48-bit key.
    const bool bound_only = (mode & SEL_WRITE_BOUND) && !(mode & (SEL_EMIT | SEL_CARRY));
    if (kk > 0) {
        uint64_t mask = 0;
        for (int b = 5; b >= (bound_only ? 4 : 0); --b) {
            hist[t] = 0;
            __syncthreads();
            const uint64_t prefix = s_prefix;
            if (b == 5) {
                // top byte of the score key: scores cluster in a handful of bins, per-key shared atomics would
                // serialise -> lanes with the same bin elect a leader that adds their population count
                for (uint32_t i0 = 0; i0 < n; i0 += SEL_THREADS) {
                    const uint32_t i = i0 + t;
                    const bool live = i < n;
                    const uint32_t bin = live ? static_cast<uint32_t>((c[i] >> 40) & 0xFFu) : 256u;
                    const uint32_t peers = __match_any_sync(0xffffffffu, bin);
                    if (live && (t & 31) == static_cast<int>(__ffs(peers)) - 1) atomicAdd(&hist[bin], __popc(peers));
                }
            } else {
                // lower bytes are close to uniform over the 256 bins: plain shared atomics, 4 keys in flight
                for (uint32_t i = t; i < n; i += SEL_THREADS) {
                    const uint64_t key = c[i];
                    if ((key & mask) == prefix) atomicAdd(&hist[(key >> (8 * b)) & 0xFFu], 1u);
                }
            }
            __syncthreads();
            if (t == 0) {
                uint32_t krem = s_krem, acc = 0;
                int d = 255;
                for (; d > 0; --d) {
                    if (acc + hist[d] >= krem) break;
                    acc += hist[d];
                }
                s_krem = krem - acc;
                s_prefix = prefix | (static_cast<uint64_t>(d) << (8 * b));
            }
            mask |= static_cast<uint64_t>(0xFFu) << (8 * b);
            __syncthreads();
        }
        const uint64_t kth = s_prefix;  // exact k-th largest key (keys are unique: ids differ)
        for (uint32_t i = t; i < n && !bound_only; i += SEL_THREADS) {
            const uint64_t key = c[i];
            if (key >= kth) {
                const uint32_t pos = atomicAdd(&s_nwin, 1u);
                if (pos < ATLAS_B200_MAX_TOPK) win[pos] = key;
            }
        }
        __syncthreads();
        // bitonic sort, descending
        for (int size = 2; size <= P && !bound_only; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int i = t; i < P / 2; i += SEL_THREADS) {
                    const int lo = 2 * i - (i & (stride - 1));
                    const int hi = lo + stride;
                    const bool desc = ((lo & size) == 0);
                    const uint64_t a = win[lo], b2 = win[hi];
                    if ((a < b2) == desc) {
                        win[lo] = b2;
                        win[hi] = a;
                    }
                }
                __syncthreads();
            }
        }
    }

    if (mode & SEL_EMIT) {
        for (int i = t; i < k; i += SEL_THREADS) {
            uint32_t hb;
            int64_t id;
            if (i < static_cast<int>(kk)) {
                const uint64_t key = win[i];
                hb = key_to_bits(static_cast<uint32_t>(key >> 32));
                id = id_base + id_stride * static_cast<int64_t>(0xFFFFFFFFu - static_cast<uint32_t>(key));
            } else {
                hb = kBF16 ? 0xFF80u : 0xFC00u;  // -inf
                id = -1;
            }
            out_scores[static_cast<size_t>(q) * k + i] = static_cast<uint16_t>(hb);
            out_ids[static_cast<size_t>(q) * k + i] = id;
        }
    }
    if (mode & SEL_CARRY) {
        __syncthreads();
        for (int i = t; i < static_cast<int>(kk); i += SEL_THREADS) c[i] = win[i];
        if (t == 0) count[q] = kk;
    }
    if (mode & SEL_WRITE_BOUND) {
        if (t == 0) {
            if (kk == static_cast<uint32_t>(k) && kk > 0) {
                // bound-only passes resolved just the 16 score bits of the k-th key (s_prefix bits 47..32)
                const uint32_t kth16 = bound_only ? static_cast<uint32_t>(s_prefix >> 32)
                                                  : static_cast<uint32_t>(win[kk - 1] >> 32);
                bound[q] = lower_bound_for_key<kBF16>(kth16);
            } else if (!(mode & SEL_CARRY)) {
                bound[q] = -INFINITY;  // refinement passes keep the previous (still valid) bound instead
            }
            if (!(mode & SEL_CARRY)) count[q] = 0;
        }
    }
}

// Candidate-list capacity per query: enough for the sampled bound of ~2*sqrt(k*n) rows and the sweep behind it.
inline uint32_t capq_for(int64_t n, int k) {
    const double s = sqrt(static_cast<double>(k) * static_cast<double>(n));
    uint64_t c = static_cast<uint64_t>(4.0 * s) + 1;
    if (c < 32768) c = 32768;
    c = (c + 1023) / 1024 * 1024;
    return static_cast<uint32_t>(c);
}

}  // namespace mips
