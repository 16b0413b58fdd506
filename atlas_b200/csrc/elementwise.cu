// Row-wise normalisation, embedding and pooling kernels of the Contriever / FiD forward pass.
// HBM-bound byte work: one warp per row, 16-byte vector loads/stores, fp32 statistics in registers,
// warp-shuffle reductions; nothing is re-read.  Rounding points follow the reference exactly:
//
//   bert_layernorm   BertLayerNorm.forward, src/modeling_bert.py:104-114 (callers pass `.float()` input,
//                    :245,386,465):  xn = (x - mean(x)) * rsqrt(mean(x^2) + eps)   [fp32, UNCENTRED 2nd moment]
//                                    y  = w * half(xn) + b                          [two 16-bit roundings]
//   t5_rmsnorm       T5LayerNorm.forward, src/modeling_t5.py:244-253:
//                                    y  = w * half(x * rsqrt(mean(x^2) + eps))
//   bert_embed_ln    BertEmbeddings.forward, src/modeling_bert.py:213-247: word + token_type (+= position),
//                    16-bit adds in that order, then BertLayerNorm on the fp32 copy
//   masked_mean_pool Contriever.forward, src/retrievers.py:50-53: masked_fill(~mask, 0).sum(1) / mask.sum(1)
//                    (sum accumulated in fp32 and rounded once, then one 16-bit division)
#include "common.cuh"
#include "host_common.h"

namespace ew {

constexpr int MAXV = 8;  // 16-byte vectors per lane -> rows of up to 8*32*8 = 2048 elements

template <bool kBF16>
__device__ __forceinline__ float lo(uint32_t w) {
    if constexpr (kBF16) return __bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(w & 0xFFFFu)));
    return __half2float(__ushort_as_half(static_cast<unsigned short>(w & 0xFFFFu)));
}
template <bool kBF16>
__device__ __forceinline__ float hi(uint32_t w) {
    if constexpr (kBF16) return __bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(w >> 16)));
    return __half2float(__ushort_as_half(static_cast<unsigned short>(w >> 16)));
}
template <bool kBF16>
__device__ __forceinline__ uint32_t rnd(float v) {
    if constexpr (kBF16) return __bfloat16_as_ushort(__float2bfloat16_rn(v));
    return __half_as_ushort(__float2half_rn(v));
}
template <bool kBF16>
__device__ __forceinline__ float rf(float v) {  // round through the 16-bit type
    if constexpr (kBF16) return __bfloat162float(__float2bfloat16_rn(v));
    return __half2float(__float2half_rn(v));
}

template <bool kBF16>
__device__ __forceinline__ uint32_t pack2_rn(float a, float b) {   // lo = a, hi = b
    uint32_t d;
    if constexpr (kBF16) {
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(b), "f"(a));
    } else {
        asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(b), "f"(a));
    }
    return d;
}
template <bool kBF16>
__device__ __forceinline__ uint32_t mul2(uint32_t a, uint32_t b) {
    uint32_t d;
    if constexpr (kBF16) {
        asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    } else {
        asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    }
    return d;
}
template <bool kBF16>
__device__ __forceinline__ uint32_t add2(uint32_t a, uint32_t b) {
    uint32_t d;
    if constexpr (kBF16) {
        asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    } else {
        asm("add.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    }
    return d;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// y = w * r16(norm(x)) (+ b), all products/sums rounded to 16 bits like torch's half kernels
template <bool kBF16, bool kCentre, bool kBias>
__device__ __forceinline__ void norm_row(float (&v)[MAXV][8], int nvec, int H, float eps, const uint16_t* w,
                                         const uint16_t* b, uint16_t* y, int lane) {
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
        if (lane + 32 * i < nvec)
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                s1 += v[i][e];
                s2 += v[i][e] * v[i][e];
            }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    const float mean = kCentre ? s1 / static_cast<float>(H) : 0.f;
    const float rstd = rsqrtf(s2 / static_cast<float>(H) + eps);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vec = lane + 32 * i;
        if (vec < nvec) {
            const uint4 wv = __ldg(reinterpret_cast<const uint4*>(w) + vec);
            const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
            uint32_t bb[4] = {0, 0, 0, 0};
            if (kBias) {
                const uint4 bv = __ldg(reinterpret_cast<const uint4*>(b) + vec);
                bb[0] = bv.x; bb[1] = bv.y; bb[2] = bv.z; bb[3] = bv.w;
            }
            uint32_t o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                // r16(norm) for two elements with one packed conversion (F2FP, ALU pipe), then the 16-bit multiply /
                // add of the reference's half kernels as native x2 instructions (products of two 16-bit values are
                // exact in fp32, so HMUL2's single rounding equals round16(fp32 product))
                const uint32_t n2 = pack2_rn<kBF16>((v[i][2 * e] - mean) * rstd, (v[i][2 * e + 1] - mean) * rstd);
                uint32_t y2 = mul2<kBF16>(ww[e], n2);
                if (kBias) y2 = add2<kBF16>(y2, bb[e]);
                o[e] = y2;
            }
            reinterpret_cast<uint4*>(y)[vec] = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

template <bool kBF16, bool kCentre, bool kBias>
__global__ void __launch_bounds__(256)
layernorm_kernel(const uint16_t* __restrict__ x, int64_t ldx, const uint16_t* __restrict__ w,
                 const uint16_t* __restrict__ b, uint16_t* __restrict__ y, int64_t ldy, int rows, int H, float eps) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int nvec = H >> 3;
    float v[MAXV][8];
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (lane + 32 * i < nvec) {
            const uint4 t = __ldg(xr + lane + 32 * i);
            const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                v[i][2 * e] = lo<kBF16>(tw[e]);
                v[i][2 * e + 1] = hi<kBF16>(tw[e]);
            }
        }
    }
    norm_row<kBF16, kCentre, kBias>(v, nvec, H, eps, w, b, y + row * ldy, lane);
}

template <bool kBF16>
__global__ void __launch_bounds__(256)
bert_embed_ln_kernel(const int64_t* __restrict__ input_ids, const int64_t* __restrict__ token_type_ids,
                     const uint16_t* __restrict__ word_emb, const uint16_t* __restrict__ type_emb,
                     const uint16_t* __restrict__ pos_emb, const uint16_t* __restrict__ w,
                     const uint16_t* __restrict__ b, uint16_t* __restrict__ y, int rows, int L, int H, float eps) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int nvec = H >> 3;
    const int64_t tok = input_ids[row];
    const int64_t typ = token_type_ids ? token_type_ids[row] : 0;
    const int pos = row % L;  // position_ids = arange(L) (modeling_bert.py:223-224)
    const uint4* we = reinterpret_cast<const uint4*>(word_emb + tok * H);
    const uint4* te = reinterpret_cast<const uint4*>(type_emb + typ * H);
    const uint4* pe = reinterpret_cast<const uint4*>(pos_emb + static_cast<int64_t>(pos) * H);
    float v[MAXV][8];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (lane + 32 * i < nvec) {
            const uint4 a = __ldg(we + lane + 32 * i), c = __ldg(te + lane + 32 * i), d = __ldg(pe + lane + 32 * i);
            const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, cw[4] = {c.x, c.y, c.z, c.w}, dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                // embeddings = inputs_embeds + token_type_embeddings; embeddings += position_embeddings (16-bit)
                v[i][2 * e] = rf<kBF16>(rf<kBF16>(lo<kBF16>(aw[e]) + lo<kBF16>(cw[e])) + lo<kBF16>(dw[e]));
                v[i][2 * e + 1] = rf<kBF16>(rf<kBF16>(hi<kBF16>(aw[e]) + hi<kBF16>(cw[e])) + hi<kBF16>(dw[e]));
            }
        }
    }
    norm_row<kBF16, true, true>(v, nvec, H, eps, w, b, y + static_cast<int64_t>(row) * H, lane);
}

// out[b, :] = sum_l mask[b,l] * x[b,l,:] / sum_l mask[b,l]; one block per (b, 256-column slab)
template <bool kBF16>
__global__ void __launch_bounds__(256)
masked_mean_pool_kernel(const uint16_t* __restrict__ x, const int64_t* __restrict__ mask, uint16_t* __restrict__ out,
                        int64_t ld_out, int L, int H) {
    const int b = blockIdx.x;
    const int col = blockIdx.y * blockDim.x + threadIdx.x;
    if (col >= H) return;
    float acc = 0.f;
    int64_t cnt = 0;
    for (int l = 0; l < L; ++l) {
        const int64_t m = mask[static_cast<int64_t>(b) * L + l];
        cnt += (m != 0);
        if (m != 0) {
            const uint16_t h = x[(static_cast<int64_t>(b) * L + l) * H + col];
            acc += kBF16 ? __bfloat162float(__ushort_as_bfloat16(h)) : __half2float(__ushort_as_half(h));
        }
    }
    const float s = rf<kBF16>(acc);                                  // last_hidden.sum(dim=1) in 16 bits
    out[b * ld_out + col] = static_cast<uint16_t>(rnd<kBF16>(s / static_cast<float>(cnt)));
}


// Reader-input assembly from the device-resident passage token bank (replaces the per-step host work of
// Atlas.tokenize_passages, src/atlas.py:261-280: bsz x n_context string formats + tokenizer calls):
//   row (b, j) = (query_ids[b, :qlen[b]] ++ bank_ids[rows[b, j], :bank_lens[...]])[: L - 1] ++ [eos], padded with `pad`
// and the attention mask of the same shape.  rows[b, j] < 0 is the "" padding passage: EOS only (src/atlas.py:26-39).
// One block per output row; 4-byte reads, 8-byte id + 1-byte mask writes (pure HBM byte work: L * 13 B per row).
__global__ void splice_tokens_kernel(const int32_t* __restrict__ bank_ids, const int32_t* __restrict__ bank_lens,
                                     int64_t bank_ld, int64_t bank_rows, const int64_t* __restrict__ rows,
                                     const int64_t* __restrict__ query_ids, const int32_t* __restrict__ query_lens,
                                     int64_t ldq, int n_ctx, int L, int eos, int pad, int64_t* __restrict__ out_ids,
                                     uint8_t* __restrict__ out_mask) {
    const int r = blockIdx.x;                 // output row = b * n_ctx + j
    const int b = r / n_ctx;
    int64_t row = rows[r];
    if (row >= bank_rows) row = -1;           // unknown passage id: treated like the padding passage
    int qlen = 0, plen = 0;
    if (row >= 0) {
        qlen = query_lens ? query_lens[b] : 0;
        plen = bank_lens[row];
    }
    const int body = min(qlen + plen, L - 1);  // tokens before the closing EOS
    const int32_t* prow = bank_ids + (row >= 0 ? row : 0) * bank_ld;
    const int64_t* qrow = query_ids ? query_ids + static_cast<int64_t>(b) * ldq : nullptr;
    int64_t* o = out_ids + static_cast<int64_t>(r) * L;
    uint8_t* m = out_mask + static_cast<int64_t>(r) * L;
    for (int t = threadIdx.x; t < L; t += blockDim.x) {
        int64_t v = pad;
        uint8_t on = 0;
        if (t < body) {
            v = t < qlen ? qrow[t] : static_cast<int64_t>(prow[t - qlen]);
            on = 1;
        } else if (t == body) {
            v = eos;
            on = 1;
        }
        o[t] = v;
        m[t] = on;
    }
}

// ---- fp16 overflow clamp of the T5 blocks (src/modeling_t5.py:657-708) ----------------------------------------------
// The reference runs, after the self-attention, cross-attention and feed-forward sub-layers of every block,
//     if hidden_states.dtype == torch.float16 and torch.isinf(hidden_states).any():
//         hidden_states = torch.clamp(hidden_states, min=-(finfo.max - 1000), max=finfo.max - 1000)
// i.e. three host synchronisations per block.  Here: a detect pass raises a device flag, the clamp pass reads it and leaves
// at once when it is clear - same values, no synchronisation, capturable in a CUDA graph.  65504 - 1000 rounds to 64512
// (0x7BE0) in fp16; NaNs stay NaNs (torch.clamp propagates them).
// rows the clamp looks at: min(max(*m_dev, 0), M), or all M without a device count (read on the device, so a captured graph
// follows the count of every replay).  Rows past it were never computed by the producing GEMM: neither read nor written.
__device__ __forceinline__ int64_t rows_in(int64_t M, const int32_t* m_dev) {
    if (m_dev == nullptr) return M;
    const int64_t m = *m_dev;
    return m < 0 ? 0 : (m < M ? m : M);
}

__global__ void __launch_bounds__(256)
inf_detect_kernel(const uint16_t* __restrict__ x, int64_t ld, int64_t M, const int32_t* __restrict__ m_dev, int N,
                  int* __restrict__ flag) {
    const int vec_per_row = N / 8;
    const int64_t nvec = rows_in(M, m_dev) * vec_per_row;
    bool found = false;
    for (int64_t v = blockIdx.x * 256ll + threadIdx.x; v < nvec; v += gridDim.x * 256ll) {
        const uint4 w = __ldg(reinterpret_cast<const uint4*>(x + (v / vec_per_row) * ld + (v % vec_per_row) * 8));
        const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) found |= ((ws[e] & 0x7FFFu) == 0x7C00u) | ((ws[e] & 0x7FFF0000u) == 0x7C000000u);
    }
    if (__any_sync(0xffffffffu, found) && (threadIdx.x & 31) == 0) atomicOr(flag, 1);
}

// one warp per row; only runs its body when the flag is raised.  row_ss (optional): the row's sum of squares of the clamped
// values, the statistic the fused RMSNorm of the next GEMM consumes (the GEMM that produced x accumulated it from the
// un-clamped values, inf included).
__global__ void __launch_bounds__(256)
inf_clamp_kernel(uint16_t* __restrict__ x, int64_t ld, int64_t M, const int32_t* __restrict__ m_dev, int N,
                 const int* __restrict__ flag, float* __restrict__ row_ss) {
    if (*flag == 0) return;
    M = rows_in(M, m_dev);
    const int lane = threadIdx.x & 31;
    for (int64_t row = blockIdx.x * 8ll + (threadIdx.x >> 5); row < M; row += gridDim.x * 8ll) {
        uint16_t* xr = x + row * ld;
        float ss = 0.f;
        for (int c = lane * 2; c < N; c += 64) {
            uint32_t w = *reinterpret_cast<uint32_t*>(xr + c);
            uint32_t o = 0;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                uint32_t h = (w >> (16 * e)) & 0xFFFFu;
                const uint32_t mag = h & 0x7FFFu;
                if (mag <= 0x7C00u && mag > 0x7BE0u) h = (h & 0x8000u) | 0x7BE0u;     // finite-or-inf above the bound; NaN kept
                const float f = __half2float(__ushort_as_half(static_cast<unsigned short>(h)));
                ss = fmaf(f, f, ss);
                o |= h << (16 * e);
            }
            *reinterpret_cast<uint32_t*>(xr + c) = o;
        }
        if (row_ss != nullptr) {
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
            if (lane == 0) row_ss[row] = ss;
        }
    }
}

// ---- compaction of the live 64-row tiles of a [rows, d] matrix (FiD decoder: only the encoder positions whose 64-key block holds a
// live key are ever read by the cross-attention, so only they get a K | V projection) --------------------------------------
// scan: tile_off[t] = number of live tiles before t (-1 for a dead tile), *count_rows = 64 x (number of live tiles)
__global__ void __launch_bounds__(1024)
live_tile_scan_kernel(const uint8_t* __restrict__ live, int n_tiles, int32_t* __restrict__ tile_off,
                      int32_t* __restrict__ count_rows) {
    __shared__ int s_warp[32];
    __shared__ int s_base;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    for (int t0 = 0; t0 < n_tiles; t0 += 1024) {
        const int t = t0 + static_cast<int>(threadIdx.x);
        const int f = (t < n_tiles && live[t] != 0) ? 1 : 0;
        int x = f;                                           // inclusive scan inside the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (static_cast<int>(threadIdx.x & 31u) >= o) x += y;
        }
        if ((threadIdx.x & 31u) == 31u) s_warp[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int w = s_warp[threadIdx.x];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, w, o);
                if (static_cast<int>(threadIdx.x) >= o) w += y;
            }
            s_warp[threadIdx.x] = w;                         // inclusive prefix over the warps
        }
        __syncthreads();
        const int before = s_base + (threadIdx.x >= 32 ? s_warp[(threadIdx.x >> 5) - 1] : 0) + x - f;
        if (t < n_tiles) tile_off[t] = f ? before : -1;
        __syncthreads();
        if (threadIdx.x == 0) s_base += s_warp[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) *count_rows = s_base * 64;
}

// copy: block t moves the 64 rows of live tile t to rows [64 tile_off[t], +64) of dst (16-byte vectors)
__global__ void __launch_bounds__(256)
live_tile_copy_kernel(const uint16_t* __restrict__ src, int64_t lds, const int32_t* __restrict__ tile_off,
                      uint16_t* __restrict__ dst, int64_t ldd, int d) {
    const int t = blockIdx.x;
    const int off = tile_off[t];
    if (off < 0) return;
    const int vec_per_row = d / 8;
    for (int v = threadIdx.x; v < 64 * vec_per_row; v += 256) {
        const int r = v / vec_per_row, c = (v % vec_per_row) * 8;
        *reinterpret_cast<uint4*>(dst + (static_cast<int64_t>(off) * 64 + r) * ldd + c) =
            __ldg(reinterpret_cast<const uint4*>(src + (static_cast<int64_t>(t) * 64 + r) * lds + c));
    }
}

// ---- padding-compacted encoder (fid.py: encode_compact): every segment (FiD passage) keeps its 64-row tiles up to the last one
// that holds a live key; the kept tiles of all segments are packed back to back ------------------------------------------------
// One block.  live [S, nb] -> keep [S, nb] (1 for tiles 0 .. last live tile of the segment; all nb tiles if none is live),
// tile_off [S * nb] (index of a kept tile in the packed order, -1 = dropped), tile_src [S * nb] (inverse: source tile of packed
// tile o, -1 past the end), *count_rows = 64 x (number of kept tiles).
__global__ void __launch_bounds__(1024)
segment_tile_scan_kernel(const uint8_t* __restrict__ live, int S, int nb, uint8_t* __restrict__ keep, int32_t* __restrict__ tile_off,
                         int32_t* __restrict__ tile_src, int32_t* __restrict__ count_rows) {
    __shared__ int s_warp[32];
    __shared__ int s_base;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    for (int s0 = 0; s0 < S; s0 += 1024) {
        const int sg = s0 + static_cast<int>(threadIdx.x);
        int f = 0;                                           // tiles this segment keeps
        if (sg < S) {
            for (int j = 0; j < nb; ++j)
                if (live[static_cast<size_t>(sg) * nb + j] != 0) f = j + 1;
            if (f == 0) f = nb;
        }
        int x = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (static_cast<int>(threadIdx.x & 31u) >= o) x += y;
        }
        if ((threadIdx.x & 31u) == 31u) s_warp[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int w = s_warp[threadIdx.x];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, w, o);
                if (static_cast<int>(threadIdx.x) >= o) w += y;
            }
            s_warp[threadIdx.x] = w;
        }
        __syncthreads();
        const int before = s_base + (threadIdx.x >= 32 ? s_warp[(threadIdx.x >> 5) - 1] : 0) + x - f;
        if (sg < S) {
            for (int j = 0; j < nb; ++j) {
                const int t = sg * nb + j;
                keep[t] = j < f ? 1 : 0;
                tile_off[t] = j < f ? before + j : -1;
                if (j < f) tile_src[before + j] = t;
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) s_base += s_warp[31];
        __syncthreads();
    }
    const int total = s_base;
    for (int o = total + static_cast<int>(threadIdx.x); o < S * nb; o += 1024) tile_src[o] = -1;
    if (threadIdx.x == 0) *count_rows = total * 64;
}

// block o writes packed tile o: the embedding rows of the 64 token ids of its source tile, zeros past the end
__global__ void __launch_bounds__(256)
embed_packed_tiles_kernel(const int64_t* __restrict__ ids, const uint16_t* __restrict__ table, int64_t ldt, int vocab,
                          const int32_t* __restrict__ tile_src, uint16_t* __restrict__ dst, int64_t ldd, int d) {
    const int o = blockIdx.x;
    const int src = tile_src[o];
    const int vec_per_row = d / 8;
    for (int v = threadIdx.x; v < 64 * vec_per_row; v += 256) {
        const int r = v / vec_per_row, c = (v % vec_per_row) * 8;
        uint4 val = make_uint4(0u, 0u, 0u, 0u);
        if (src >= 0) {
            int64_t id = __ldg(ids + static_cast<int64_t>(src) * 64 + r);
            id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
            val = __ldg(reinterpret_cast<const uint4*>(table + id * ldt + c));
        }
        *reinterpret_cast<uint4*>(dst + (static_cast<int64_t>(o) * 64 + r) * ldd + c) = val;
    }
}

// block t writes source tile t of the padded layout: its packed rows, zeros for a dropped tile
__global__ void __launch_bounds__(256)
expand_packed_tiles_kernel(const uint16_t* __restrict__ src, int64_t lds, const int32_t* __restrict__ tile_off,
                           uint16_t* __restrict__ dst, int64_t ldd, int d) {
    const int t = blockIdx.x;
    const int off = tile_off[t];
    const int vec_per_row = d / 8;
    for (int v = threadIdx.x; v < 64 * vec_per_row; v += 256) {
        const int r = v / vec_per_row, c = (v % vec_per_row) * 8;
        uint4 val = make_uint4(0u, 0u, 0u, 0u);
        if (off >= 0) val = __ldg(reinterpret_cast<const uint4*>(src + (static_cast<int64_t>(off) * 64 + r) * lds + c));
        *reinterpret_cast<uint4*>(dst + (static_cast<int64_t>(t) * 64 + r) * ldd + c) = val;
    }
}

}  // namespace ew

extern "C" {

int atlas_b200_segment_tile_scan(const uint8_t* live, int32_t S, int32_t nb, uint8_t* keep, int32_t* tile_off, int32_t* tile_src,
                                 int32_t* count_rows, void* stream) {
    AB_REQUIRE(S > 0 && nb > 0 && nb <= 64 && live != nullptr && keep != nullptr && tile_off != nullptr && tile_src != nullptr &&
                   count_rows != nullptr, "segment_tile_scan: S > 0, 0 < nb <= 64, all tables required");
    ew::segment_tile_scan_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(live, S, nb, keep, tile_off, tile_src, count_rows);
    abh::count_launch(1);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_embed_packed_tiles(const int64_t* ids, const void* table, int64_t ldt, int32_t vocab, const int32_t* tile_src,
                                  int32_t n_tiles, void* dst, int64_t ldd, int32_t d, void* stream) {
    AB_REQUIRE(n_tiles >= 0 && vocab > 0 && d > 0 && d % 8 == 0 && ldt % 8 == 0 && ldd % 8 == 0 && ids != nullptr && tile_src != nullptr,
               "embed_packed_tiles: d and the strides must be multiples of 8");
    AB_REQUIRE(abh::aligned(table, 16) && abh::aligned(dst, 16), "embed_packed_tiles: table and dst must be 16-byte aligned");
    if (n_tiles == 0) return ATLAS_B200_OK;
    ew::embed_packed_tiles_kernel<<<n_tiles, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        ids, static_cast<const uint16_t*>(table), ldt, vocab, tile_src, static_cast<uint16_t*>(dst), ldd, d);
    abh::count_launch(1);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_expand_packed_tiles(const void* src, int64_t lds, const int32_t* tile_off, int32_t n_tiles, void* dst, int64_t ldd,
                                   int32_t d, void* stream) {
    AB_REQUIRE(n_tiles >= 0 && d > 0 && d % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0 && tile_off != nullptr,
               "expand_packed_tiles: d and the strides must be multiples of 8");
    AB_REQUIRE(abh::aligned(src, 16) && abh::aligned(dst, 16), "expand_packed_tiles: src and dst must be 16-byte aligned");
    if (n_tiles == 0) return ATLAS_B200_OK;
    ew::expand_packed_tiles_kernel<<<n_tiles, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint16_t*>(src), lds, tile_off, static_cast<uint16_t*>(dst), ldd, d);
    abh::count_launch(1);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_compact_live_tiles(const void* src, int64_t lds, const uint8_t* tile_live, int32_t n_tiles, int32_t d, void* dst,
                                  int64_t ldd, int32_t* tile_off, int32_t* count_rows, void* stream) {
    AB_REQUIRE(n_tiles >= 0 && d > 0 && d % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0 && tile_off != nullptr && count_rows != nullptr,
               "compact_live_tiles: d and the strides must be multiples of 8");
    AB_REQUIRE(abh::aligned(src, 16) && abh::aligned(dst, 16), "compact_live_tiles: src and dst must be 16-byte aligned");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    ew::live_tile_scan_kernel<<<1, 1024, 0, s>>>(tile_live, n_tiles, tile_off, count_rows);
    if (n_tiles > 0)
        ew::live_tile_copy_kernel<<<n_tiles, 256, 0, s>>>(static_cast<const uint16_t*>(src), lds, tile_off,
                                                          static_cast<uint16_t*>(dst), ldd, d);
    abh::count_launch(2);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_clamp_inf_fp16(void* x, int64_t ld, int64_t M, int32_t N, const int32_t* m_dev, int32_t* flag, float* row_ss,
                              void* stream) {
    AB_REQUIRE(M >= 0 && N > 0 && N % 8 == 0 && ld % 8 == 0 && flag != nullptr, "clamp_inf_fp16: N and ld must be multiples of 8");
    AB_REQUIRE(abh::aligned(x, 16), "clamp_inf_fp16: x must be 16-byte aligned");
    if (M == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    AB_CUDA_CHECK(cudaMemsetAsync(flag, 0, sizeof(int32_t), s));
    const int64_t blocks = (M * (N / 8) + 255) / 256;
    const int64_t cap = static_cast<int64_t>(abh::num_sms()) * 16;
    ew::inf_detect_kernel<<<static_cast<unsigned>(blocks < cap ? blocks : cap), 256, 0, s>>>(
        static_cast<const uint16_t*>(x), ld, M, m_dev, N, flag);
    const int64_t rb = (M + 7) / 8;
    ew::inf_clamp_kernel<<<static_cast<unsigned>(rb < cap ? rb : cap), 256, 0, s>>>(static_cast<uint16_t*>(x), ld, M, m_dev, N,
                                                                                   flag, row_ss);
    abh::count_launch(2);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_layernorm(const void* x, int64_t ldx, const void* weight, const void* bias, void* y, int64_t ldy,
                         int32_t rows, int32_t H, float eps, int32_t kind, int32_t is_bf16, void* stream) {
    AB_REQUIRE(rows >= 0 && H > 0 && H % 8 == 0 && H <= ew::MAXV * 256, "layernorm: H=%d must be a multiple of 8, <= %d",
               H, ew::MAXV * 256);
    AB_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0, "layernorm: row strides must be multiples of 8");
    AB_REQUIRE(kind == 0 || kind == 1, "layernorm: kind must be 0 (BertLayerNorm) or 1 (T5 RMSNorm)");
    AB_REQUIRE(kind == 1 || bias != nullptr, "BertLayerNorm needs a bias");
    AB_REQUIRE(abh::aligned(x, 16) && abh::aligned(weight, 16) && abh::aligned(bias, 16) && abh::aligned(y, 16),
               "layernorm: x, weight, bias and y must be 16-byte aligned");
    if (rows == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = (rows + 7) / 8;
    const uint16_t *xp = static_cast<const uint16_t*>(x), *wp = static_cast<const uint16_t*>(weight),
                   *bp = static_cast<const uint16_t*>(bias);
    uint16_t* yp = static_cast<uint16_t*>(y);
    if (kind == 0) {
        if (is_bf16) ew::layernorm_kernel<true, true, true><<<grid, 256, 0, s>>>(xp, ldx, wp, bp, yp, ldy, rows, H, eps);
        else ew::layernorm_kernel<false, true, true><<<grid, 256, 0, s>>>(xp, ldx, wp, bp, yp, ldy, rows, H, eps);
    } else {
        if (is_bf16) ew::layernorm_kernel<true, false, false><<<grid, 256, 0, s>>>(xp, ldx, wp, bp, yp, ldy, rows, H, eps);
        else ew::layernorm_kernel<false, false, false><<<grid, 256, 0, s>>>(xp, ldx, wp, bp, yp, ldy, rows, H, eps);
    }
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_bert_embed_ln(const int64_t* input_ids, const int64_t* token_type_ids, const void* word_emb,
                             const void* type_emb, const void* pos_emb, const void* ln_weight, const void* ln_bias,
                             void* y, int32_t batch, int32_t L, int32_t H, float eps, int32_t is_bf16, void* stream) {
    AB_REQUIRE(batch >= 0 && L > 0 && H > 0 && H % 8 == 0 && H <= ew::MAXV * 256, "bert_embed_ln: bad shape");
    AB_REQUIRE(abh::aligned(word_emb, 16) && abh::aligned(type_emb, 16) && abh::aligned(pos_emb, 16) &&
                   abh::aligned(ln_weight, 16) && abh::aligned(ln_bias, 16) && abh::aligned(y, 16),
               "bert_embed_ln: the tables, weight, bias and y must be 16-byte aligned");
    const int rows = batch * L;
    if (rows == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = (rows + 7) / 8;
    const uint16_t *we = static_cast<const uint16_t*>(word_emb), *te = static_cast<const uint16_t*>(type_emb),
                   *pe = static_cast<const uint16_t*>(pos_emb), *w = static_cast<const uint16_t*>(ln_weight),
                   *b = static_cast<const uint16_t*>(ln_bias);
    if (is_bf16)
        ew::bert_embed_ln_kernel<true><<<grid, 256, 0, s>>>(input_ids, token_type_ids, we, te, pe, w, b,
                                                            static_cast<uint16_t*>(y), rows, L, H, eps);
    else
        ew::bert_embed_ln_kernel<false><<<grid, 256, 0, s>>>(input_ids, token_type_ids, we, te, pe, w, b,
                                                             static_cast<uint16_t*>(y), rows, L, H, eps);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_masked_mean_pool(const void* x, const int64_t* mask, void* out, int64_t ld_out, int32_t batch, int32_t L,
                                int32_t H, int32_t is_bf16, void* stream) {
    AB_REQUIRE(batch >= 0 && L > 0 && H > 0, "masked_mean_pool: bad shape");
    if (batch == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid(batch, (H + 255) / 256);
    if (is_bf16)
        ew::masked_mean_pool_kernel<true><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(x), mask,
                                                               static_cast<uint16_t*>(out), ld_out, L, H);
    else
        ew::masked_mean_pool_kernel<false><<<grid, 256, 0, s>>>(static_cast<const uint16_t*>(x), mask,
                                                                static_cast<uint16_t*>(out), ld_out, L, H);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_splice_tokens(const int32_t* bank_ids, const int32_t* bank_lens, int64_t bank_ld, int64_t bank_rows,
                             const int64_t* rows, const int64_t* query_ids, const int32_t* query_lens, int64_t ldq,
                             int32_t batch, int32_t n_ctx, int32_t L, int32_t eos_id, int32_t pad_id, int64_t* out_ids,
                             uint8_t* out_mask, void* stream) {
    AB_REQUIRE(batch >= 0 && n_ctx > 0 && L > 1 && bank_ld > 0 && bank_rows >= 0, "splice_tokens: bad shape");
    AB_REQUIRE((query_ids == nullptr) == (query_lens == nullptr), "splice_tokens: query ids and lengths come together");
    if (batch == 0) return ATLAS_B200_OK;
    ew::splice_tokens_kernel<<<batch * n_ctx, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        bank_ids, bank_lens, bank_ld, bank_rows, rows, query_ids, query_lens, ldq, n_ctx, L, eos_id, pad_id, out_ids,
        out_mask);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
