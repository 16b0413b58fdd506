// Beam selection of `FiD.generate(num_beams > 1)` (reference: src/atlas.py:592-619 -> transformers 4.18 `beam_search` with
// `BeamSearchScorer` / `BeamHypotheses`, early_stopping=False).  Two kernels per decode step, no host synchronisation; every
// step-dependent quantity (the step index, the beam scores, the hypotheses, the ancestry) lives in device memory, so one
// captured CUDA graph serves every step.
//
//   beam_topk_kernel     one block per beam row r = b * nb + beam.  Sweep 1: fp32 max and sum-exp of the 16-bit logits
//                        (online).  Sweep 2 (the row is L1/L2-resident): log-prob = (x - max) - log(sum), rounded to the
//                        16-bit type when asked (4.18's log_softmax returns the logits' dtype), EOS -> -inf while
//                        cur_len < min_length, + the optional additive mask (prefix constraint, 0 / -inf), + the row's fp32
//                        beam score; a per-thread top-K in registers, a warp merge, a block merge -> the row's top-2nb
//                        candidates.  Every candidate of the batch element's top-2nb is in its own row's top-2nb, so this
//                        pre-filter is exact.
//   beam_select_kernel   one block per batch element: merges its nb x 2nb candidates into the top-2nb (rank counting), then
//                        thread 0 runs `BeamSearchScorer.process` (EOS at rank < nb -> hypothesis, EOS at rank >= nb skipped,
//                        the other candidates fill the nb beams) and `BeamHypotheses.add` / `is_done` in fp64.  The block then
//                        copies the new hypotheses' tokens and rewrites the ancestry table of its rows.
//
// Order of candidates: the larger score first; NaN above every number; among equal scores (or NaNs) the lower flat index
// beam * V + token first (torch.topk leaves this undefined; the rule makes ties deterministic).
//
// Ancestry instead of a cache reorder: anc [2, R, Tmax] int32, buffer (t & 1) current at step t.  Entry (r, j) is the cache
// slot row that holds row r's position j: its self K | V at cache[anc[r, j], j] and its token at tok[anc[r, j], j].  After the
// selection anc'[r, :t+1] = anc[parent(r), :t+1], anc'[r, t+1] = r (the buffer of parity t + 1).  This replaces the
// reference's per-step index_select of every layer's cache (`_reorder_cache`, src/modeling_t5.py:1702).
#include "common.cuh"
#include "host_common.h"

#include <math.h>

namespace beam {

constexpr int TOPK_THREADS = 256;
constexpr int SELECT_THREADS = 256;
constexpr int MAX_BEAMS = ATLAS_B200_MAX_BEAMS;
constexpr int MAX_CAND = 2 * MAX_BEAMS;
constexpr int NO_INDEX = 0x7fffffff;

// (x, i) ranks above (y, j): NaN above every number, then the larger value; among equal values or among NaNs the lower index
__device__ __forceinline__ bool ranks_above(float x, int i, float y, int j) {
    const bool xn = isnan(x), yn = isnan(y);
    if (xn != yn) return xn;
    return x > y || ((xn || x == y) && i < j);
}

template <bool kBF16>
__device__ __forceinline__ float ld16(uint16_t v) {
    if constexpr (kBF16) return __uint_as_float(static_cast<uint32_t>(v) << 16);
    return __half2float(__ushort_as_half(v));
}

template <bool kBF16>
__device__ __forceinline__ float round16(float x) {
    if constexpr (kBF16) return __bfloat162float(__float2bfloat16_rn(x));
    return __half2float(__float2half_rn(x));
}

// running (max, sum of exp(x - max)) pairs; a -inf max carries a zero sum, a NaN anywhere makes the sum NaN
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
    const float mn = fmaxf(m, m2);
    if (mn == -INFINITY) return;
    s = s * expf(m - mn) + s2 * expf(m2 - mn);
    m = mn;
}

// grid = R rows, block = 256.  KK >= k: the per-thread list length (a power of two, kept in registers).
template <bool kBF16, int KK>
__global__ void __launch_bounds__(TOPK_THREADS)
beam_topk_kernel(const uint16_t* __restrict__ logits, int64_t ld, int V, const float* __restrict__ add_mask, int64_t ld_mask,
                 const float* __restrict__ beam_scores, const int32_t* __restrict__ t_dev, int eos, int min_length, int round_lp,
                 int k, float* __restrict__ cand_score, int32_t* __restrict__ cand_tok, float* __restrict__ lp_out) {
    const int r = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int WARPS = TOPK_THREADS / 32;
    const uint16_t* row = logits + static_cast<int64_t>(r) * ld;
    __shared__ float s_m[WARPS], s_s[WARPS];
    __shared__ float w_sc[WARPS][KK];
    __shared__ int w_ix[WARPS][KK];

    // sweep 1: max and sum-exp (fp32, online)
    float m = -INFINITY, s = 0.f;
    for (int v = threadIdx.x; v < V; v += TOPK_THREADS) {
        const float x = ld16<kBF16>(row[v]);
        if (isnan(x)) s = x;
        else lse_merge(m, s, x, 1.f);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, off), s2 = __shfl_xor_sync(0xffffffffu, s, off);
        if (isnan(s2)) s = s2;
        else if (!isnan(s)) lse_merge(m, s, m2, s2);
    }
    if (lane == 0) s_m[warp] = m, s_s[warp] = s;
    __syncthreads();
    m = s_m[0], s = s_s[0];
    for (int w = 1; w < WARPS; ++w) {
        if (isnan(s_s[w])) s = s_s[w];
        else if (!isnan(s)) lse_merge(m, s, s_m[w], s_s[w]);
    }
    const float log_sum = logf(s);       // all -inf: (x - max) is NaN everywhere, as torch's log_softmax gives

    // sweep 2: scores and the per-thread top-KK
    const int t = *t_dev;
    const bool ban_eos = t + 1 < min_length;                        // cur_len = t + 1
    const float bs = beam_scores[r];
    const float* mrow = add_mask ? add_mask + static_cast<int64_t>(r) * ld_mask : nullptr;
    float* lrow = lp_out ? lp_out + static_cast<int64_t>(r) * V : nullptr;
    float sc[KK];
    int ix[KK];
#pragma unroll
    for (int i = 0; i < KK; ++i) sc[i] = -INFINITY, ix[i] = NO_INDEX;
    for (int v = threadIdx.x; v < V; v += TOPK_THREADS) {
        float lp = (ld16<kBF16>(row[v]) - m) - log_sum;
        if (round_lp) lp = round16<kBF16>(lp);
        if (ban_eos && v == eos) lp = -INFINITY;
        if (mrow) lp += mrow[v];
        if (lrow) lrow[v] = lp;
        float x = lp + bs;
        int xi = v;
        if (!ranks_above(x, xi, sc[KK - 1], ix[KK - 1])) continue;
#pragma unroll
        for (int i = 0; i < KK; ++i) {                              // insertion into the sorted list, static indices only
            if (ranks_above(x, xi, sc[i], ix[i])) {
                const float ts = sc[i];
                const int ti = ix[i];
                sc[i] = x, ix[i] = xi;
                x = ts, xi = ti;
            }
        }
    }

    // warp merge: k rounds of "best head of the 32 lists, popped from its owner"
    for (int i = 0; i < k; ++i) {
        float bsc = sc[0];
        int bix = ix[0];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float os = __shfl_xor_sync(0xffffffffu, bsc, off);
            const int oi = __shfl_xor_sync(0xffffffffu, bix, off);
            if (ranks_above(os, oi, bsc, bix)) bsc = os, bix = oi;
        }
        if (bix != NO_INDEX && ix[0] == bix) {                       // token indices are unique across the lanes
#pragma unroll
            for (int j = 0; j < KK - 1; ++j) sc[j] = sc[j + 1], ix[j] = ix[j + 1];
            sc[KK - 1] = -INFINITY, ix[KK - 1] = NO_INDEX;
        }
        if (lane == 0) w_sc[warp][i] = bsc, w_ix[warp][i] = bix;
    }
    __syncthreads();

    // block merge: rank of each of the WARPS x k entries (equal entries, i.e. "no index" fillers, ordered by position)
    const int n = WARPS * k;
    for (int e = threadIdx.x; e < n; e += TOPK_THREADS) {
        const float x = w_sc[e / k][e % k];
        const int xi = w_ix[e / k][e % k];
        int rank = 0;
        for (int f = 0; f < n; ++f) {
            const float y = w_sc[f / k][f % k];
            const int yi = w_ix[f / k][f % k];
            rank += ranks_above(y, yi, x, xi) || (f < e && yi == xi && __float_as_uint(y) == __float_as_uint(x));
        }
        if (rank < k) {
            cand_score[static_cast<int64_t>(r) * k + rank] = x;
            cand_tok[static_cast<int64_t>(r) * k + rank] = xi;
        }
    }
}

// length_penalty normaliser cur_len ** lp, as Python computes it (exact for lp = 0, 1, 2, correctly rounded for 0.5)
__device__ __forceinline__ double lp_denominator(int cur_len, double lp) {
    const double x = static_cast<double>(cur_len);
    if (lp == 0.0) return 1.0;
    if (lp == 1.0) return x;
    if (lp == 2.0) return x * x;
    if (lp == 0.5) return sqrt(x);
    return pow(x, lp);
}

// grid = B, block = 256.
__global__ void __launch_bounds__(SELECT_THREADS)
beam_select_kernel(const float* __restrict__ cand_score, const int32_t* __restrict__ cand_tok, int nb, int V,
                   float* __restrict__ beam_scores, int64_t* __restrict__ tok_in, int32_t* __restrict__ parent,
                   uint8_t* __restrict__ done, int32_t* __restrict__ anc, int32_t* __restrict__ tok, int Tmax,
                   const int32_t* __restrict__ t_dev, double* __restrict__ hyp_score, int32_t* __restrict__ hyp_len,
                   int32_t* __restrict__ hyp_ins, int32_t* __restrict__ hyp_tok, int32_t* __restrict__ hyp_state,
                   double* __restrict__ hyp_worst, int eos, int pad, double length_penalty) {
    const int b = blockIdx.x;
    const int R = gridDim.x * nb;
    const int k = 2 * nb;
    const int t = *t_dev;
    const int cur_len = t + 1;
    if (t < 0 || t + 1 >= Tmax) return;                            // no position left to write
    const int32_t* anc_cur = anc + static_cast<int64_t>(t & 1) * R * Tmax;
    int32_t* anc_nxt = anc + static_cast<int64_t>((t + 1) & 1) * R * Tmax;
    __shared__ float c_sc[MAX_BEAMS * MAX_CAND];
    __shared__ int c_flat[MAX_BEAMS * MAX_CAND];
    __shared__ float top_sc[MAX_CAND];
    __shared__ int top_flat[MAX_CAND];
    __shared__ float n_sc[MAX_BEAMS];
    __shared__ int n_tok[MAX_BEAMS], n_par[MAX_BEAMS], h_src[MAX_BEAMS];
    const bool was_done = done[b] != 0;

    if (!was_done) {
        const int n = nb * k;
        for (int e = threadIdx.x; e < n; e += SELECT_THREADS) {
            const int64_t g = static_cast<int64_t>(b) * n + e;       // rows b*nb .. b*nb+nb-1 are consecutive
            const int tk = cand_tok[g];
            c_sc[e] = cand_score[g];
            c_flat[e] = tk == NO_INDEX ? NO_INDEX : (e / k) * V + tk;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < n; e += SELECT_THREADS) {
            const float x = c_sc[e];
            const int xi = c_flat[e];
            int rank = 0;
            for (int f = 0; f < n; ++f)
                rank += ranks_above(c_sc[f], c_flat[f], x, xi) ||
                        (f < e && c_flat[f] == xi && __float_as_uint(c_sc[f]) == __float_as_uint(x));
            if (rank < k) top_sc[rank] = x, top_flat[rank] = xi;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            // BeamSearchScorer.process for this batch element (hypothesis list order = insertion number order)
            double* hs = hyp_score + static_cast<int64_t>(b) * nb;
            int32_t* hl = hyp_len + static_cast<int64_t>(b) * nb;
            int32_t* hi = hyp_ins + static_cast<int64_t>(b) * nb;
            int count = hyp_state[2 * b], next_ins = hyp_state[2 * b + 1];
            double worst = hyp_worst[b];
            const double denom = lp_denominator(cur_len, length_penalty);
            for (int i = 0; i < nb; ++i) h_src[i] = -1;
            int filled = 0;
            for (int rank = 0; rank < k && filled < nb; ++rank) {
                const int flat = top_flat[rank];
                const int bm = flat / V, tk = flat % V;
                const int prow = b * nb + bm;
                if (tk == eos) {
                    if (rank >= nb) continue;
                    const double score = static_cast<double>(top_sc[rank]) / denom;
                    if (count < nb || score > worst) {
                        if (count < nb) {                                // append
                            const int slot = count++;
                            hs[slot] = score, hl[slot] = cur_len, hi[slot] = next_ins++;
                            h_src[slot] = prow;
                            worst = worst < score ? worst : score;       // Python's min(score, worst)
                        } else {
                            // append then delete the lowest (score, list index): the earliest inserted among equal
                            // scores.  score > worst = the lowest score, so the new one survives and takes that slot.
                            int slot = 0;
                            for (int j = 0; j < nb; ++j) {
                                const bool earlier = hi[j] < hi[slot];
                                if (hs[j] < hs[slot] || (hs[j] == hs[slot] && earlier)) slot = j;
                            }
                            hs[slot] = score, hl[slot] = cur_len, hi[slot] = next_ins++;
                            h_src[slot] = prow;
                            worst = hs[0];                               // the second lowest before = the lowest now
                            for (int j = 1; j < nb; ++j) worst = hs[j] < worst ? hs[j] : worst;
                        }
                    }
                } else {
                    n_sc[filled] = top_sc[rank], n_tok[filled] = tk, n_par[filled] = prow;
                    ++filled;
                }
            }
            const double best = static_cast<double>(top_sc[0]) / denom;
            if (count == nb && worst >= best) done[b] = 1;
            hyp_state[2 * b] = count, hyp_state[2 * b + 1] = next_ins;
            hyp_worst[b] = worst;
        }
    } else if (threadIdx.x < nb) {                                   // finished: pad tokens, score 0, rows stay in place
        n_sc[threadIdx.x] = 0.f, n_tok[threadIdx.x] = pad, n_par[threadIdx.x] = b * nb + threadIdx.x;
        h_src[threadIdx.x] = -1;
    }
    __syncthreads();

    // the new hypotheses' tokens (positions 0 .. t of the parent, through the current ancestry) and the new ancestry rows
    for (int e = threadIdx.x; e < nb * (t + 2); e += SELECT_THREADS) {
        const int i = e / (t + 2), j = e % (t + 2);
        const int r = b * nb + i;
        if (j <= t) {
            const int p = n_par[i];
            anc_nxt[static_cast<int64_t>(r) * Tmax + j] = anc_cur[static_cast<int64_t>(p) * Tmax + j];
            const int hp = h_src[i];
            if (hp >= 0) {
                const int src = anc_cur[static_cast<int64_t>(hp) * Tmax + j];
                hyp_tok[static_cast<int64_t>(r) * Tmax + j] = tok[static_cast<int64_t>(src) * Tmax + j];
            }
        } else {
            anc_nxt[static_cast<int64_t>(r) * Tmax + j] = r;
            tok[static_cast<int64_t>(r) * Tmax + j] = n_tok[i];
        }
    }
    if (threadIdx.x < nb) {
        const int r = b * nb + threadIdx.x;
        beam_scores[r] = n_sc[threadIdx.x];
        tok_in[r] = n_tok[threadIdx.x];
        parent[r] = n_par[threadIdx.x];
    }
}

__global__ void advance_step_kernel(int32_t* t_dev) { *t_dev += 1; }

template <bool kBF16>
int launch_topk(int KK, dim3 grid, cudaStream_t s, const uint16_t* logits, int64_t ld, int V, const float* add_mask,
                int64_t ld_mask, const float* beam_scores, const int32_t* t_dev, int eos, int min_length, int round_lp, int k,
                float* cand_score, int32_t* cand_tok, float* lp_out) {
#define AB_BEAM_TOPK(K_)                                                                                                 \
    beam_topk_kernel<kBF16, K_><<<grid, TOPK_THREADS, 0, s>>>(logits, ld, V, add_mask, ld_mask, beam_scores, t_dev, eos, \
                                                              min_length, round_lp, k, cand_score, cand_tok, lp_out)
    if (KK <= 4) AB_BEAM_TOPK(4);
    else if (KK <= 8) AB_BEAM_TOPK(8);
    else if (KK <= 16) AB_BEAM_TOPK(16);
    else AB_BEAM_TOPK(32);
#undef AB_BEAM_TOPK
    return 0;
}

}  // namespace beam

extern "C" {

int atlas_b200_beam_topk(const void* logits, int64_t ld, int32_t V, const float* add_mask, int64_t ld_mask,
                         const float* beam_scores, const int32_t* t_dev, int32_t eos_id, int32_t min_length, int32_t round_lp,
                         int32_t k, float* cand_score, int32_t* cand_tok, float* lp_out, int32_t R, int32_t is_bf16,
                         void* stream) {
    AB_REQUIRE(R >= 0 && V > 0 && k > 0 && k <= beam::MAX_CAND && t_dev != nullptr && beam_scores != nullptr &&
                   cand_score != nullptr && cand_tok != nullptr,
               "beam_topk: bad arguments (R=%d V=%d k=%d; k must be in [1, %d])", R, V, k, beam::MAX_CAND);
    if (R == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    abh::prof_begin(s, abh::PROF_BEAM_SELECT);
    if (is_bf16)
        beam::launch_topk<true>(k, dim3(R), s, static_cast<const uint16_t*>(logits), ld, V, add_mask, ld_mask, beam_scores,
                                t_dev, eos_id, min_length, round_lp, k, cand_score, cand_tok, lp_out);
    else
        beam::launch_topk<false>(k, dim3(R), s, static_cast<const uint16_t*>(logits), ld, V, add_mask, ld_mask, beam_scores,
                                 t_dev, eos_id, min_length, round_lp, k, cand_score, cand_tok, lp_out);
    abh::prof_end(s, abh::PROF_BEAM_SELECT, 2.0 * R * static_cast<double>(V));     // = 16-bit logit bytes read
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int atlas_b200_beam_select(const float* cand_score, const int32_t* cand_tok, int32_t B, int32_t nb, int32_t V,
                           float* beam_scores, int64_t* tok_in, int32_t* parent, uint8_t* done, int32_t* anc, int32_t* tok,
                           int32_t Tmax, int32_t* t_dev, double* hyp_score, int32_t* hyp_len, int32_t* hyp_ins,
                           int32_t* hyp_tok, int32_t* hyp_state, double* hyp_worst, int32_t eos_id, int32_t pad_id,
                           double length_penalty, void* stream) {
    AB_REQUIRE(B >= 0 && nb >= 1 && nb <= beam::MAX_BEAMS && V >= 2 && Tmax >= 1 && t_dev != nullptr,
               "beam_select: bad arguments (B=%d nb=%d V=%d Tmax=%d; need 1 <= nb <= %d, V >= 2)", B, nb, V, Tmax,
               beam::MAX_BEAMS);
    AB_REQUIRE(B <= 65535, "beam_select: grid too large");
    if (B == 0) return ATLAS_B200_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    abh::prof_begin(s, abh::PROF_BEAM_SELECT);
    beam::beam_select_kernel<<<B, beam::SELECT_THREADS, 0, s>>>(cand_score, cand_tok, nb, V, beam_scores, tok_in, parent, done,
                                                               anc, tok, Tmax, t_dev, hyp_score, hyp_len, hyp_ins, hyp_tok,
                                                               hyp_state, hyp_worst, eos_id, pad_id, length_penalty);
    abh::prof_end(s, abh::PROF_BEAM_SELECT, 8.0 * B * nb * 2.0 * nb);                // = candidate bytes read
    beam::advance_step_kernel<<<1, 1, 0, s>>>(t_dev);
    abh::count_launch(2);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // extern "C"
