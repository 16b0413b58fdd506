// Product-quantized passage index (`--index_mode faiss`, types pq and ivfpq) for sm_90a.
//
// Replaces faiss's IndexPQ / GpuIndexIVFPQ behind `DistributedFAISSIndex` (src/index.py:163-381):
//   pq     a row x [768] is stored as M one-byte codes; code m is the nearest (L2) of 256 centroids of the m-th
//          sub-vector x[m*dsub, (m+1)*dsub), dsub = 768 / M.  score(q, x) = sum_m <q_m, cb_m[code_m]>.
//   ivfpq  n_list coarse centroids (inner-product assignment); the residual x - c_list is product-quantized.
//          score(q, x) = sum_m <q_m, cb_m[code_m]> + <q, c_list>.  The reference probes every list
//          (nprobe = n_list, src/index.py:212,269), so the search is a full scan of these scores.
//
// Training (one call, both quantizers): faiss's k-means defaults - the caller passes a training sample in a seeded random
// order (<= 256 points per centroid), the first k rows are the initial centroids, `iters` Lloyd iterations, an empty
// cluster is re-seeded by splitting the largest one with a symmetric 1/1024 perturbation.  Deterministic: assignments are
// argmin / argmax with the lowest index on ties, centroid sums run over the members in sample order (no float atomics).
//   coarse assignment  the wgmma GEMM atlas_b200_linear_rows (fp16 rows x fp16 copy of the centroids) + a row argmax
//   PQ assignment      ||c||^2 - 2 <r, c> in fp32 on CUDA cores (pq_subdot_kernel + pq_argmin_kernel), residuals in fp32
//
// Search per block of <= 256 queries: fp32 lookup tables LUT[q][m][256] (and coarse terms T[q][list] for ivfpq) from the
// fp16 queries, then mips.cu's exact top-k pipeline on the scores of a code sweep:
//   sample sweep -> bound (mips_select_kernel) -> full sweep with the bound -> select + emit, `status` on overflow,
//   and the chunked exhaustive variant.  Scores accumulate in fp32 over m = 0..M-1, then + T, and are rounded ONCE to fp16.
// Scan kernel: one row per thread, QPC queries per CTA whose LUTs (and coarse terms) sit in shared memory for the whole
// sweep; a row's codes are read once per query group.
//
// The IVF-SQ index (type ivfsq) shares the coarse k-means, the coarse assignment and the top-k driver: its training,
// encoding and search host code are at the end of this file, its scan kernel in ivfsq.cu.  The IVF-Flat index (types
// ivfflat and flat) trains with ivfsq's entry point (coarse quantizer only) and shares the driver and the probe
// selection; its search host code follows ivfsq's, its scan kernel is in ivfflat.cu.
#include "ivf_probe.cuh"
#include "ivfflat.cuh"
#include "ivfsq.cuh"
#include "mips_select.cuh"

#include <math.h>

namespace pq {

constexpr int DIM = ATLAS_B200_EMBEDDINGS_DIM;
constexpr int KSUB = 256;             // 8-bit codes
constexpr int QBLOCK = 256;           // queries per select block (mips.cu's candidate layout)
constexpr int PQ_TRAIN_MAX = 256 * KSUB;
constexpr int SCAN_THREADS = 512;     // rows per scan tile
constexpr int SCAN_SMEM_MAX = 200 * 1024;
constexpr size_t CHUNK_BUDGET = 128ull << 20;   // per-chunk scratch of training / encoding
constexpr float SPLIT_EPS = 1.0f / 1024.0f;

inline bool valid_m(int M) { return M >= 1 && DIM % M == 0 && DIM / M >= 8; }
inline int pad8(int x) { return (x + 7) / 8 * 8; }

// ---------------------------------------------------------------------------------------------
// elementwise helpers
// ---------------------------------------------------------------------------------------------
// out[i, :] = float(x[i, :]) - (coarse ? coarse[assign[i], :] : 0)
__global__ void pq_residual_kernel(const __half* __restrict__ x, int64_t n, const float* __restrict__ coarse,
                                   const int32_t* __restrict__ assign, float* __restrict__ out) {
    const int64_t total = n * DIM;
    for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < total;
         e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t i = e / DIM;
        const int d = static_cast<int>(e - i * DIM);
        float v = __half2float(x[e]);
        if (coarse) v -= coarse[static_cast<int64_t>(assign[i]) * DIM + d];
        out[e] = v;
    }
}

// dst[r, :] = src[r, :] for r < rows (fp32 rows of width `width`, source stride lds, destination stride ldd)
__global__ void pq_copy_rows_kernel(const float* __restrict__ src, int64_t lds, float* __restrict__ dst, int64_t ldd,
                                    int rows, int width, int src_col_step, int64_t dst_block_step) {
    // grid.y = block m: dst block m (dst + m * dst_block_step) takes columns [m * src_col_step, + width) of src
    const int m = blockIdx.y;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < rows * width; e += gridDim.x * blockDim.x) {
        const int r = e / width, d = e - r * width;
        dst[m * dst_block_step + static_cast<int64_t>(r) * ldd + d] = src[static_cast<int64_t>(r) * lds + m * src_col_step + d];
    }
}

__global__ void pq_half_to_float_kernel(const __half* __restrict__ x, int64_t count, float* __restrict__ out) {
    for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < count;
         e += static_cast<int64_t>(gridDim.x) * blockDim.x)
        out[e] = __half2float(x[e]);
}

// norms[b] = sum_d c[b, d]^2 over nb rows of width D
__global__ void pq_norms_kernel(const float* __restrict__ c, int nb, int D, float* __restrict__ norms) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    float s = 0.f;
    for (int d = 0; d < D; ++d) s = fmaf(c[static_cast<int64_t>(b) * D + d], c[static_cast<int64_t>(b) * D + d], s);
    norms[b] = s;
}

// ---------------------------------------------------------------------------------------------
// out[i][m][j] = sum_{d < dsub} A[i, m*dsub + d] * B[m][j][d]   (fp32, d ascending, fmaf)
// 64 x 64 output tile per CTA, 4 x 4 per thread.  Serves the LUTs (B = codebooks), the coarse terms (M = 1, B = centroids)
// and the PQ distances of training / encoding.
// ---------------------------------------------------------------------------------------------
constexpr int SD_T = 64, SD_KC = 16;

__global__ void __launch_bounds__(256) pq_subdot_kernel(const float* __restrict__ A, int64_t lda, int rows,
                                                        const float* __restrict__ B, int nb, int dsub, int M,
                                                        float* __restrict__ out) {
    __shared__ float As[SD_KC][SD_T];
    __shared__ float Bs[SD_KC][SD_T + 1];
    const int m = blockIdx.z;
    const int i0 = blockIdx.y * SD_T, j0 = blockIdx.x * SD_T;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const float* Bm = B + static_cast<int64_t>(m) * nb * dsub;
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
    for (int d0 = 0; d0 < dsub; d0 += SD_KC) {
        for (int e = threadIdx.x; e < SD_T * SD_KC; e += 256) {
            const int r = e / SD_KC, kk = e % SD_KC;
            const int d = d0 + kk;
            const int i = i0 + r, j = j0 + r;
            As[kk][r] = (i < rows && d < dsub) ? A[static_cast<int64_t>(i) * lda + m * dsub + d] : 0.f;
            Bs[kk][r] = (j < nb && d < dsub) ? Bm[static_cast<int64_t>(j) * dsub + d] : 0.f;
        }
        __syncthreads();
        const int kmax = min(SD_KC, dsub - d0);
        for (int kk = 0; kk < kmax; ++kk) {
            float a[4], b[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) a[r] = As[kk][ty + 16 * r];
#pragma unroll
            for (int c = 0; c < 4; ++c) b[c] = Bs[kk][tx + 16 * c];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(a[r], b[c], acc[r][c]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int i = i0 + ty + 16 * r;
        if (i >= rows) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int j = j0 + tx + 16 * c;
            if (j < nb) out[(static_cast<int64_t>(i) * M + m) * nb + j] = acc[r][c];
        }
    }
}

// codes[i, m] = argmin_j (norms[m][j] - 2 dots[i][m][j]), lowest j on ties.  One warp per (i, m), grid-stride.
__global__ void pq_argmin_kernel(const float* __restrict__ dots, const float* __restrict__ norms, int64_t rows, int M,
                                 uint8_t* __restrict__ codes) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t w = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5; w < rows * M; w += warps) {
        const int m = static_cast<int>(w % M);
        const float* dv = dots + w * KSUB;
        float best = INFINITY;
        int bj = KSUB;
#pragma unroll
        for (int t = 0; t < KSUB / 32; ++t) {
            const int j = lane + 32 * t;
            const float v = norms[m * KSUB + j] - 2.0f * dv[j];
            if (v < best) { best = v; bj = j; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (ob < best || (ob == best && oj < bj)) { best = ob; bj = oj; }
        }
        if (lane == 0) codes[w] = static_cast<uint8_t>(bj < KSUB ? bj : 0);
    }
}

// assign[i] = argmax_{l < n_list} scores[i, l] (16-bit GEMM output, row stride ld), lowest l on ties; one warp per row.
// Optionally also writes the list id in its storage type (uint16 when n_list <= 65535, else int32).  Grid-stride.
__global__ void pq_argmax_rows_kernel(const __half* __restrict__ scores, int64_t ld, int64_t rows, int n_list,
                                      int32_t* __restrict__ assign, void* __restrict__ lists, int list_u16) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t i = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5; i < rows; i += warps) {
        const __half* s = scores + i * ld;
        float best = -INFINITY;
        int bl = n_list;
        for (int l = lane; l < n_list; l += 32) {
            const float v = __half2float(s[l]);
            if (bl == n_list || v > best) { best = v; bl = l; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
            if (ol < n_list && (bl >= n_list || ob > best || (ob == best && ol < bl))) { best = ob; bl = ol; }
        }
        if (lane == 0) {
            if (bl >= n_list) bl = 0;
            if (assign) assign[i] = bl;
            if (lists) {
                if (list_u16) static_cast<uint16_t*>(lists)[i] = static_cast<uint16_t>(bl);
                else static_cast<int32_t*>(lists)[i] = bl;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// k-means update: one CTA per (cluster c, block m).  Members are collected in sample order 256 rows at a time and summed
// in that order, so the centroids are bitwise reproducible.  Empty clusters keep their centroid (split below).
//   X rows of width D at column m * D (row stride ldx); assign[i * lda + m] = cluster of row i in block m.
// ---------------------------------------------------------------------------------------------
template <typename XT, typename AT>
__global__ void __launch_bounds__(256) pq_update_kernel(const XT* __restrict__ X, int64_t ldx, const AT* __restrict__ assign,
                                                        int lda, int S, int K, int D, float* __restrict__ cent,
                                                        int32_t* __restrict__ counts) {
    __shared__ int32_t s_idx[256];
    __shared__ int32_t s_warp[8];
    const int c = blockIdx.x, m = blockIdx.y;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    constexpr int PER = (DIM + 255) / 256;
    float acc[PER];
#pragma unroll
    for (int r = 0; r < PER; ++r) acc[r] = 0.f;
    int cnt = 0;
    for (int base = 0; base < S; base += 256) {
        const int i = base + t;
        const bool flag = i < S && static_cast<int>(assign[static_cast<int64_t>(i) * lda + m]) == c;
        const uint32_t bal = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) s_warp[w] = __popc(bal);
        __syncthreads();
        int off = 0, tot = 0;
#pragma unroll
        for (int w2 = 0; w2 < 8; ++w2) {
            off += w2 < w ? s_warp[w2] : 0;
            tot += s_warp[w2];
        }
        if (flag) s_idx[off + __popc(bal & ((1u << lane) - 1u))] = i;
        __syncthreads();
        for (int j = 0; j < tot; ++j) {
            const XT* row = X + static_cast<int64_t>(s_idx[j]) * ldx + static_cast<int64_t>(m) * D;
#pragma unroll
            for (int r = 0; r < PER; ++r) {
                const int d = t + 256 * r;
                if (d < D) acc[r] += static_cast<float>(row[d]);
            }
        }
        cnt += tot;
        __syncthreads();
    }
    float* cc = cent + (static_cast<int64_t>(m) * K + c) * D;
    if (cnt > 0) {
        const float inv = 1.0f / static_cast<float>(cnt);
#pragma unroll
        for (int r = 0; r < PER; ++r) {
            const int d = t + 256 * r;
            if (d < D) cc[d] = acc[r] * inv;
        }
    }
    if (t == 0) counts[static_cast<int64_t>(m) * K + c] = cnt;
}

// Empty clusters of block m = blockIdx.x, in index order: copy the currently largest cluster (lowest index on ties) with a
// symmetric perturbation (even dims *(1 + eps) / *(1 - eps), odd dims the other way round) and split its count.
__global__ void __launch_bounds__(256) pq_split_kernel(float* __restrict__ cent, int32_t* __restrict__ counts, int K, int D) {
    __shared__ int32_t s_best[256], s_bidx[256];
    const int m = blockIdx.x, t = threadIdx.x;
    float* cm = cent + static_cast<int64_t>(m) * K * D;
    int32_t* nm = counts + static_cast<int64_t>(m) * K;
    for (int c = 0; c < K; ++c) {
        __syncthreads();
        if (nm[c] != 0) continue;
        int best = -1, bidx = K;
        for (int j = t; j < K; j += 256)
            if (nm[j] > best) { best = nm[j]; bidx = j; }
        s_best[t] = best;
        s_bidx[t] = bidx;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if (t < o) {
                const int ob = s_best[t + o], oi = s_bidx[t + o];
                if (ob > s_best[t] || (ob == s_best[t] && oi < s_bidx[t])) { s_best[t] = ob; s_bidx[t] = oi; }
            }
            __syncthreads();
        }
        const int cj = s_bidx[0];
        if (cj >= K || s_best[0] <= 0) continue;
        for (int d = t; d < D; d += 256) {
            const float v = cm[static_cast<int64_t>(cj) * D + d];
            const float up = v * (1.0f + SPLIT_EPS), dn = v * (1.0f - SPLIT_EPS);
            cm[static_cast<int64_t>(c) * D + d] = (d % 2 == 0) ? up : dn;
            cm[static_cast<int64_t>(cj) * D + d] = (d % 2 == 0) ? dn : up;
        }
        __syncthreads();
        if (t == 0) {
            const int half = nm[cj] / 2;
            nm[c] = half;
            nm[cj] -= half;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// scan: one row per thread; LUTs (+ coarse terms) of QPC queries in shared memory; candidates in mips.cu's format
// ---------------------------------------------------------------------------------------------
struct ScanParams {
    const uint8_t* codes;    // [n, M]
    const void* lists;       // [n] uint16 / int32 (ivfpq) or nullptr (pq)
    int list_u16;
    int n_rows;
    int M;
    const float* lut;        // [QBLOCK][M][256]
    const float* cterm;      // [QBLOCK][n_list] or nullptr
    int n_list;
    int cterm_smem;          // coarse terms staged in shared memory
    int nq;                  // valid queries in this block
    int tile_begin, tile_step, num_tiles;
    const float* bound;
    uint32_t* count;
    uint64_t* cand;
    uint32_t capq;
};

// A probed scan's state (a separate kernel argument: the full scan's parameters stay as they are)
struct ProbeScan {
    const int2* items;             // (list, first list position) chunks of PROBE_CHUNK positions, and their count
    const int32_t* item_count;
    const int32_t* list_order;     // rows in list order (stable) and each list's first position [n_list + 1]
    const int32_t* list_offsets;
    const uint32_t* probed;        // [n_list][PROBE_WORDS] probe bits of the block's queries
};

constexpr int PROBE_CHUNK = SCAN_THREADS;   // list positions per work item of a probed scan: one per thread

// PROBED: a work item is one chunk of one list (ivf_probe.cuh), so the list, its coarse terms and the probe bits of the
// CTA's queries are known once per item; an item none of them probes is skipped, and a row is appended for query q only
// when q probes its list.
template <int QPC, bool PROBED>
__global__ void __launch_bounds__(SCAN_THREADS) pq_scan_kernel(const ScanParams p, const ProbeScan pr) {
    extern __shared__ float s_tab[];
    __shared__ float s_bnd[QPC];
    const int t = threadIdx.x, lane = t & 31;
    const int q0 = blockIdx.y * QPC;
    const int nqg = min(QPC, p.nq - q0);
    const int M = p.M;
    const int lut_q = M * KSUB;
    for (int e = t; e < nqg * lut_q; e += SCAN_THREADS) s_tab[e] = p.lut[static_cast<int64_t>(q0) * lut_q + e];
    float* s_ct = s_tab + QPC * lut_q;
    if (p.cterm && p.cterm_smem)
        for (int e = t; e < nqg * p.n_list; e += SCAN_THREADS) s_ct[e] = p.cterm[static_cast<int64_t>(q0) * p.n_list + e];
    if (t < QPC) s_bnd[t] = t < nqg ? p.bound[q0 + t] : INFINITY;
    __syncthreads();
    int begin = p.tile_begin, step = p.tile_step, num = p.num_tiles;
    if constexpr (PROBED) ivfp::resolve_items(*pr.item_count, p.tile_begin, p.tile_step, p.num_tiles, begin, step, num);

    for (int it = blockIdx.x; it < num; it += gridDim.x) {
        int row, l = 0;
        bool live;
        if constexpr (PROBED) {
            const int2 item = pr.items[begin + it * step];
            l = item.x;
            if (!ivfp::group_probes(pr.probed, l, q0, nqg)) continue;
            const int pos = item.y + t;
            live = pos < __ldg(pr.list_offsets + l + 1);
            row = live ? __ldg(pr.list_order + pos) : 0;
        } else {
            row = (begin + it * step) * SCAN_THREADS + t;
            live = row < p.n_rows;
        }
        float acc[QPC];
#pragma unroll
        for (int q = 0; q < QPC; ++q) acc[q] = 0.f;
        if (live) {
            const uint8_t* c = p.codes + static_cast<int64_t>(row) * M;
            if ((M & 3) == 0) {
                const uint32_t* cw = reinterpret_cast<const uint32_t*>(c);
                for (int wi = 0; wi < M / 4; ++wi) {
                    const uint32_t word = __ldg(cw + wi);
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        const int off = (4 * wi + b) * KSUB + ((word >> (8 * b)) & 0xFFu);
#pragma unroll
                        for (int q = 0; q < QPC; ++q) acc[q] += s_tab[q * lut_q + off];
                    }
                }
            } else {
                for (int m = 0; m < M; ++m) {
                    const int off = m * KSUB + __ldg(c + m);
#pragma unroll
                    for (int q = 0; q < QPC; ++q) acc[q] += s_tab[q * lut_q + off];
                }
            }
            if (p.cterm) {
                if constexpr (!PROBED)
                    l = p.list_u16 ? static_cast<int>(static_cast<const uint16_t*>(p.lists)[row])
                                   : static_cast<const int32_t*>(p.lists)[row];
#pragma unroll
                for (int q = 0; q < QPC; ++q)
                    if (q < nqg)
                        acc[q] += p.cterm_smem ? s_ct[q * p.n_list + l]
                                               : p.cterm[static_cast<int64_t>(q0 + q) * p.n_list + l];
            }
        }
#pragma unroll
        for (int q = 0; q < QPC; ++q) {
            if (q >= nqg) break;
            const bool pass = live && (!PROBED || ivfp::probes(pr.probed, l, q0 + q)) && acc[q] >= s_bnd[q];
            const uint32_t bal = __ballot_sync(0xffffffffu, pass);
            if (bal == 0) continue;
            const int leader = __ffs(bal) - 1;
            uint32_t base = 0;
            if (lane == leader) base = atomicAdd(&p.count[q0 + q], static_cast<uint32_t>(__popc(bal)));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (pass) {
                const uint32_t pos = base + __popc(bal & ((1u << lane) - 1u));
                if (pos < p.capq)
                    p.cand[static_cast<size_t>(q0 + q) * p.capq + pos] =
                        mips::pack_candidate(mips::bits_to_key(mips::round_to_bits<false>(acc[q])), static_cast<uint32_t>(row));
            }
        }
    }
}

__global__ void pq_prep_kernel(uint32_t* __restrict__ count, float* __restrict__ bound) {
    if (threadIdx.x < QBLOCK) {
        count[threadIdx.x] = 0;
        bound[threadIdx.x] = -INFINITY;
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int grid_1d(int64_t work, int threads) {
    int64_t b = (work + threads - 1) / threads;
    if (b > 8192) b = 8192;
    return static_cast<int>(b < 1 ? 1 : b);
}

struct Carver {
    uint8_t* base;
    size_t off = 0;
    template <typename T>
    T* take(size_t count) {
        const size_t o = off;
        off = abh::align_up(off + count * sizeof(T), 256);
        return base ? reinterpret_cast<T*>(base + o) : nullptr;
    }
};

// rows per chunk of training / encoding: GEMM scores + assignment + residuals + PQ distances of one chunk in the budget
static int64_t chunk_rows(int M, int n_list) {
    const size_t per_row = static_cast<size_t>(M) * KSUB * 4 + static_cast<size_t>(pad8(n_list)) * 2 + DIM * 4 + 4;
    int64_t r = static_cast<int64_t>(CHUNK_BUDGET / per_row);
    if (r > 65536) r = 65536;
    r = r / 64 * 64;
    return r < 64 ? 64 : r;
}

struct ChunkWs {
    __half* gemm;      // [R][pad8(n_list)]
    int32_t* assign;   // [R]
    float* resid;      // [R][768]
    float* dots;       // [R][M][256]
    __half* coarse16;  // [pad8(n_list)][768]
    float* norms;      // [M][256]
};

static void carve_chunk(Carver& cv, ChunkWs& w, int M, int n_list) {
    const int64_t R = chunk_rows(M, n_list);
    const int nlp = pad8(n_list);
    w.gemm = cv.take<__half>(n_list > 0 ? static_cast<size_t>(R) * nlp : 0);
    w.assign = cv.take<int32_t>(R);
    w.resid = cv.take<float>(static_cast<size_t>(R) * DIM);
    w.dots = cv.take<float>(static_cast<size_t>(R) * M * KSUB);
    w.coarse16 = cv.take<__half>(static_cast<size_t>(nlp) * DIM);
    w.norms = cv.take<float>(static_cast<size_t>(M) * KSUB);
}

static size_t train_bytes(int64_t S, int M, int n_list, ChunkWs* w, float** resid_all, uint8_t** codes_t, int32_t** counts,
                          int32_t** assign_all, void* base) {
    Carver cv{static_cast<uint8_t*>(base)};
    ChunkWs tmp;
    carve_chunk(cv, w ? *w : tmp, M, n_list);
    const int64_t sp = S < PQ_TRAIN_MAX ? S : PQ_TRAIN_MAX;
    float* r = cv.take<float>(static_cast<size_t>(sp) * DIM);
    uint8_t* c = cv.take<uint8_t>(static_cast<size_t>(sp) * M);
    int32_t* n = cv.take<int32_t>(static_cast<size_t>(M) * KSUB > static_cast<size_t>(n_list) ? static_cast<size_t>(M) * KSUB
                                                                                            : static_cast<size_t>(n_list));
    int32_t* a = cv.take<int32_t>(static_cast<size_t>(S));
    if (resid_all) *resid_all = r;
    if (codes_t) *codes_t = c;
    if (counts) *counts = n;
    if (assign_all) *assign_all = a;
    return cv.off;
}

static size_t encode_bytes(int M, int n_list, ChunkWs* w, void* base) {
    Carver cv{static_cast<uint8_t*>(base)};
    ChunkWs tmp;
    carve_chunk(cv, w ? *w : tmp, M, n_list);
    return cv.off;
}

struct SearchWs {
    uint32_t* count;
    float* bound;
    uint64_t* cand;
    uint32_t capq;
    float* qf32;   // [QBLOCK][768]
    float* lut;    // [QBLOCK][M][256]
    float* cterm;  // [QBLOCK][n_list]
};

// A probed search (nprobe < n_list) takes the tables of its lists and carves its probe state after the search scratch.
struct ProbeArgs {
    int nprobe;
    const int32_t* list_order;     // ivfpq: rows in list order (stable), [n]
    const int32_t* list_offsets;   // ivfpq: first list position of every list, [n_list + 1]; ivfsq: first tile
    const int32_t* list_rows;      // ivfsq: real rows of every list, [n_list]
};

struct ProbeWs {
    uint32_t* probed;         // [n_list][PROBE_WORDS]
    uint32_t* sample_lists;   // [n_list]
    int2* items;              // [max_items]
    int2* sample;             // [max_sample]
    int32_t* count;           // [2]: items, sample items
    int sample_units;         // sampled items at the front of a sample list
    int64_t max_sample;
};

// Each sample list contributes its first max(PROBE_CHUNK, k) positions (ivf_probe.cuh), in whole units.
static int sample_units(int k, int unit) { return ((k > PROBE_CHUNK ? k : PROBE_CHUNK) + unit - 1) / unit; }

static size_t probe_bytes(size_t off, int n_list, int64_t max_items, int k, int unit, ProbeWs* w, void* base) {
    Carver cv{static_cast<uint8_t*>(base), off};
    const int su = sample_units(k, unit);
    const int64_t max_sample = static_cast<int64_t>(n_list) * su < max_items ? static_cast<int64_t>(n_list) * su : max_items;
    uint32_t* probed = cv.take<uint32_t>(static_cast<size_t>(n_list) * ivfp::PROBE_WORDS);
    uint32_t* sample_lists = cv.take<uint32_t>(static_cast<size_t>(n_list));
    int2* items = cv.take<int2>(static_cast<size_t>(max_items));
    int2* sample = cv.take<int2>(static_cast<size_t>(max_sample));
    int32_t* count = cv.take<int32_t>(2);
    if (w) *w = ProbeWs{probed, sample_lists, items, sample, count, su, max_sample};
    return cv.off;
}

// ivfpq: chunks of PROBE_CHUNK positions, at most one partial chunk per list
static int64_t pq_max_items(int64_t n, int n_list) { return (n + PROBE_CHUNK - 1) / PROBE_CHUNK + n_list; }

static size_t search_bytes(int64_t n, int M, int n_list, int k, SearchWs* w, void* base) {
    Carver cv{static_cast<uint8_t*>(base)};
    const uint32_t capq = mips::capq_for(n, k);
    uint32_t* count = cv.take<uint32_t>(QBLOCK);
    float* bound = cv.take<float>(QBLOCK);
    uint64_t* cand = cv.take<uint64_t>(static_cast<size_t>(QBLOCK) * capq);
    float* qf = cv.take<float>(static_cast<size_t>(QBLOCK) * DIM);
    float* lut = cv.take<float>(static_cast<size_t>(QBLOCK) * M * KSUB);
    float* ct = cv.take<float>(static_cast<size_t>(QBLOCK) * (n_list > 0 ? n_list : 0));
    if (w) *w = SearchWs{count, bound, cand, capq, qf, lut, ct};
    return cv.off;
}

static int subdot(const float* A, int64_t lda, int rows, const float* B, int nb, int dsub, int M, float* out, cudaStream_t s) {
    if (rows <= 0) return ATLAS_B200_OK;
    dim3 grid((nb + SD_T - 1) / SD_T, (rows + SD_T - 1) / SD_T, M);
    pq_subdot_kernel<<<grid, 256, 0, s>>>(A, lda, rows, B, nb, dsub, M, out);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

static int residual(const __half* x, int64_t n, const float* coarse, const int32_t* assign, float* out, cudaStream_t s) {
    if (n <= 0) return ATLAS_B200_OK;
    pq_residual_kernel<<<grid_1d(n * DIM, 256), 256, 0, s>>>(x, n, coarse, assign, out);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

// fp16 copy of the coarse centroids for the GEMM, zero rows up to a multiple of 8
static int coarse_to_half(const float* coarse, int n_list, __half* out, cudaStream_t s) {
    const int nlp = pad8(n_list);
    if (nlp > n_list)
        AB_CUDA_CHECK(cudaMemsetAsync(out + static_cast<size_t>(n_list) * DIM, 0, static_cast<size_t>(nlp - n_list) * DIM * 2, s));
    return atlas_b200_cast_f32(coarse, out, static_cast<int64_t>(n_list) * DIM, 0, s);
}

// coarse assignment of rows [n] (inner product, GEMM + argmax), in chunks of R rows
static int coarse_assign(const __half* x, int64_t n, const __half* coarse16, int n_list, const ChunkWs& w, int64_t R,
                         int32_t* assign, void* lists, int list_u16, cudaStream_t s) {
    const int nlp = pad8(n_list);
    for (int64_t r0 = 0; r0 < n; r0 += R) {
        const int rows = static_cast<int>(n - r0 < R ? n - r0 : R);
        int rc = atlas_b200_linear_rows(x + r0 * DIM, DIM, coarse16, DIM, nullptr, nullptr, 0, w.gemm, nlp, rows, nlp, DIM, 0, 0,
                                        nullptr, nullptr, 0.f, nullptr, s);
        if (rc) return rc;
        pq_argmax_rows_kernel<<<grid_1d(static_cast<int64_t>(rows) * 32, 256), 256, 0, s>>>(
            w.gemm, nlp, rows, n_list, assign ? assign + r0 : nullptr,
            lists ? static_cast<void*>(static_cast<uint8_t*>(lists) + r0 * (list_u16 ? 2 : 4)) : nullptr, list_u16);
        abh::count_launch();
        AB_CUDA_CHECK(cudaGetLastError());
    }
    return ATLAS_B200_OK;
}

// PQ codes of fp32 rows [n][768] (residuals), in chunks of R rows; norms must hold the codebook norms
static int pq_assign(const float* rows32, int64_t n, int M, const float* codebooks, const ChunkWs& w, int64_t R, uint8_t* codes,
                     cudaStream_t s) {
    const int dsub = DIM / M;
    for (int64_t r0 = 0; r0 < n; r0 += R) {
        const int rows = static_cast<int>(n - r0 < R ? n - r0 : R);
        int rc = subdot(rows32 + r0 * DIM, DIM, rows, codebooks, KSUB, dsub, M, w.dots, s);
        if (rc) return rc;
        pq_argmin_kernel<<<grid_1d(static_cast<int64_t>(rows) * M * 32, 256), 256, 0, s>>>(w.dots, w.norms, rows, M,
                                                                                          codes + r0 * M);
        abh::count_launch();
        AB_CUDA_CHECK(cudaGetLastError());
    }
    return ATLAS_B200_OK;
}

static int codebook_norms(const float* codebooks, int M, float* norms, cudaStream_t s) {
    pq_norms_kernel<<<(M * KSUB + 255) / 256, 256, 0, s>>>(codebooks, M * KSUB, DIM / M, norms);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

// Coarse quantizer (ivfpq, ivfsq): inner-product k-means on the first min(S, 256 n_list) sample rows (n_list >= 1,
// S >= n_list); the first n_list rows are the initial centroids.  Leaves the fp16 copy of the result in w.coarse16.
static int coarse_kmeans(const __half* sample, int64_t S, int n_list, int iters, float* coarse, const ChunkWs& w, int64_t R,
                         int32_t* assign, int32_t* counts, cudaStream_t s) {
    int rc;
    const int64_t sc = S < static_cast<int64_t>(n_list) * KSUB ? S : static_cast<int64_t>(n_list) * KSUB;
    pq_half_to_float_kernel<<<grid_1d(static_cast<int64_t>(n_list) * DIM, 256), 256, 0, s>>>(
        sample, static_cast<int64_t>(n_list) * DIM, coarse);
    abh::count_launch();
    for (int it = 0; it < iters; ++it) {
        if ((rc = coarse_to_half(coarse, n_list, w.coarse16, s))) return rc;
        if ((rc = coarse_assign(sample, sc, w.coarse16, n_list, w, R, assign, nullptr, 0, s))) return rc;
        pq_update_kernel<__half, int32_t><<<dim3(n_list, 1), 256, 0, s>>>(sample, DIM, assign, 1, static_cast<int>(sc),
                                                                        n_list, DIM, coarse, counts);
        pq_split_kernel<<<1, 256, 0, s>>>(coarse, counts, n_list, DIM);
        abh::count_launch(2);
        AB_CUDA_CHECK(cudaGetLastError());
    }
    return coarse_to_half(coarse, n_list, w.coarse16, s);
}

static int check_shape(int M, int n_list) {
    AB_REQUIRE(valid_m(M), "code_size M=%d is not supported: M must divide 768 with 768 / M >= 8 "
               "(1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64, 96)", M);
    AB_REQUIRE(n_list >= 0, "n_list=%d must be >= 0 (0 = pq without a coarse quantizer)", n_list);
    return ATLAS_B200_OK;
}

static int train(const __half* sample, int64_t S, int M, int n_list, int iters, float* codebooks, float* coarse, void* ws,
                 size_t ws_bytes, cudaStream_t s) {
    int rc = check_shape(M, n_list);
    if (rc) return rc;
    AB_REQUIRE(sample != nullptr && codebooks != nullptr && (n_list == 0 || coarse != nullptr), "null pointer argument");
    AB_REQUIRE(S >= KSUB && S >= n_list && S < (1ll << 31), "training needs at least max(256, n_list) rows (got %lld)",
               (long long)S);
    AB_REQUIRE(iters >= 0, "iters=%d must be >= 0", iters);
    ChunkWs w;
    float* resid;
    uint8_t* codes_t;
    int32_t* counts;
    int32_t* assign;
    const size_t need = train_bytes(S, M, n_list, &w, &resid, &codes_t, &counts, &assign, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    const int64_t R = chunk_rows(M, n_list);
    const int dsub = DIM / M;

    // ---- coarse quantizer: inner-product k-means on the first min(S, 256 n_list) rows
    if (n_list > 0 && (rc = coarse_kmeans(sample, S, n_list, iters, coarse, w, R, assign, counts, s))) return rc;

    // ---- product quantizer: L2 k-means per sub-space on the residuals of the first min(S, 65536) rows
    const int64_t sp = S < PQ_TRAIN_MAX ? S : PQ_TRAIN_MAX;
    if (n_list > 0 && (rc = coarse_assign(sample, sp, w.coarse16, n_list, w, R, assign, nullptr, 0, s))) return rc;
    if ((rc = residual(sample, sp, n_list > 0 ? coarse : nullptr, assign, resid, s))) return rc;
    // initial centroids: rows 0..255 of the (randomly ordered) sample
    pq_copy_rows_kernel<<<dim3(grid_1d(static_cast<int64_t>(KSUB) * dsub, 256), M), 256, 0, s>>>(
        resid, DIM, codebooks, dsub, KSUB, dsub, dsub, static_cast<int64_t>(KSUB) * dsub);
    abh::count_launch();
    for (int it = 0; it < iters; ++it) {
        if ((rc = codebook_norms(codebooks, M, w.norms, s))) return rc;
        if ((rc = pq_assign(resid, sp, M, codebooks, w, R, codes_t, s))) return rc;
        pq_update_kernel<float, uint8_t><<<dim3(KSUB, M), 256, 0, s>>>(resid, DIM, codes_t, M, static_cast<int>(sp), KSUB,
                                                                      dsub, codebooks, counts);
        pq_split_kernel<<<M, 256, 0, s>>>(codebooks, counts, KSUB, dsub);
        abh::count_launch(2);
        AB_CUDA_CHECK(cudaGetLastError());
    }
    return ATLAS_B200_OK;
}

static int encode(const __half* rows, int64_t n, int M, const float* codebooks, const float* coarse, int n_list,
                  uint8_t* codes, void* lists, void* ws, size_t ws_bytes, cudaStream_t s) {
    int rc = check_shape(M, n_list);
    if (rc) return rc;
    AB_REQUIRE(n >= 0, "n=%lld must be >= 0", (long long)n);
    if (n == 0) return ATLAS_B200_OK;
    AB_REQUIRE(rows != nullptr && codebooks != nullptr && codes != nullptr &&
               (n_list == 0 || (coarse != nullptr && lists != nullptr)), "null pointer argument");
    ChunkWs w;
    const size_t need = encode_bytes(M, n_list, &w, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    const int64_t R = chunk_rows(M, n_list);
    const int list_u16 = n_list <= 65535 ? 1 : 0;
    if ((rc = codebook_norms(codebooks, M, w.norms, s))) return rc;
    if (n_list > 0 && (rc = coarse_to_half(coarse, n_list, w.coarse16, s))) return rc;
    for (int64_t r0 = 0; r0 < n; r0 += R) {
        const int64_t cn = n - r0 < R ? n - r0 : R;
        const __half* x = rows + r0 * DIM;
        if (n_list > 0) {
            void* l = static_cast<uint8_t*>(lists) + r0 * (list_u16 ? 2 : 4);
            if ((rc = coarse_assign(x, cn, w.coarse16, n_list, w, R, w.assign, l, list_u16, s))) return rc;
        }
        if ((rc = residual(x, cn, n_list > 0 ? coarse : nullptr, w.assign, w.resid, s))) return rc;
        if ((rc = pq_assign(w.resid, cn, M, codebooks, w, R, codes + r0 * M, s))) return rc;
    }
    return ATLAS_B200_OK;
}

// queries per scan CTA: the largest power of two <= 16 (and not above the block's query count) whose tables fit
static int choose_qpc(int M, int n_list, int nq, bool* cterm_smem) {
    int cap = 1;
    while (cap < nq && cap < 16) cap <<= 1;
    for (int with_ct = (n_list > 0); with_ct >= 0; --with_ct) {
        for (int qpc = cap; qpc >= 1; qpc >>= 1) {
            const size_t bytes = static_cast<size_t>(qpc) * (static_cast<size_t>(M) * KSUB * 4 + (with_ct ? n_list * 4ull : 0));
            if (bytes <= SCAN_SMEM_MAX) {
                *cterm_smem = with_ct != 0;
                return qpc;
            }
        }
    }
    *cterm_smem = false;
    return 1;
}

template <int QPC, bool PROBED>
static int launch_scan_q(const ScanParams& p, const ProbeScan& pr, size_t smem, cudaStream_t s) {
    static bool attr_set = false;
    if (!attr_set) {
        AB_CUDA_CHECK(cudaFuncSetAttribute(pq_scan_kernel<QPC, PROBED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SCAN_SMEM_MAX));
        attr_set = true;
    }
    const int groups = (p.nq + QPC - 1) / QPC;
    const int per_sm = static_cast<int>((228 * 1024) / (smem + 2048)) > 0 ? static_cast<int>((228 * 1024) / (smem + 2048)) : 1;
    const int resident = abh::num_sms() * (per_sm < 4 ? per_sm : 4);
    int gx = (resident + groups - 1) / groups;
    if (gx > p.num_tiles) gx = p.num_tiles;
    if (gx < 1) gx = 1;
    pq_scan_kernel<QPC, PROBED><<<dim3(gx, groups), SCAN_THREADS, smem, s>>>(p, pr);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

template <bool PROBED>
static int launch_scan(int qpc, const ScanParams& p, const ProbeScan& pr, size_t smem, cudaStream_t s) {
    if (p.num_tiles <= 0) return ATLAS_B200_OK;
    switch (qpc) {
        case 16: return launch_scan_q<16, PROBED>(p, pr, smem, s);
        case 8: return launch_scan_q<8, PROBED>(p, pr, smem, s);
        case 4: return launch_scan_q<4, PROBED>(p, pr, smem, s);
        case 2: return launch_scan_q<2, PROBED>(p, pr, smem, s);
        default: return launch_scan_q<1, PROBED>(p, pr, smem, s);
    }
}

// The exact top-k pipeline of one block of nqb queries over the scores of a code sweep (mips.cu's one-stage sample):
//   bound from a strided sample of ~2 sqrt(k n) rows (every score kept) -> full sweep with the bound -> select + emit,
//   `status` on overflow; or the chunked exhaustive variant (every score of a chunk is a candidate, winners carried).
// scan(tile_begin, tile_step, num_tiles, sample) launches the scan kernel over tiles of `tile_rows` rows (n rows or slots in
// all; sample marks the bound's sampling launch); it appends only real rows, so the sampled bound is the k-th best among
// real rows.  A probed scan takes these tile counts as upper bounds of its compacted items and resolves them against the
// item count in device memory (ivf_probe.cuh); its sampling launch scans the sample items instead, which reach every
// query's own probe set.  The sweep is profiled as kind 1.
template <class Scan>
static int sweep_select(const Scan& scan, int64_t n, int total_tiles, int tile_rows, int nqb, int k, uint64_t* cand,
                        uint32_t* count, float* bound, uint32_t capq, uint16_t* os16, int64_t* oi_b, int64_t id_base,
                        int64_t id_stride, int32_t* status, bool exhaustive, double sweep_work, cudaStream_t s) {
    int rc;
    if (!exhaustive) {
        if (n > static_cast<int64_t>(capq)) {
            double m = 2.0 * sqrt(static_cast<double>(k) * static_cast<double>(n));
            if (m < 4096) m = 4096;
            if (m > capq / 2) m = capq / 2;
            int sample_tiles = static_cast<int>(m / tile_rows);
            if (sample_tiles < 1) sample_tiles = 1;
            if (sample_tiles > total_tiles) sample_tiles = total_tiles;
            if ((rc = scan(0, total_tiles / sample_tiles, sample_tiles, true))) return rc;
            mips::mips_select_kernel<false><<<nqb, mips::SEL_THREADS, 0, s>>>(
                cand, count, capq, k, mips::SEL_WRITE_BOUND, bound, nullptr, nullptr, 0, 0, nullptr);
            abh::count_launch();
        }
        abh::prof_begin(s, abh::PROF_SCAN);
        rc = scan(0, 1, total_tiles, false);
        abh::prof_end(s, abh::PROF_SCAN, sweep_work);
        if (rc) return rc;
        mips::mips_select_kernel<false><<<nqb, mips::SEL_THREADS, 0, s>>>(
            cand, count, capq, k, mips::SEL_EMIT, bound, os16, oi_b, id_base, id_stride, status);
        abh::count_launch();
    } else {
        int chunk_tiles = static_cast<int>((capq - static_cast<uint32_t>(k)) / tile_rows);
        if (chunk_tiles < 1) chunk_tiles = 1;
        for (int t0 = 0; t0 < total_tiles; t0 += chunk_tiles) {
            const bool last = t0 + chunk_tiles >= total_tiles;
            if ((rc = scan(t0, 1, last ? total_tiles - t0 : chunk_tiles, false))) return rc;
            mips::mips_select_kernel<false><<<nqb, mips::SEL_THREADS, 0, s>>>(
                cand, count, capq, k, last ? mips::SEL_EMIT : mips::SEL_CARRY, bound, os16, oi_b, id_base, id_stride,
                nullptr);
            abh::count_launch();
        }
    }
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

static int topk(const uint8_t* codes, const void* lists, int64_t n, int M, const float* codebooks, const float* coarse,
                int n_list, const __half* queries, int nq, int k, __half* out_scores, int64_t* out_ids, int64_t id_base,
                int64_t id_stride, int32_t* status, void* ws, size_t ws_bytes, cudaStream_t s, bool exhaustive,
                const ProbeArgs* probe = nullptr) {
    int rc = check_shape(M, n_list);
    if (rc) return rc;
    if (probe) {
        AB_REQUIRE(n_list >= 1, "a probed search needs inverted lists (n_list=%d)", n_list);
        AB_REQUIRE(probe->nprobe >= 1, "nprobe=%d must be >= 1", probe->nprobe);
        AB_REQUIRE(probe->list_order != nullptr && probe->list_offsets != nullptr, "null list table");
        if (probe->nprobe >= n_list) probe = nullptr;     // every list: the full scan
    }
    AB_REQUIRE(nq >= 0 && k >= 1, "nq must be >= 0 and k >= 1 (nq=%d k=%d)", nq, k);
    AB_REQUIRE(k <= ATLAS_B200_MAX_TOPK, "k=%d exceeds ATLAS_B200_MAX_TOPK=%d", k, ATLAS_B200_MAX_TOPK);
    AB_REQUIRE(n >= 1 && n < (1ll << 31) - SCAN_THREADS, "rows n=%lld out of range", (long long)n);
    AB_REQUIRE(k <= n, "selected index k out of range: k=%d > n=%lld", k, (long long)n);
    AB_REQUIRE(codes != nullptr && codebooks != nullptr && (n_list == 0 || (coarse != nullptr && lists != nullptr)),
               "null pointer argument");
    AB_REQUIRE((M & 3) != 0 || (reinterpret_cast<uintptr_t>(codes) & 3u) == 0, "codes must be 4-byte aligned");
    AB_REQUIRE(nq == 0 || queries != nullptr, "queries is null");
    if (status) AB_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int32_t), s));
    if (nq == 0) return ATLAS_B200_OK;
    SearchWs w;
    ProbeWs pw{};
    const int64_t max_items = pq_max_items(n, n_list);
    size_t need = search_bytes(n, M, n_list, k, &w, ws);
    if (probe) need = probe_bytes(need, n_list, max_items, k, PROBE_CHUNK, &pw, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    const int dsub = DIM / M;
    const int total_tiles = static_cast<int>((n + SCAN_THREADS - 1) / SCAN_THREADS);
    for (int q0 = 0; q0 < nq; q0 += QBLOCK) {
        const int nqb = nq - q0 < QBLOCK ? nq - q0 : QBLOCK;
        if ((rc = residual(queries + static_cast<int64_t>(q0) * DIM, nqb, nullptr, nullptr, w.qf32, s))) return rc;
        if ((rc = subdot(w.qf32, DIM, nqb, codebooks, KSUB, dsub, M, w.lut, s))) return rc;
        if (n_list > 0 && (rc = subdot(w.qf32, DIM, nqb, coarse, n_list, DIM, 1, w.cterm, s))) return rc;
        pq_prep_kernel<<<1, QBLOCK, 0, s>>>(w.count, w.bound);
        abh::count_launch();
        bool cterm_smem = false;
        const int qpc = choose_qpc(M, n_list, nqb, &cterm_smem);
        const size_t smem = static_cast<size_t>(qpc) * (static_cast<size_t>(M) * KSUB * 4 + (cterm_smem ? n_list * 4ull : 0));
        ScanParams p;
        p.codes = codes;
        p.lists = lists;
        p.list_u16 = n_list <= 65535 ? 1 : 0;
        p.n_rows = static_cast<int>(n);
        p.M = M;
        p.lut = w.lut;
        p.cterm = n_list > 0 ? w.cterm : nullptr;
        p.n_list = n_list;
        p.cterm_smem = cterm_smem ? 1 : 0;
        p.nq = nqb;
        p.bound = w.bound;
        p.count = w.count;
        p.cand = w.cand;
        p.capq = w.capq;
        int64_t* oi_b = out_ids + static_cast<size_t>(q0) * k;
        uint16_t* os16 = reinterpret_cast<uint16_t*>(out_scores + static_cast<size_t>(q0) * k);
        if (probe) {
            // P(q) and its sample lists from the coarse terms the scan adds, then the chunks of every list some query
            // probes and the sample chunks
            if ((rc = ivfp::select_probes(w.cterm, n_list, 1, nqb, n_list, probe->list_offsets, nullptr, probe->nprobe, k,
                                          w.capq, pw.sample_units * PROBE_CHUNK, pw.probed, pw.sample_lists, s)))
                return rc;
            if ((rc = ivfp::compact_items(pw.probed, pw.sample_lists, probe->list_offsets, n_list, PROBE_CHUNK,
                                          pw.sample_units, pw.items, pw.sample, pw.count, s)))
                return rc;
        }
        ProbeScan pr{pw.items, pw.count, probe ? probe->list_order : nullptr, probe ? probe->list_offsets : nullptr,
                     pw.probed};
        auto scan = [&](int tile_begin, int tile_step, int num_tiles, bool sample) {
            p.tile_begin = tile_begin;
            p.tile_step = tile_step;
            p.num_tiles = num_tiles;
            if (!probe) return launch_scan<false>(qpc, p, pr, smem, s);
            ProbeScan ps = pr;
            if (sample) {     // the bound's scan: every sample chunk (ivf_probe.cuh), not a stride over the sweep
                ps.items = pw.sample;
                ps.item_count = pw.count + 1;
                p.tile_begin = 0;
                p.tile_step = 1;
                p.num_tiles = static_cast<int>(pw.max_sample);
            }
            return launch_scan<true>(qpc, p, ps, smem, s);
        };
        if ((rc = sweep_select(scan, n, probe ? static_cast<int>(max_items) : total_tiles, SCAN_THREADS, nqb, k, w.cand, w.count, w.bound, w.capq, os16, oi_b, id_base,
                               id_stride, status, exhaustive, static_cast<double>(n) * M * ((nqb + qpc - 1) / qpc), s)))
            return rc;
    }
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// IVF-SQ (faiss IndexIVFScalarQuantizer, QT_4bit, residuals, inner product; layout: ivfsq.cuh, scan: ivfsq.cu)
//   range    per dim: vmin = min r_d, vdiff = max r_d - vmin over the residuals r = fp32(x) - coarse[list(x)] of the
//            first min(S, 100000) sample rows (faiss RS_minmax, non-uniform)
//   encode   xi = (r_d - vmin_d) / vdiff_d (0 when vdiff_d == 0), clamped to [0, 1]; code = (int)(xi * 15.0) in double
//   search   w^[q][d] = fp16(2^e_q * q_d * (vdiff_d / 15)), e_q putting max_d |w^| in [2^14, 2^15);
//            C[q] = sum_d q_d (vmin_d + 0.5 vdiff_d / 15) + 2^-e_q * 8 sum_d w^[q][d], T[l][q] = <q, c_l> (fp32);
//            s = fp16(T[list][q] + C[q] + 2^-e_q * sum_d w^[q][d] (code_d - 8))
// ---------------------------------------------------------------------------------------------
constexpr int64_t SQ_RANGE_MAX = 100000;   // faiss ScalarQuantizer::train_residual's subsample
constexpr int SQ_RANGE_ROWS = 512;         // rows per partial min / max block

// partial per-dim min / max of the residuals of rows [c * SQ_RANGE_ROWS, ...) of the first ns rows, c = blockIdx.x
__global__ void __launch_bounds__(256) sq_range_partial_kernel(const __half* __restrict__ x, int64_t ns,
                                                               const float* __restrict__ coarse,
                                                               const int32_t* __restrict__ assign, float* __restrict__ pmin,
                                                               float* __restrict__ pmax) {
    const int64_t r0 = static_cast<int64_t>(blockIdx.x) * SQ_RANGE_ROWS;
    const int64_t r1 = r0 + SQ_RANGE_ROWS < ns ? r0 + SQ_RANGE_ROWS : ns;
    for (int d = threadIdx.x; d < DIM; d += 256) {
        float lo = INFINITY, hi = -INFINITY;
        for (int64_t i = r0; i < r1; ++i) {
            const float r = __fsub_rn(__half2float(x[i * DIM + d]), coarse[static_cast<int64_t>(assign[i]) * DIM + d]);
            lo = fminf(lo, r);
            hi = fmaxf(hi, r);
        }
        pmin[static_cast<int64_t>(blockIdx.x) * DIM + d] = lo;
        pmax[static_cast<int64_t>(blockIdx.x) * DIM + d] = hi;
    }
}

__global__ void sq_range_final_kernel(const float* __restrict__ pmin, const float* __restrict__ pmax, int parts,
                                      float* __restrict__ vmin, float* __restrict__ vdiff) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= DIM) return;
    float lo = INFINITY, hi = -INFINITY;
    for (int c = 0; c < parts; ++c) {
        lo = fminf(lo, pmin[static_cast<int64_t>(c) * DIM + d]);
        hi = fmaxf(hi, pmax[static_cast<int64_t>(c) * DIM + d]);
    }
    vmin[d] = lo;
    vdiff[d] = __fsub_rn(hi, lo);
}

// 4-bit codes of rows [n] (list assign[i]) into slot row_slot[i] of `codes`, in the slot's nibble order; one thread per
// 32-bit output word
__global__ void sq_encode_kernel(const __half* __restrict__ x, int64_t n, const float* __restrict__ coarse,
                                 const int32_t* __restrict__ assign, const float* __restrict__ vmin,
                                 const float* __restrict__ vdiff, const int32_t* __restrict__ row_slot,
                                 uint8_t* __restrict__ codes) {
    constexpr int WORDS = ivfsq::SQ_CODE_BYTES / 4;
    const int64_t total = n * WORDS;
    for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < total;
         e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t i = e / WORDS;
        const int wd = static_cast<int>(e - i * WORDS);
        const float* c = coarse + static_cast<int64_t>(assign[i]) * DIM;
        uint32_t word = 0;
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const int d = ivfsq::sq_dim_of_nibble(8 * wd + b);
            const float r = __fsub_rn(__half2float(x[i * DIM + d]), c[d]);
            float xi = 0.f;
            if (vdiff[d] != 0.f) {
                xi = __fdiv_rn(__fsub_rn(r, vmin[d]), vdiff[d]);
                xi = xi < 0.f ? 0.f : (xi > 1.f ? 1.f : xi);
            }
            const uint32_t code = static_cast<uint32_t>(static_cast<int>(static_cast<double>(xi) * 15.0));
            word |= code << (4 * b);
        }
        reinterpret_cast<uint32_t*>(codes + static_cast<int64_t>(row_slot[i]) * ivfsq::SQ_CODE_BYTES)[wd] = word;
    }
}

// Per query row q of a block (one CTA each, rows past nq are zero): the fp16 operand w^, the fp32 row, C[q], 2^-e_q;
// resets the block's candidate counters and bounds.
__global__ void __launch_bounds__(256) sq_query_kernel(const __half* __restrict__ q16, int nq, const float* __restrict__ vmin,
                                                       const float* __restrict__ vdiff, __half* __restrict__ what,
                                                       float* __restrict__ qf32, float* __restrict__ cterm,
                                                       float* __restrict__ scale, uint32_t* __restrict__ count,
                                                       float* __restrict__ bound) {
    __shared__ float s_max[256], s_sum[256], s_wsum[256];
    const int q = blockIdx.x, t = threadIdx.x;
    float pv[DIM / 256];
    float mx = 0.f, cs = 0.f;
#pragma unroll
    for (int r = 0; r < DIM / 256; ++r) {
        const int d = t + 256 * r;
        const float qf = q < nq ? __half2float(q16[static_cast<int64_t>(q) * DIM + d]) : 0.f;
        qf32[static_cast<int64_t>(q) * DIM + d] = qf;
        pv[r] = __fmul_rn(qf, __fdiv_rn(vdiff[d], 15.f));
        mx = fmaxf(mx, fabsf(pv[r]));
        cs = __fadd_rn(cs, __fmul_rn(qf, __fadd_rn(vmin[d], __fdiv_rn(__fmul_rn(0.5f, vdiff[d]), 15.f))));
    }
    s_max[t] = mx;
    s_sum[t] = cs;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (t < o) {
            s_max[t] = fmaxf(s_max[t], s_max[t + o]);
            s_sum[t] = __fadd_rn(s_sum[t], s_sum[t + o]);
        }
        __syncthreads();
    }
    int e = 0;
    if (s_max[0] > 0.f && s_max[0] < INFINITY) {
        int x;
        frexpf(s_max[0], &x);     // max in [2^(x-1), 2^x)  ->  max * 2^(15 - x) in [2^14, 2^15)
        e = 15 - x;
    }
    float ws = 0.f;
#pragma unroll
    for (int r = 0; r < DIM / 256; ++r) {
        const __half w = __float2half_rn(ldexpf(pv[r], e));
        what[static_cast<int64_t>(q) * DIM + t + 256 * r] = w;
        ws = __fadd_rn(ws, __half2float(w));
    }
    s_wsum[t] = ws;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (t < o) s_wsum[t] = __fadd_rn(s_wsum[t], s_wsum[t + o]);
        __syncthreads();
    }
    if (t == 0) {
        // the MMA sums w^ (code - 8): C carries the offset 8 sum_d w^
        cterm[q] = __fadd_rn(s_sum[0], ldexpf(8.f * s_wsum[0], -e));
        scale[q] = ldexpf(1.f, -e);
        count[q] = 0;
        bound[q] = -INFINITY;
    }
}

static int64_t sq_chunk_rows(int n_list) {
    int64_t r = static_cast<int64_t>(CHUNK_BUDGET / (static_cast<size_t>(pad8(n_list)) * 2 + 4));
    if (r > 65536) r = 65536;
    r = r / 64 * 64;
    return r < 64 ? 64 : r;
}

static size_t sq_train_bytes(int64_t S, int n_list, ChunkWs* w, int32_t** assign, int32_t** counts, float** pmin,
                             float** pmax, void* base) {
    Carver cv{static_cast<uint8_t*>(base)};
    const int64_t R = sq_chunk_rows(n_list);
    const int64_t ns = S < SQ_RANGE_MAX ? S : SQ_RANGE_MAX;
    const int parts = static_cast<int>((ns + SQ_RANGE_ROWS - 1) / SQ_RANGE_ROWS);
    ChunkWs tmp{};
    ChunkWs& c = w ? *w : tmp;
    c.gemm = cv.take<__half>(static_cast<size_t>(R) * pad8(n_list));
    c.coarse16 = cv.take<__half>(static_cast<size_t>(pad8(n_list)) * DIM);
    int32_t* a = cv.take<int32_t>(static_cast<size_t>(S));
    int32_t* n = cv.take<int32_t>(static_cast<size_t>(n_list));
    float* lo = cv.take<float>(static_cast<size_t>(parts) * DIM);
    float* hi = cv.take<float>(static_cast<size_t>(parts) * DIM);
    if (assign) *assign = a;
    if (counts) *counts = n;
    if (pmin) *pmin = lo;
    if (pmax) *pmax = hi;
    return cv.off;
}

static size_t sq_encode_bytes(int n_list, ChunkWs* w, void* base) {
    Carver cv{static_cast<uint8_t*>(base)};
    const int64_t R = sq_chunk_rows(n_list);
    ChunkWs tmp{};
    ChunkWs& c = w ? *w : tmp;
    c.gemm = cv.take<__half>(static_cast<size_t>(R) * pad8(n_list));
    c.coarse16 = cv.take<__half>(static_cast<size_t>(pad8(n_list)) * DIM);
    c.assign = cv.take<int32_t>(static_cast<size_t>(R));
    return cv.off;
}

struct SqSearchWs {
    uint32_t* count;
    float* bound;
    uint64_t* cand;
    uint32_t capq;
    __half* what;   // [QBLOCK][768]
    float* qf32;    // [QBLOCK][768]
    float* tterm;   // [n_list][nqb]
    float* cterm;   // [QBLOCK]
    float* scale;   // [QBLOCK]
};

static size_t sq_search_bytes(int64_t n_slots, int n_list, int k, SqSearchWs* w, void* base) {
    Carver cv{static_cast<uint8_t*>(base)};
    const uint32_t capq = mips::capq_for(n_slots, k);
    SqSearchWs x;
    x.count = cv.take<uint32_t>(QBLOCK);
    x.bound = cv.take<float>(QBLOCK);
    x.cand = cv.take<uint64_t>(static_cast<size_t>(QBLOCK) * capq);
    x.capq = capq;
    x.what = cv.take<__half>(static_cast<size_t>(QBLOCK) * DIM);
    x.qf32 = cv.take<float>(static_cast<size_t>(QBLOCK) * DIM);
    x.tterm = cv.take<float>(static_cast<size_t>(n_list) * QBLOCK);
    x.cterm = cv.take<float>(QBLOCK);
    x.scale = cv.take<float>(QBLOCK);
    if (w) *w = x;
    return cv.off;
}

static int sq_train(const __half* sample, int64_t S, int n_list, int iters, float* coarse, float* vmin, float* vdiff, void* ws,
                    size_t ws_bytes, cudaStream_t s) {
    AB_REQUIRE(sample != nullptr && coarse != nullptr && (vmin == nullptr) == (vdiff == nullptr), "null pointer argument");
    AB_REQUIRE(n_list >= 1, "n_list=%d must be >= 1", n_list);
    AB_REQUIRE(S >= n_list && S < (1ll << 31), "training needs at least n_list=%d rows (got %lld)", n_list, (long long)S);
    AB_REQUIRE(iters >= 0, "iters=%d must be >= 0", iters);
    ChunkWs w{};
    int32_t *assign, *counts;
    float *pmin, *pmax;
    const size_t need = sq_train_bytes(S, n_list, &w, &assign, &counts, &pmin, &pmax, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    const int64_t R = sq_chunk_rows(n_list);
    int rc = coarse_kmeans(sample, S, n_list, iters, coarse, w, R, assign, counts, s);
    if (rc) return rc;
    if (vmin == nullptr) return ATLAS_B200_OK;      // the coarse quantizer alone (ivfflat)
    const int64_t ns = S < SQ_RANGE_MAX ? S : SQ_RANGE_MAX;
    if ((rc = coarse_assign(sample, ns, w.coarse16, n_list, w, R, assign, nullptr, 0, s))) return rc;
    const int parts = static_cast<int>((ns + SQ_RANGE_ROWS - 1) / SQ_RANGE_ROWS);
    sq_range_partial_kernel<<<parts, 256, 0, s>>>(sample, ns, coarse, assign, pmin, pmax);
    sq_range_final_kernel<<<(DIM + 255) / 256, 256, 0, s>>>(pmin, pmax, parts, vmin, vdiff);
    abh::count_launch(2);
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

static int sq_encode(const __half* rows, int64_t n, const float* coarse, int n_list, const float* vmin, const float* vdiff,
                     int32_t* lists, const int32_t* row_slot, uint8_t* codes, void* ws, size_t ws_bytes, cudaStream_t s) {
    AB_REQUIRE(n >= 0, "n=%lld must be >= 0", (long long)n);
    AB_REQUIRE(n_list >= 1, "n_list=%d must be >= 1", n_list);
    if (n == 0) return ATLAS_B200_OK;
    AB_REQUIRE(rows != nullptr && coarse != nullptr, "null pointer argument");
    AB_REQUIRE(lists != nullptr || codes != nullptr, "nothing to write: list_ids and codes are both NULL");
    AB_REQUIRE(codes == nullptr || (row_slot != nullptr && vmin != nullptr && vdiff != nullptr &&
                                    abh::aligned(codes, 4)),
               "codes need row_slot, vmin and vdiff, and must be 4-byte aligned");
    ChunkWs w{};
    const size_t need = sq_encode_bytes(n_list, &w, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    const int64_t R = sq_chunk_rows(n_list);
    int rc = coarse_to_half(coarse, n_list, w.coarse16, s);
    if (rc) return rc;
    for (int64_t r0 = 0; r0 < n; r0 += R) {
        const int64_t cn = n - r0 < R ? n - r0 : R;
        const __half* x = rows + r0 * DIM;
        if ((rc = coarse_assign(x, cn, w.coarse16, n_list, w, R, w.assign, lists ? lists + r0 : nullptr, 0, s))) return rc;
        if (codes) {
            sq_encode_kernel<<<grid_1d(cn * (ivfsq::SQ_CODE_BYTES / 4), 256), 256, 0, s>>>(x, cn, coarse, w.assign, vmin, vdiff,
                                                                                        row_slot + r0, codes);
            abh::count_launch();
            AB_CUDA_CHECK(cudaGetLastError());
        }
    }
    return ATLAS_B200_OK;
}

static int sq_topk(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists, int64_t n_tiles, int64_t n_rows,
                   const float* coarse, int n_list, const float* vmin, const float* vdiff, const __half* queries, int nq, int k,
                   __half* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride, int32_t* status, void* ws,
                   size_t ws_bytes, cudaStream_t s, bool exhaustive, const ProbeArgs* probe = nullptr) {
    AB_REQUIRE(nq >= 0 && k >= 1, "nq must be >= 0 and k >= 1 (nq=%d k=%d)", nq, k);
    if (probe) {
        AB_REQUIRE(probe->nprobe >= 1, "nprobe=%d must be >= 1", probe->nprobe);
        AB_REQUIRE(probe->list_offsets != nullptr && probe->list_rows != nullptr, "null list table");
        if (probe->nprobe >= n_list) probe = nullptr;     // every list: the full scan
    }
    AB_REQUIRE(k <= ATLAS_B200_MAX_TOPK, "k=%d exceeds ATLAS_B200_MAX_TOPK=%d", k, ATLAS_B200_MAX_TOPK);
    AB_REQUIRE(n_list >= 1, "n_list=%d must be >= 1", n_list);
    AB_REQUIRE(n_rows >= 1 && n_tiles >= 1 && n_rows <= n_tiles * ivfsq::SQ_TILE &&
                   n_tiles * ivfsq::SQ_TILE < (1ll << 31) - ivfsq::SQ_TILE,
               "rows n=%lld / tiles %lld out of range", (long long)n_rows, (long long)n_tiles);
    AB_REQUIRE(k <= n_rows, "selected index k out of range: k=%d > n=%lld", k, (long long)n_rows);
    AB_REQUIRE(codes != nullptr && slot_rows != nullptr && tile_lists != nullptr && coarse != nullptr && vmin != nullptr &&
                   vdiff != nullptr, "null pointer argument");
    AB_REQUIRE(abh::aligned(codes, 16), "codes must be 16-byte aligned");
    AB_REQUIRE(nq == 0 || queries != nullptr, "queries is null");
    if (status) AB_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int32_t), s));
    if (nq == 0) return ATLAS_B200_OK;
    SqSearchWs w;
    ProbeWs pw{};
    const int64_t n_slots = n_tiles * ivfsq::SQ_TILE;
    size_t need = sq_search_bytes(n_slots, n_list, k, &w, ws);
    if (probe) need = probe_bytes(need, n_list, n_tiles, k, ivfsq::SQ_TILE, &pw, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    int rc;
    for (int q0 = 0; q0 < nq; q0 += QBLOCK) {
        const int nqb = nq - q0 < QBLOCK ? nq - q0 : QBLOCK;
        sq_query_kernel<<<QBLOCK, 256, 0, s>>>(queries + static_cast<int64_t>(q0) * DIM, nqb, vmin, vdiff, w.what, w.qf32,
                                               w.cterm, w.scale, w.count, w.bound);
        abh::count_launch();
        // T[l][q] = <c_l, q>: the coarse centroids against the block's queries
        if ((rc = subdot(coarse, DIM, n_list, w.qf32, nqb, DIM, 1, w.tterm, s))) return rc;
        ivfsq::ScanParams p;
        p.codes = codes;
        p.slot_rows = slot_rows;
        p.tile_lists = tile_lists;
        p.n_tiles = static_cast<int>(n_tiles);
        p.what = w.what;
        p.tterm = w.tterm;
        p.ldt = nqb;
        p.cterm = w.cterm;
        p.scale = w.scale;
        p.nq = nqb;
        p.bound = w.bound;
        p.count = w.count;
        p.cand = w.cand;
        p.capq = w.capq;
        int64_t* oi_b = out_ids + static_cast<size_t>(q0) * k;
        uint16_t* os16 = reinterpret_cast<uint16_t*>(out_scores + static_cast<size_t>(q0) * k);
        if (probe) {
            // P(q) and its sample lists from T[l][q] (strided by list), then the tiles of every list some query probes
            // and the sample tiles
            if ((rc = ivfp::select_probes(w.tterm, 1, nqb, nqb, n_list, nullptr, probe->list_rows, probe->nprobe, k, w.capq,
                                          pw.sample_units * ivfsq::SQ_TILE, pw.probed, pw.sample_lists, s)))
                return rc;
            if ((rc = ivfp::compact_items(pw.probed, pw.sample_lists, probe->list_offsets, n_list, 1, pw.sample_units,
                                          pw.items, pw.sample, pw.count, s)))
                return rc;
        }
        const ivfsq::ProbeScan pr{pw.items, pw.count, pw.probed};
        const ivfsq::ProbeScan ps{pw.sample, pw.count + 1, pw.probed};
        auto scan = [&](int tile_begin, int tile_step, int num_tiles, bool sample) {
            p.tile_begin = tile_begin;
            p.tile_step = tile_step;
            p.num_tiles = num_tiles;
            if (!probe) return ivfsq::launch_scan(p, nullptr, s);
            if (sample) {     // the bound's scan: every sample tile (ivf_probe.cuh), not a stride over the sweep
                p.tile_begin = 0;
                p.tile_step = 1;
                p.num_tiles = static_cast<int>(pw.max_sample);
                return ivfsq::launch_scan(p, &ps, s);
            }
            return ivfsq::launch_scan(p, &pr, s);
        };
        // work = code bytes swept (once per 128 queries of the block)
        const double sweep_bytes = static_cast<double>(n_slots) * ivfsq::SQ_CODE_BYTES * ((nqb + 127) / 128);
        if ((rc = sweep_select(scan, n_slots, static_cast<int>(n_tiles), ivfsq::SQ_TILE, nqb, k, w.cand, w.count, w.bound,
                               w.capq, os16, oi_b, id_base, id_stride, status, exhaustive, sweep_bytes, s)))
            return rc;
    }
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// IVF-Flat search (types ivfflat and flat): the scan kernel is in ivfflat.cu
// ---------------------------------------------------------------------------------------------
// Per query row q of a block (one CTA each, rows past nq are zero): the fp16 row for the scan's TMA, its fp32 copy for
// the coarse terms; resets the block's candidate counters and bounds.
__global__ void __launch_bounds__(256) flat_query_kernel(const __half* __restrict__ q16, int nq, __half* __restrict__ qstage,
                                                         float* __restrict__ qf32, uint32_t* __restrict__ count,
                                                         float* __restrict__ bound) {
    const int q = blockIdx.x;
    for (int d = threadIdx.x; d < DIM; d += blockDim.x) {
        const __half h = q < nq ? q16[static_cast<int64_t>(q) * DIM + d] : __float2half_rn(0.f);
        qstage[static_cast<int64_t>(q) * DIM + d] = h;
        qf32[static_cast<int64_t>(q) * DIM + d] = __half2float(h);
    }
    if (threadIdx.x == 0) {
        count[q] = 0;
        bound[q] = -INFINITY;
    }
}

struct FlatSearchWs {
    uint32_t* count;
    float* bound;
    uint64_t* cand;
    uint32_t capq;
    __half* qstage;  // [QBLOCK][768]
    float* qf32;     // [QBLOCK][768]
    float* tterm;    // [n_list][nqb] (probed search only)
};

static size_t flat_search_bytes(int64_t n_slots, int n_list, int k, bool probed, FlatSearchWs* w, void* base) {
    Carver cv{static_cast<uint8_t*>(base)};
    const uint32_t capq = mips::capq_for(n_slots, k);
    FlatSearchWs x;
    x.count = cv.take<uint32_t>(QBLOCK);
    x.bound = cv.take<float>(QBLOCK);
    x.cand = cv.take<uint64_t>(static_cast<size_t>(QBLOCK) * capq);
    x.capq = capq;
    x.qstage = cv.take<__half>(static_cast<size_t>(QBLOCK) * DIM);
    x.qf32 = cv.take<float>(static_cast<size_t>(QBLOCK) * DIM);
    x.tterm = cv.take<float>(probed ? static_cast<size_t>(n_list) * QBLOCK : 0);
    if (w) *w = x;
    return cv.off;
}

// nprobe = 0 or >= n_list: every tile (list tables and coarse unused, may be NULL); else the probed search.
static int flat_topk(const __half* rows, const int32_t* slot_rows, int64_t n_tiles, int64_t n_rows, const int32_t* list_tile_off,
                     const int32_t* list_rows, const float* coarse, int n_list, int nprobe, const __half* queries, int nq, int k,
                     __half* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride, int32_t* status, void* ws,
                     size_t ws_bytes, cudaStream_t s, bool exhaustive) {
    AB_REQUIRE(nq >= 0 && k >= 1, "nq must be >= 0 and k >= 1 (nq=%d k=%d)", nq, k);
    AB_REQUIRE(k <= ATLAS_B200_MAX_TOPK, "k=%d exceeds ATLAS_B200_MAX_TOPK=%d", k, ATLAS_B200_MAX_TOPK);
    AB_REQUIRE(n_list >= 1, "n_list=%d must be >= 1", n_list);
    AB_REQUIRE(nprobe >= 0, "nprobe=%d must be >= 1 (or 0 for every list)", nprobe);
    AB_REQUIRE(n_rows >= 1 && n_tiles >= 1 && n_rows <= n_tiles * ivfflat::FLAT_TILE &&
                   n_tiles * ivfflat::FLAT_TILE < (1ll << 31) - ivfflat::FLAT_TILE,
               "rows n=%lld / tiles %lld out of range", (long long)n_rows, (long long)n_tiles);
    AB_REQUIRE(k <= n_rows, "selected index k out of range: k=%d > n=%lld", k, (long long)n_rows);
    AB_REQUIRE(rows != nullptr && slot_rows != nullptr, "null pointer argument");
    AB_REQUIRE(abh::aligned(rows, 16), "rows must be 16-byte aligned");
    const bool probed = nprobe > 0 && nprobe < n_list;
    AB_REQUIRE(!probed || (coarse != nullptr && list_tile_off != nullptr && list_rows != nullptr),
               "a probed search needs coarse, list_tile_off and list_rows");
    AB_REQUIRE(nq == 0 || queries != nullptr, "queries is null");
    if (status) AB_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int32_t), s));
    if (nq == 0) return ATLAS_B200_OK;
    FlatSearchWs w;
    ProbeWs pw{};
    const int64_t n_slots = n_tiles * ivfflat::FLAT_TILE;
    size_t need = flat_search_bytes(n_slots, n_list, k, probed, &w, ws);
    if (probed) need = probe_bytes(need, n_list, n_tiles, k, ivfflat::FLAT_TILE, &pw, ws);
    if (ws == nullptr || ws_bytes < need) {
        abh::set_error("workspace too small: have %zu need %zu", ws_bytes, need);
        return ATLAS_B200_EWORKSPACE;
    }
    int rc;
    for (int q0 = 0; q0 < nq; q0 += QBLOCK) {
        const int nqb = nq - q0 < QBLOCK ? nq - q0 : QBLOCK;
        flat_query_kernel<<<QBLOCK, 256, 0, s>>>(queries + static_cast<int64_t>(q0) * DIM, nqb, w.qstage, w.qf32, w.count,
                                                 w.bound);
        abh::count_launch();
        ivfflat::ScanParams p;
        p.rows = rows;
        p.slot_rows = slot_rows;
        p.n_tiles = static_cast<int>(n_tiles);
        p.qstage = w.qstage;
        p.nq = nqb;
        p.bound = w.bound;
        p.count = w.count;
        p.cand = w.cand;
        p.capq = w.capq;
        int64_t* oi_b = out_ids + static_cast<size_t>(q0) * k;
        uint16_t* os16 = reinterpret_cast<uint16_t*>(out_scores + static_cast<size_t>(q0) * k);
        if (probed) {
            // T[l][q] = <c_l, q> (ivfsq's coarse terms), P(q) and its sample lists, then the tiles of every list some
            // query probes and the sample tiles
            if ((rc = subdot(coarse, DIM, n_list, w.qf32, nqb, DIM, 1, w.tterm, s))) return rc;
            if ((rc = ivfp::select_probes(w.tterm, 1, nqb, nqb, n_list, nullptr, list_rows, nprobe, k, w.capq,
                                          pw.sample_units * ivfflat::FLAT_TILE, pw.probed, pw.sample_lists, s)))
                return rc;
            if ((rc = ivfp::compact_items(pw.probed, pw.sample_lists, list_tile_off, n_list, 1, pw.sample_units, pw.items,
                                          pw.sample, pw.count, s)))
                return rc;
        }
        const ivfsq::ProbeScan pr{pw.items, pw.count, pw.probed};
        const ivfsq::ProbeScan ps{pw.sample, pw.count + 1, pw.probed};
        auto scan = [&](int tile_begin, int tile_step, int num_tiles, bool sample) {
            p.tile_begin = tile_begin;
            p.tile_step = tile_step;
            p.num_tiles = num_tiles;
            if (!probed) return ivfflat::launch_scan(p, nullptr, s);
            if (sample) {     // the bound's scan: every sample tile (ivf_probe.cuh), not a stride over the sweep
                p.tile_begin = 0;
                p.tile_step = 1;
                p.num_tiles = static_cast<int>(pw.max_sample);
                return ivfflat::launch_scan(p, &ps, s);
            }
            return ivfflat::launch_scan(p, &pr, s);
        };
        // work = row bytes swept (once per block)
        const double sweep_bytes = static_cast<double>(n_slots) * DIM * 2;
        if ((rc = sweep_select(scan, n_slots, static_cast<int>(n_tiles), ivfflat::FLAT_TILE, nqb, k, w.cand, w.count, w.bound,
                               w.capq, os16, oi_b, id_base, id_stride, status, exhaustive, sweep_bytes, s)))
            return rc;
    }
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // namespace pq

extern "C" {

size_t atlas_b200_pq_workspace_bytes(int32_t op, int64_t n, int32_t M, int32_t n_list, int32_t k) {
    if (!pq::valid_m(M) || n_list < 0) return 0;
    if (n < 1) n = 1;
    if (k < 1) k = 1;
    switch (op) {
        case ATLAS_B200_PQ_OP_TRAIN: return pq::train_bytes(n, M, n_list, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
        case ATLAS_B200_PQ_OP_ENCODE: return pq::encode_bytes(M, n_list, nullptr, nullptr);
        case ATLAS_B200_PQ_OP_SEARCH: return pq::search_bytes(n, M, n_list, k, nullptr, nullptr);
        case ATLAS_B200_PQ_OP_SEARCH_PROBED:
            if (n_list < 1) return 0;
            return pq::probe_bytes(pq::search_bytes(n, M, n_list, k, nullptr, nullptr), n_list, pq::pq_max_items(n, n_list),
                                   k, pq::PROBE_CHUNK, nullptr, nullptr);
        default: return 0;
    }
}

int atlas_b200_pq_train(const void* sample, int64_t n_sample, int32_t M, int32_t n_list, int32_t iters, float* codebooks,
                        float* coarse, void* workspace, size_t workspace_bytes, void* stream) {
    return pq::train(static_cast<const __half*>(sample), n_sample, M, n_list, iters, codebooks, coarse, workspace,
                     workspace_bytes, static_cast<cudaStream_t>(stream));
}

int atlas_b200_pq_encode(const void* rows, int64_t n, int32_t M, const float* codebooks, const float* coarse, int32_t n_list,
                         uint8_t* codes, void* list_ids, void* workspace, size_t workspace_bytes, void* stream) {
    return pq::encode(static_cast<const __half*>(rows), n, M, codebooks, coarse, n_list, codes, list_ids, workspace,
                      workspace_bytes, static_cast<cudaStream_t>(stream));
}

int atlas_b200_pq_topk(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M, const float* codebooks,
                       const float* coarse, int32_t n_list, const void* queries, int32_t nq, int32_t k, void* out_scores,
                       int64_t* out_ids, int64_t id_base, int64_t id_stride, int32_t* status, void* workspace,
                       size_t workspace_bytes, void* stream) {
    return pq::topk(codes, list_ids, n, M, codebooks, coarse, n_list, static_cast<const __half*>(queries), nq, k,
                    static_cast<__half*>(out_scores), out_ids, id_base, id_stride, status, workspace, workspace_bytes,
                    static_cast<cudaStream_t>(stream), false);
}

int atlas_b200_pq_topk_exhaustive(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M, const float* codebooks,
                                  const float* coarse, int32_t n_list, const void* queries, int32_t nq, int32_t k,
                                  void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride, void* workspace,
                                  size_t workspace_bytes, void* stream) {
    return pq::topk(codes, list_ids, n, M, codebooks, coarse, n_list, static_cast<const __half*>(queries), nq, k,
                    static_cast<__half*>(out_scores), out_ids, id_base, id_stride, nullptr, workspace, workspace_bytes,
                    static_cast<cudaStream_t>(stream), true);
}

int atlas_b200_pq_topk_probed(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M, const float* codebooks,
                              const float* coarse, int32_t n_list, const int32_t* list_order, const int32_t* list_offsets,
                              int32_t nprobe, const void* queries, int32_t nq, int32_t k, void* out_scores,
                              int64_t* out_ids, int64_t id_base, int64_t id_stride, int32_t* status, void* workspace,
                              size_t workspace_bytes, void* stream) {
    const pq::ProbeArgs probe{nprobe, list_order, list_offsets, nullptr};
    return pq::topk(codes, list_ids, n, M, codebooks, coarse, n_list, static_cast<const __half*>(queries), nq, k,
                    static_cast<__half*>(out_scores), out_ids, id_base, id_stride, status, workspace, workspace_bytes,
                    static_cast<cudaStream_t>(stream), false, &probe);
}

int atlas_b200_pq_topk_probed_exhaustive(const uint8_t* codes, const void* list_ids, int64_t n, int32_t M,
                                         const float* codebooks, const float* coarse, int32_t n_list,
                                         const int32_t* list_order, const int32_t* list_offsets, int32_t nprobe,
                                         const void* queries, int32_t nq, int32_t k, void* out_scores, int64_t* out_ids,
                                         int64_t id_base, int64_t id_stride, void* workspace, size_t workspace_bytes,
                                         void* stream) {
    const pq::ProbeArgs probe{nprobe, list_order, list_offsets, nullptr};
    return pq::topk(codes, list_ids, n, M, codebooks, coarse, n_list, static_cast<const __half*>(queries), nq, k,
                    static_cast<__half*>(out_scores), out_ids, id_base, id_stride, nullptr, workspace, workspace_bytes,
                    static_cast<cudaStream_t>(stream), true, &probe);
}

size_t atlas_b200_ivfsq_workspace_bytes(int32_t op, int64_t n, int32_t n_list, int32_t k) {
    if (n_list < 1) return 0;
    if (n < 1) n = 1;
    if (k < 1) k = 1;
    switch (op) {
        case ATLAS_B200_PQ_OP_TRAIN: return pq::sq_train_bytes(n, n_list, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
        case ATLAS_B200_PQ_OP_ENCODE: return pq::sq_encode_bytes(n_list, nullptr, nullptr);
        case ATLAS_B200_PQ_OP_SEARCH: return pq::sq_search_bytes(n, n_list, k, nullptr, nullptr);
        case ATLAS_B200_PQ_OP_SEARCH_PROBED:
            return pq::probe_bytes(pq::sq_search_bytes(n, n_list, k, nullptr, nullptr), n_list,
                                   (n + ivfsq::SQ_TILE - 1) / ivfsq::SQ_TILE, k, ivfsq::SQ_TILE, nullptr, nullptr);
        default: return 0;
    }
}

int atlas_b200_ivfsq_train(const void* sample, int64_t n_sample, int32_t n_list, int32_t iters, float* coarse, float* vmin,
                           float* vdiff, void* workspace, size_t workspace_bytes, void* stream) {
    return pq::sq_train(static_cast<const __half*>(sample), n_sample, n_list, iters, coarse, vmin, vdiff, workspace,
                        workspace_bytes, static_cast<cudaStream_t>(stream));
}

int atlas_b200_ivfsq_encode(const void* rows, int64_t n, const float* coarse, int32_t n_list, const float* vmin,
                            const float* vdiff, int32_t* list_ids, const int32_t* row_slot, uint8_t* codes, void* workspace,
                            size_t workspace_bytes, void* stream) {
    return pq::sq_encode(static_cast<const __half*>(rows), n, coarse, n_list, vmin, vdiff, list_ids, row_slot, codes,
                         workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int atlas_b200_ivfsq_topk(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists, int64_t n_tiles,
                          int64_t n_rows, const float* coarse, int32_t n_list, const float* vmin, const float* vdiff,
                          const void* queries, int32_t nq, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                          int64_t id_stride, int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
    return pq::sq_topk(codes, slot_rows, tile_lists, n_tiles, n_rows, coarse, n_list, vmin, vdiff,
                       static_cast<const __half*>(queries), nq, k, static_cast<__half*>(out_scores), out_ids, id_base,
                       id_stride, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), false);
}

int atlas_b200_ivfsq_topk_exhaustive(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists,
                                     int64_t n_tiles, int64_t n_rows, const float* coarse, int32_t n_list, const float* vmin,
                                     const float* vdiff, const void* queries, int32_t nq, int32_t k, void* out_scores,
                                     int64_t* out_ids, int64_t id_base, int64_t id_stride, void* workspace,
                                     size_t workspace_bytes, void* stream) {
    return pq::sq_topk(codes, slot_rows, tile_lists, n_tiles, n_rows, coarse, n_list, vmin, vdiff,
                       static_cast<const __half*>(queries), nq, k, static_cast<__half*>(out_scores), out_ids, id_base,
                       id_stride, nullptr, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), true);
}

int atlas_b200_ivfsq_topk_probed(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists, int64_t n_tiles,
                                 int64_t n_rows, const int32_t* list_tile_off, const int32_t* list_rows, const float* coarse,
                                 int32_t n_list, const float* vmin, const float* vdiff, int32_t nprobe, const void* queries,
                                 int32_t nq, int32_t k, void* out_scores, int64_t* out_ids, int64_t id_base,
                                 int64_t id_stride, int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
    const pq::ProbeArgs probe{nprobe, nullptr, list_tile_off, list_rows};
    return pq::sq_topk(codes, slot_rows, tile_lists, n_tiles, n_rows, coarse, n_list, vmin, vdiff,
                       static_cast<const __half*>(queries), nq, k, static_cast<__half*>(out_scores), out_ids, id_base,
                       id_stride, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), false, &probe);
}

int atlas_b200_ivfsq_topk_probed_exhaustive(const uint8_t* codes, const int32_t* slot_rows, const int32_t* tile_lists,
                                            int64_t n_tiles, int64_t n_rows, const int32_t* list_tile_off,
                                            const int32_t* list_rows, const float* coarse, int32_t n_list, const float* vmin,
                                            const float* vdiff, int32_t nprobe, const void* queries, int32_t nq, int32_t k,
                                            void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride,
                                            void* workspace, size_t workspace_bytes, void* stream) {
    const pq::ProbeArgs probe{nprobe, nullptr, list_tile_off, list_rows};
    return pq::sq_topk(codes, slot_rows, tile_lists, n_tiles, n_rows, coarse, n_list, vmin, vdiff,
                       static_cast<const __half*>(queries), nq, k, static_cast<__half*>(out_scores), out_ids, id_base,
                       id_stride, nullptr, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), true, &probe);
}

size_t atlas_b200_ivfflat_workspace_bytes(int32_t op, int64_t n_slots, int32_t n_list, int32_t k) {
    if (n_list < 1) return 0;
    if (n_slots < 1) n_slots = 1;
    if (k < 1) k = 1;
    switch (op) {
        case ATLAS_B200_PQ_OP_SEARCH: return pq::flat_search_bytes(n_slots, n_list, k, false, nullptr, nullptr);
        case ATLAS_B200_PQ_OP_SEARCH_PROBED:
            return pq::probe_bytes(pq::flat_search_bytes(n_slots, n_list, k, true, nullptr, nullptr), n_list,
                                   (n_slots + ivfflat::FLAT_TILE - 1) / ivfflat::FLAT_TILE, k, ivfflat::FLAT_TILE, nullptr,
                                   nullptr);
        default: return 0;
    }
}

int atlas_b200_ivfflat_topk(const void* rows, const int32_t* slot_rows, int64_t n_tiles, int64_t n_rows,
                            const int32_t* list_tile_off, const int32_t* list_rows, const float* coarse, int32_t n_list,
                            int32_t nprobe, const void* queries, int32_t nq, int32_t k, void* out_scores, int64_t* out_ids,
                            int64_t id_base, int64_t id_stride, int32_t* status, void* workspace, size_t workspace_bytes,
                            void* stream) {
    return pq::flat_topk(static_cast<const __half*>(rows), slot_rows, n_tiles, n_rows, list_tile_off, list_rows, coarse, n_list,
                         nprobe, static_cast<const __half*>(queries), nq, k, static_cast<__half*>(out_scores), out_ids, id_base,
                         id_stride, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), false);
}

int atlas_b200_ivfflat_topk_exhaustive(const void* rows, const int32_t* slot_rows, int64_t n_tiles, int64_t n_rows,
                                       const int32_t* list_tile_off, const int32_t* list_rows, const float* coarse,
                                       int32_t n_list, int32_t nprobe, const void* queries, int32_t nq, int32_t k,
                                       void* out_scores, int64_t* out_ids, int64_t id_base, int64_t id_stride, void* workspace,
                                       size_t workspace_bytes, void* stream) {
    return pq::flat_topk(static_cast<const __half*>(rows), slot_rows, n_tiles, n_rows, list_tile_off, list_rows, coarse, n_list,
                         nprobe, static_cast<const __half*>(queries), nq, k, static_cast<__half*>(out_scores), out_ids, id_base,
                         id_stride, nullptr, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), true);
}

}  // extern "C"
