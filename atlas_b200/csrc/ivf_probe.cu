// Probed IVF search (`nprobe`, ivfpq and ivfsq): the per-query probe selection and the compaction of the probed lists
// into the work items of the sweep.  Rule and state: ivf_probe.cuh.
#include "common.cuh"
#include "host_common.h"
#include "ivf_probe.cuh"

namespace ivfp {

constexpr int SEL_THREADS = 256;
constexpr int COMPACT_THREADS = 1024;

// order key of list l for one query: sortable fp32 bits of T (-0 as +0) above the complemented list id, so that the
// larger key is the larger T and, on equal T, the lower list id
__device__ __forceinline__ uint64_t list_key(float v, int l) {
    uint32_t b = __float_as_uint(v);
    if (b == 0x80000000u) b = 0;
    b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return (static_cast<uint64_t>(b) << 32) | static_cast<uint64_t>(0xFFFFFFFFu - static_cast<uint32_t>(l));
}

__device__ __forceinline__ uint64_t block_max_u64(uint64_t v, uint64_t* s_red) {
    for (int o = 16; o > 0; o >>= 1) {
        const uint64_t y = __shfl_xor_sync(0xffffffffu, v, o);
        v = y > v ? y : v;
    }
    const int w = threadIdx.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[w] = v;
    __syncthreads();
    uint64_t r = 0;
    for (int i = 0; i < SEL_THREADS / 32; ++i) r = s_red[i] > r ? s_red[i] : r;
    return r;
}

__device__ __forceinline__ int64_t block_sum_i64(int64_t v, int64_t* s_red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[w] = v;
    __syncthreads();
    int64_t r = 0;
    for (int i = 0; i < SEL_THREADS / 32; ++i) r += s_red[i];
    return r;
}

// One CTA per query: radix select of the nprobe-th largest list key (8-bit digits, most significant first), then the
// extension by the next lists while the selected ones hold fewer than k rows (small shards only: one block max each),
// then the sample lists: the best probed lists, one block max each, until their first sample_rows positions hold
// the query's sample target.
__global__ void __launch_bounds__(SEL_THREADS)
ivf_probe_select_kernel(const float* __restrict__ T, int64_t ldq, int64_t ldl, int n_list, const int32_t* __restrict__ row_off,
                        const int32_t* __restrict__ row_cnt, int nprobe, int k, uint32_t capq, int sample_rows,
                        uint32_t* __restrict__ probed, uint32_t* __restrict__ sample_lists) {
    __shared__ uint32_t hist[256];
    __shared__ uint64_t s_prefix;
    __shared__ uint32_t s_krem;
    __shared__ uint64_t s_red64[SEL_THREADS / 32];
    __shared__ int64_t s_redi[SEL_THREADS / 32];
    const int q = blockIdx.x, t = threadIdx.x;
    const float* Tq = T + static_cast<int64_t>(q) * ldq;
    auto key = [&](int l) { return list_key(Tq[static_cast<int64_t>(l) * ldl], l); };
    auto rows = [&](int l) { return row_cnt ? row_cnt[l] : row_off[l + 1] - row_off[l]; };

    const uint32_t p = static_cast<uint32_t>(nprobe < n_list ? nprobe : n_list);
    if (t == 0) {
        s_prefix = 0;
        s_krem = p;
    }
    uint64_t mask = 0;
    for (int b = 7; b >= 0; --b) {
        hist[t] = 0;
        __syncthreads();
        const uint64_t prefix = s_prefix;
        for (int l = t; l < n_list; l += SEL_THREADS) {
            const uint64_t kl = key(l);
            if ((kl & mask) == prefix) atomicAdd(&hist[(kl >> (8 * b)) & 0xFFu], 1u);
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
    uint64_t thr = s_prefix;   // the p-th largest key: the lists with key >= thr are the first p of the order

    int64_t held = 0;
    for (int l = t; l < n_list; l += SEL_THREADS)
        if (key(l) >= thr) held += rows(l);
    held = block_sum_i64(held, s_redi);
    while (held < k) {
        uint64_t next = 0;
        for (int l = t; l < n_list; l += SEL_THREADS) {
            const uint64_t kl = key(l);
            if (kl < thr && kl > next) next = kl;
        }
        next = block_max_u64(next, s_red64);
        if (next == 0) break;      // every list is selected (k <= the rows of all lists: not reached)
        thr = next;
        held += rows(static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(thr)));
    }
    for (int l = t; l < n_list; l += SEL_THREADS)
        if (key(l) >= thr) atomicOr(&probed[static_cast<int64_t>(l) * PROBE_WORDS + (q >> 5)], 1u << (q & 31));

    // sample lists: the query's best lists until their sampled prefixes hold max(k, 4 k |P(q)| / capq) of its rows
    double want = 4.0 * static_cast<double>(k) * static_cast<double>(held) / static_cast<double>(capq);
    if (want < k) want = k;
    const int64_t target = want < static_cast<double>(held) ? static_cast<int64_t>(ceil(want)) : held;
    int64_t sampled = 0;
    uint64_t cur = ~0ull;
    while (sampled < target) {
        uint64_t next = 0;
        for (int l = t; l < n_list; l += SEL_THREADS) {
            const uint64_t kl = key(l);
            if (kl >= thr && kl < cur && kl > next) next = kl;
        }
        next = block_max_u64(next, s_red64);
        if (next == 0) break;      // P(q) used up
        cur = next;
        const int l = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(cur));
        const int r = rows(l);
        sampled += r < sample_rows ? r : sample_rows;
        if (t == 0) sample_lists[l] = 1u;
    }
}

// exclusive block scan of v over COMPACT_THREADS threads, plus the block total
__device__ __forceinline__ int block_scan(int v, int* s_warp, int& total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    __syncthreads();
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();
    int off = 0;
    total = 0;
    for (int i = 0; i < COMPACT_THREADS / 32; ++i) {
        off += i < w ? s_warp[i] : 0;
        total += s_warp[i];
    }
    return off + incl - v;
}

// One CTA: lists in order, COMPACT_THREADS at a time; each probed list's item count and each sample list's sample item
// count, block exclusive scans, the items.
__global__ void __launch_bounds__(COMPACT_THREADS)
ivf_compact_kernel(const uint32_t* __restrict__ probed, const uint32_t* __restrict__ sample_lists,
                   const int32_t* __restrict__ unit_off, int n_list, int unit, int sample_units, int2* __restrict__ items,
                   int2* __restrict__ sample, int32_t* __restrict__ count) {
    __shared__ int s_warp[COMPACT_THREADS / 32];
    const int t = threadIdx.x;
    int base = 0, sbase = 0;     // block-uniform
    for (int l0 = 0; l0 < n_list; l0 += COMPACT_THREADS) {
        const int l = l0 + t;
        int nu = 0, ns = 0;
        if (l < n_list) {
            uint32_t any = 0;
#pragma unroll
            for (int i = 0; i < PROBE_WORDS; ++i) any |= probed[static_cast<int64_t>(l) * PROBE_WORDS + i];
            if (any) nu = (unit_off[l + 1] - unit_off[l] + unit - 1) / unit;
            if (sample_lists[l]) ns = nu < sample_units ? nu : sample_units;
        }
        int total, stotal;
        const int off = base + block_scan(nu, s_warp, total);
        const int soff = sbase + block_scan(ns, s_warp, stotal);
        for (int j = 0; j < nu; ++j) items[off + j] = make_int2(l, unit_off[l] + unit * j);
        for (int j = 0; j < ns; ++j) sample[soff + j] = make_int2(l, unit_off[l] + unit * j);
        base += total;
        sbase += stotal;
    }
    if (t == 0) {
        count[0] = base;
        count[1] = sbase;
    }
}

int select_probes(const float* T, int64_t ldq, int64_t ldl, int nqb, int n_list, const int32_t* row_off,
                  const int32_t* row_cnt, int nprobe, int k, uint32_t capq, int sample_rows, uint32_t* probed,
                  uint32_t* sample_lists, cudaStream_t s) {
    AB_CUDA_CHECK(cudaMemsetAsync(probed, 0, static_cast<size_t>(n_list) * PROBE_WORDS * sizeof(uint32_t), s));
    AB_CUDA_CHECK(cudaMemsetAsync(sample_lists, 0, static_cast<size_t>(n_list) * sizeof(uint32_t), s));
    ivf_probe_select_kernel<<<nqb, SEL_THREADS, 0, s>>>(T, ldq, ldl, n_list, row_off, row_cnt, nprobe, k, capq, sample_rows,
                                                        probed, sample_lists);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

int compact_items(const uint32_t* probed, const uint32_t* sample_lists, const int32_t* unit_off, int n_list, int unit,
                  int sample_units, int2* items, int2* sample, int32_t* count, cudaStream_t s) {
    ivf_compact_kernel<<<1, COMPACT_THREADS, 0, s>>>(probed, sample_lists, unit_off, n_list, unit, sample_units, items,
                                                     sample, count);
    abh::count_launch();
    AB_CUDA_CHECK(cudaGetLastError());
    return ATLAS_B200_OK;
}

}  // namespace ivfp
