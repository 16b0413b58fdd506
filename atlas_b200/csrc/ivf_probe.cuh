// Probed IVF search (`nprobe`): the probe selection and the work-list compaction shared by the ivfpq scan (csrc/pq.cu)
// and the ivfsq scan (csrc/ivfsq.cu).  The kernels are in ivf_probe.cu.
//
// Rule (restated in oracle/ivf_probe_oracle.py): for query q of a select block, with T[q][l] the fp32 coarse term the
// scan adds (<q, c_l> from the fp16-rounded query), the lists are ordered by T descending, then by list id ascending;
// the probe set P(q) is the shortest prefix of that order with at least nprobe lists that holds at least k real rows.
//
// Device state of one select block:
//   probed  uint32 [n_list][PROBE_WORDS]: bit q % 32 of word q / 32 of list l is set when l is in P(q) (32 B per list)
//   items   int2 [count]: the work items of the probed sweep, (list, first unit), in list order - one 64-slot tile of
//           an ivfsq list, or one chunk of `unit` list positions of an ivfpq list - for every list some query probes
//   count   int32 in device memory: the scans read it; the host sizes their grids from an upper bound, so nothing
//           synchronises with the host
//   sample  the items of the scan that sets each query's candidate bound: the first `sample_rows` positions of each of
//           the first lists of every query's order, until they hold max(k, 4 k |P(q)| / capq) of its rows (or P(q) is
//           used up); `sample_lists[l]` marks them, and the sample items and their count sit next to the others.  Every
//           query's sample lies inside its own probe set, so its bound is the k-th best of at least k of its own rows
//           (k <= sample_rows), and about 4 k / capq of its probed rows pass it: the sweep's candidates fit.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace ivfp {

constexpr int PROBE_QBLOCK = 256;                // queries per select block
constexpr int PROBE_WORDS = PROBE_QBLOCK / 32;   // mask words per list

// does any query of [q0, q0 + nq) probe list l?  (nq >= 1)
__device__ __forceinline__ bool group_probes(const uint32_t* __restrict__ probed, int l, int q0, int nq) {
    const uint32_t* words = probed + static_cast<int64_t>(l) * PROBE_WORDS;
    uint32_t any = 0;
    for (int w = q0 >> 5; w <= (q0 + nq - 1) >> 5; ++w) {
        const int lo = (q0 > 32 * w ? q0 : 32 * w) - 32 * w;                          // the group's bits [lo, hi) of word w
        const int hi = (q0 + nq < 32 * w + 32 ? q0 + nq : 32 * w + 32) - 32 * w;
        any |= __ldg(words + w) & (hi - lo == 32 ? 0xFFFFFFFFu : ((1u << (hi - lo)) - 1u) << lo);
    }
    return any != 0;
}

__device__ __forceinline__ bool probes(const uint32_t* __restrict__ probed, int l, int q) {
    return (__ldg(probed + static_cast<int64_t>(l) * PROBE_WORDS + (q >> 5)) >> (q & 31)) & 1u;
}

// The items a scan launch covers, given the compacted count n read from device memory: items begin + i * step,
// i < num, that lie below n (chunks past the count do nothing).
__device__ __forceinline__ void resolve_items(int n, int begin, int step, int num, int& b, int& st, int& cnt) {
    b = begin;
    st = step;
    const int left = n > begin ? (n - begin + step - 1) / step : 0;
    cnt = num < left ? num : left;
}

// probed = 0 and sample_lists = 0, then P(q) and the sample lists of every query q < nqb: T[q][l] = T[q * ldq +
// l * ldl]; the real rows of list l are row_cnt[l], or row_off[l + 1] - row_off[l] when row_cnt is NULL, and lead
// the list.  1 <= k <= the rows of all lists, k <= sample_rows.
int select_probes(const float* T, int64_t ldq, int64_t ldl, int nqb, int n_list, const int32_t* row_off,
                  const int32_t* row_cnt, int nprobe, int k, uint32_t capq, int sample_rows, uint32_t* probed,
                  uint32_t* sample_lists, cudaStream_t s);

// items / count[0] of a select block: list l, when some query probes it, contributes its ceil((unit_off[l + 1] -
// unit_off[l]) / unit) items (l, unit_off[l] + unit * j), at most n_list + sum of those, which the caller bounds;
// sample / count[1]: the first min(that, sample_units) items of every sample list.  One CTA; the items of a list are
// written by one thread, so a list far longer than the others serialises its part.
int compact_items(const uint32_t* probed, const uint32_t* sample_lists, const int32_t* unit_off, int n_list, int unit,
                  int sample_units, int2* items, int2* sample, int32_t* count, cudaStream_t s);

}  // namespace ivfp
