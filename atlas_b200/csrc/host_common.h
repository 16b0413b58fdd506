// Host-side helpers shared by the C-ABI translation units: error reporting, launch counting,
// TMA tensor-map creation through the runtime's driver entry point (so the library does not link
// libcuda and still dlopen()s on a machine without a GPU driver).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/atlas_b200.h"

namespace abh {

void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

inline void count_launch(int n = 1) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

#define AB_CUDA_CHECK(expr)                                                                       \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) {                                                                  \
            abh::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return ATLAS_B200_ECUDA;                                                              \
        }                                                                                         \
    } while (0)

#define AB_REQUIRE(cond, ...)           \
    do {                                \
        if (!(cond)) {                  \
            abh::set_error(__VA_ARGS__); \
            return ATLAS_B200_EINVAL;   \
        }                               \
    } while (0)

// 2-D row-major tensor map: `rows` x `cols` elements of 2 bytes, row stride `ld` elements,
// box = {box_cols, box_rows}, 128-byte swizzle (box_cols * 2 must be 128).
int make_tmap_2d_16bit(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols, bool bf16);

// 2-D row-major tensor map of bytes: `rows` x `cols`, row stride `ld` bytes, box = {box_cols, box_rows}, no swizzle.
int make_tmap_2d_bytes(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                       uint32_t box_cols);

int num_sms();

// Optional CUDA-event bracketing of the dominant kernel (bench.py's roofline measurement): when
// enabled, callers wrap that launch with prof_begin/prof_end on the launching stream.
enum ProfKind {
    PROF_SCAN = 1,
    PROF_LINEAR = 2,
    PROF_ATTENTION = 3,
    PROF_ATTENTION_BWD = 4,
    PROF_DECODE_CROSS = 5,
    PROF_BEAM_SELECT = 6,     // beam_topk + beam_select (csrc/beam.cu); work = bytes read
    PROF_PQ_REFINE = 7,       // pq_refine_kernel (csrc/pq_refine.cu); work = host-row bytes read
};
void prof_begin(cudaStream_t s, int kind);
void prof_end(cudaStream_t s, int kind, double work);   // work = algorithmic bytes (scan) or FLOPs of this launch
// ... of a launch whose row count lives in device memory: work = work_per_row * min(m_max, *m_dev), resolved when read
void prof_end_dyn(cudaStream_t s, int kind, double work_per_row, const int32_t* m_dev, int32_t m_max);
// ... of a launch over the packed encoder rows (atlas_b200_segment_tile_scan's keep [S, nb]): work = work_per_pair times the
// (query tile, key tile) pairs of the kept tiles, counted on the device only while `kind` is being measured
void prof_end_tile_pairs(cudaStream_t s, int kind, double work_per_pair, const uint8_t* keep, int32_t S, int32_t nb);

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// true when p is a multiple of `a` bytes (a power of two); NULL counts as aligned (optional operands are checked by the caller)
inline bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace abh
