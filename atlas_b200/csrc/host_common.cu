#include "host_common.h"

#include <stdarg.h>
#include <string.h>

#include <utility>
#include <vector>

namespace abh {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
        set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
        return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

int make_tmap_2d_16bit(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols, bool bf16) {
    EncodeTiledFn fn = get_encode();
    if (!fn) return ATLAS_B200_ECUDA;
    if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0 || (ld * 2) % 16 != 0) {
        set_error("tensor map: base must be 16-byte aligned and the row stride a multiple of 16 bytes");
        return ATLAS_B200_EINVAL;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                    const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%llu cols=%llu ld=%llu box=%ux%u)", (int)r,
                  (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows, box_cols);
        return ATLAS_B200_ECUDA;
    }
    return ATLAS_B200_OK;
}

int make_tmap_2d_bytes(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                       uint32_t box_cols) {
    EncodeTiledFn fn = get_encode();
    if (!fn) return ATLAS_B200_ECUDA;
    if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0 || ld % 16 != 0) {
        set_error("tensor map: base must be 16-byte aligned and the row stride a multiple of 16 bytes");
        return ATLAS_B200_EINVAL;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%llu cols=%llu ld=%llu box=%ux%u)", (int)r,
                  (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows, box_cols);
        return ATLAS_B200_ECUDA;
    }
    return ATLAS_B200_OK;
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

// ---- profiling of the dominant kernel -------------------------------------------------------
static int g_prof_on = 0;   // 0 off, otherwise the ProfKind being bracketed
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;
static size_t g_prof_used = 0;
static double g_prof_work = 0;
struct DynWork {                 // launches whose row count lives in device memory: the count is copied to a pinned host slot
    double work_per_row;         // in stream order right behind the launch (the device tensor may be recycled by the caller's
    int slot;                    // allocator before the work is read) and resolved when the work is read
    int32_t m_max;
};
static std::vector<DynWork> g_prof_dyn;
struct LaunchWork {              // per bracketed launch, in launch order: static work, or the index of its DynWork entry
    double work;
    int dyn;
};
static std::vector<LaunchWork> g_prof_launch;
static int32_t* g_prof_rows = nullptr;          // pinned host slots
constexpr int PROF_ROW_SLOTS = 4096;

void prof_begin(cudaStream_t s, int kind) {
    if (g_prof_on != kind) return;
    if (g_prof_used == g_prof_events.size()) {
        cudaEvent_t a, b;
        if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return;
        g_prof_events.emplace_back(a, b);
    }
    cudaEventRecord(g_prof_events[g_prof_used].first, s);
}

void prof_end(cudaStream_t s, int kind, double work) {
    if (g_prof_on != kind || g_prof_used >= g_prof_events.size()) return;
    cudaEventRecord(g_prof_events[g_prof_used].second, s);
    ++g_prof_used;
    g_prof_work += work;
    g_prof_launch.push_back({work, -1});
}

// the work of the launch just bracketed: work_per_row * *m_dev, copied to a pinned host slot in stream order
static void dyn_work(cudaStream_t s, double work_per_row, const int32_t* m_dev, int32_t m_max) {
    if (g_prof_rows == nullptr && cudaMallocHost(reinterpret_cast<void**>(&g_prof_rows), PROF_ROW_SLOTS * sizeof(int32_t)) != cudaSuccess)
        g_prof_rows = nullptr;
    const int slot = static_cast<int>(g_prof_dyn.size());
    if (g_prof_rows != nullptr && slot < PROF_ROW_SLOTS) {
        g_prof_rows[slot] = m_max;
        if (cudaMemcpyAsync(g_prof_rows + slot, m_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, s) == cudaSuccess) {
            g_prof_dyn.push_back({work_per_row, slot, m_max});
            g_prof_launch.push_back({0.0, slot});
            return;
        }
    }
    g_prof_work += work_per_row * m_max;          // no slot: counted at full height
    g_prof_launch.push_back({work_per_row * m_max, -1});
}

void prof_end_dyn(cudaStream_t s, int kind, double work_per_row, const int32_t* m_dev, int32_t m_max) {
    if (g_prof_on != kind || g_prof_used >= g_prof_events.size()) return;
    cudaEventRecord(g_prof_events[g_prof_used].second, s);
    ++g_prof_used;
    dyn_work(s, work_per_row, m_dev, m_max);
}

// sum over the segments of popcount(keep[b, :])^2: the (query tile, key tile) pairs of the packed encoder's attention
__global__ void tile_pairs_kernel(const uint8_t* __restrict__ keep, int S, int nb, int32_t* __restrict__ pairs) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < S; b += gridDim.x * blockDim.x) {
        int n = 0;
        for (int t = 0; t < nb; ++t) n += keep[static_cast<size_t>(b) * nb + t] != 0;
        atomicAdd(pairs, n * n);
    }
}

void prof_end_tile_pairs(cudaStream_t s, int kind, double work_per_pair, const uint8_t* keep, int32_t S, int32_t nb) {
    if (g_prof_on != kind || g_prof_used >= g_prof_events.size()) return;
    cudaEventRecord(g_prof_events[g_prof_used].second, s);
    ++g_prof_used;
    static int32_t* pairs = nullptr;               // one counter, reused in stream order (each count is copied out behind it)
    if (pairs == nullptr && cudaMalloc(reinterpret_cast<void**>(&pairs), sizeof(int32_t)) != cudaSuccess) pairs = nullptr;
    if (pairs != nullptr && cudaMemsetAsync(pairs, 0, sizeof(int32_t), s) == cudaSuccess) {
        tile_pairs_kernel<<<(S + 255) / 256, 256, 0, s>>>(keep, S, nb, pairs);
        if (cudaGetLastError() == cudaSuccess) {
            dyn_work(s, work_per_pair, pairs, S * nb * nb);
            return;
        }
    }
    g_prof_work += work_per_pair * S * nb * nb;    // no count: every tile pair
    g_prof_launch.push_back({work_per_pair * S * nb * nb, -1});
}

}  // namespace abh

extern "C" {

void atlas_b200_profile_enable(int32_t kind) {
    abh::g_prof_on = kind;
    abh::g_prof_used = 0;
    abh::g_prof_work = 0;
    abh::g_prof_dyn.clear();
    abh::g_prof_launch.clear();
}

// the work of the bracketed launches; launches with a device-side row count are counted with the rows they really computed
// (read back here: call after the stream has been synchronised)
double atlas_b200_profile_work(void) {
    double w = abh::g_prof_work;
    for (const auto& d : abh::g_prof_dyn) {
        int32_t m = abh::g_prof_rows[d.slot];
        if (m > d.m_max) m = d.m_max;
        if (m < 0) m = 0;
        w += d.work_per_row * m;
    }
    return w;
}

// per bracketed launch, in launch order: its event-bracketed time and its work (device-side row counts resolved); returns the number
// of launches written (<= cap).  Call after the stream has been synchronised and BEFORE atlas_b200_profile_collect.
int32_t atlas_b200_profile_launches(double* ms, double* work, int32_t cap) {
    const size_t n = abh::g_prof_used < abh::g_prof_launch.size() ? abh::g_prof_used : abh::g_prof_launch.size();
    int32_t written = 0;
    for (size_t i = 0; i < n && written < cap; ++i, ++written) {
        float t = 0;
        if (cudaEventSynchronize(abh::g_prof_events[i].second) != cudaSuccess ||
            cudaEventElapsedTime(&t, abh::g_prof_events[i].first, abh::g_prof_events[i].second) != cudaSuccess)
            t = 0;
        const abh::LaunchWork& lw = abh::g_prof_launch[i];
        double w = lw.work;
        if (lw.dyn >= 0) {
            const abh::DynWork& d = abh::g_prof_dyn[lw.dyn];
            int32_t m = abh::g_prof_rows[d.slot];
            m = m > d.m_max ? d.m_max : (m < 0 ? 0 : m);
            w = d.work_per_row * m;
        }
        if (ms) ms[written] = t;
        if (work) work[written] = w;
    }
    return written;
}

int atlas_b200_profile_collect(double* total_ms, int32_t* launches) {
    double tot = 0;
    for (size_t i = 0; i < abh::g_prof_used; ++i) {
        float ms = 0;
        AB_CUDA_CHECK(cudaEventSynchronize(abh::g_prof_events[i].second));
        AB_CUDA_CHECK(cudaEventElapsedTime(&ms, abh::g_prof_events[i].first, abh::g_prof_events[i].second));
        tot += ms;
    }
    if (total_ms) *total_ms = tot;
    if (launches) *launches = static_cast<int32_t>(abh::g_prof_used);
    abh::g_prof_used = 0;
    return ATLAS_B200_OK;
}


const char* atlas_b200_last_error(void) { return abh::g_err; }
const char* atlas_b200_version(void) { return "atlas_b200 0.2 (sm_90a)"; }
uint64_t atlas_b200_launch_count(void) { return abh::g_launches.load(); }

}  // extern "C"
