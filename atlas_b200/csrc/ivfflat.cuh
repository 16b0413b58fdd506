// IVF-Flat passage index (`--index_mode faiss`, types ivfflat and flat): the device layout shared by the search host code
// (csrc/pq.cu) and the row scan (csrc/ivfflat.cu).
//
// The layout is ivfsq's (ivfsq.cuh) with fp16 rows in place of codes: rows are stable-sorted by list and every list is
// padded to a multiple of FLAT_TILE slots, so each FLAT_TILE-slot tile belongs to one list.  A slot holds the 768 fp16
// values of one row (1536 bytes, zero for padding); `slot_rows[slot]` is its local row (-1 for padding).  Type flat is
// the same layout with one list: the rows in row order, padded to a multiple of FLAT_TILE.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/atlas_b200.h"
#include "ivfsq.cuh"

namespace ivfflat {

constexpr int FLAT_DIM = ATLAS_B200_EMBEDDINGS_DIM;
constexpr int FLAT_TILE = 64;        // slots per tile: one list per tile, two tiles per wgmma N = 128 step
constexpr int FLAT_QBLOCK = 256;     // queries per select block (mips.cu's candidate layout)

struct ScanParams {
    const __half* rows;          // [n_tiles * FLAT_TILE][768], 16-byte aligned
    const int32_t* slot_rows;    // [n_tiles * FLAT_TILE]
    int n_tiles;
    const __half* qstage;        // [FLAT_QBLOCK][768] fp16 queries (zero rows past nq)
    int nq;                      // valid queries in this block
    int tile_begin, tile_step, num_tiles;
    const float* bound;
    uint32_t* count;
    uint64_t* cand;
    uint32_t capq;
};

// Scans tiles tile_begin + i * tile_step, i < num_tiles, for every query of the block; appends (fp16 score, row) of every
// real slot whose score is >= bound[q] to the query's candidate list.
// probe != NULL: the tiles are those of probe->items (ivf_probe.cuh's resolve_items over *item_count), and a slot is
// appended for query q only when q probes the tile's list; num_tiles is then the host's upper bound of the item count.
int launch_scan(const ScanParams& p, const ivfsq::ProbeScan* probe, cudaStream_t s);

}  // namespace ivfflat
