// IVF-SQ passage index (`--index_mode faiss`, type ivfsq): the device layout shared by the encoder (csrc/pq.cu) and the
// code scan (csrc/ivfsq.cu).
//
// Rows are stored in inverted-list order: rows are stable-sorted by list and every list is padded to a multiple of
// SQ_TILE slots, so each SQ_TILE-slot tile belongs to one list.  A slot holds the 768 4-bit codes of one row in
// SQ_CODE_BYTES bytes; `slot_rows[slot]` is its local row (-1 for padding) and `tile_lists[tile]` its list.
//
// Nibble order inside a slot (chosen for the register-A fragment of wgmma m64nNk16): K-block kb (64 dims) owns the
// 32 bytes [32 kb, 32 kb + 32).  In it, quad lane j = 0..3 of the fragment owns 8 bytes: two 32-bit words, one per pair
// of k16 steps (s, s + 1).  Of the fragment's dims c = 2j, c + 1, c + 8, c + 9 of step s, the low nibbles of bytes 0
// and 2 hold c and c + 1, the high nibbles c + 8 and c + 9; bytes 1 and 3 hold the same dims of step s + 1.  So
// `w & 0x000F000F`, OR-ed with 0x6400 0x6400, is the fp16 pair (c, c + 1) of step s plus 1024, and the other three
// pairs follow with the mask 0x00F000F0 and a shift by 8.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/atlas_b200.h"

namespace ivfsq {

constexpr int SQ_DIM = ATLAS_B200_EMBEDDINGS_DIM;
constexpr int SQ_TILE = 64;                  // slots per tile (wgmma M)
constexpr int SQ_CODE_BYTES = SQ_DIM / 2;    // 384
constexpr int SQ_KBLOCK_BYTES = 32;          // code bytes of one slot per 64-dim K-block
constexpr int SQ_QBLOCK = 256;               // queries per select block (mips.cu's candidate layout)

// nibble position (2 * byte + high) of dim d inside a slot
__host__ __device__ inline int sq_nibble_of_dim(int d) {
    const int kb = d / 64, s = (d % 64) / 16, c = d % 16;
    const int j = (c % 8) / 2, e = c % 2, hi = c / 8;
    const int byte = kb * 32 + j * 8 + (s / 2) * 4 + (s % 2) + 2 * e;
    return 2 * byte + hi;
}

// dim held by nibble position p of a slot (the inverse of sq_nibble_of_dim)
__host__ __device__ inline int sq_dim_of_nibble(int p) {
    const int byte = p / 2, hi = p % 2;
    const int kb = byte / 32, j = (byte % 32) / 8, w = (byte % 8) / 4, b = byte % 2, e = (byte % 4) / 2;
    return kb * 64 + (2 * w + b) * 16 + hi * 8 + 2 * j + e;
}

struct ScanParams {
    const uint8_t* codes;        // [n_tiles * SQ_TILE][SQ_CODE_BYTES], 16-byte aligned
    const int32_t* slot_rows;    // [n_tiles * SQ_TILE]
    const int32_t* tile_lists;   // [n_tiles]
    int n_tiles;
    const __half* what;          // [SQ_QBLOCK][768] fp16 query operand w^ (zero rows past nq)
    const float* tterm;          // [n_list][ldt]: <q, c_l> of this block's queries
    int ldt;
    const float* cterm;          // [SQ_QBLOCK]
    const float* scale;          // [SQ_QBLOCK] 2^-e_q
    int nq;                      // valid queries in this block
    int tile_begin, tile_step, num_tiles;
    const float* bound;
    uint32_t* count;
    uint64_t* cand;
    uint32_t capq;
};

// A probed scan's state (a separate kernel argument: the full scan's parameters stay as they are)
struct ProbeScan {
    const int2* items;           // the block's compacted (list, tile) items and their count in device memory
    const int32_t* item_count;
    const uint32_t* probed;      // [n_list][PROBE_WORDS] probe bits of the block's queries
};

// Scans tiles tile_begin + i * tile_step, i < num_tiles, for every query of the block; appends (fp16 key, row) of every
// real slot whose score is >= bound[q] to the query's candidate list.
// probe != NULL: the tiles are those of probe->items (ivf_probe.cuh's resolve_items over *item_count), and a slot is
// appended for query q only when q probes the tile's list; num_tiles is then the host's upper bound of the item count.
int launch_scan(const ScanParams& p, const ProbeScan* probe, cudaStream_t s);

}  // namespace ivfsq
