"""TEST INFRASTRUCTURE - CPU restatement of the padding-compaction tables (atlas_b200_segment_tile_scan, include/atlas_b200.h).

The reference has no such table: it encodes every reader passage padded to `text_maxlength` (src/atlas.py:261-270 builds the
padded batch, src/fid.py:32-78 runs T5Stack on all `[B * n, L]` positions) and masks the padding keys with -10000
(transformers 4.18 `get_extended_attention_mask`, call site src/modeling_t5.py:941).  The product keeps, per passage, the
64-position tiles up to the LAST one holding a live key; this module states that rule in plain numpy so the CUDA tables can be
checked element by element (tests/test_packed_encoder_gpu.py) and pins the rule itself on hand-written cases
(tests/test_padding_invariance_cpu.py).  Only tests may import it."""
import numpy as np

TILE = 64


def live_tiles(attention_mask, tile=TILE):
    """attention_mask [S, L] (1 = real token) -> uint8 [S, ceil(L / tile)]: 1 where the tile holds a real token; a segment
    without any real token keeps every tile live (its softmax is uniform over masked keys in the reference too)."""
    m = np.asarray(attention_mask).astype(bool)
    S, L = m.shape
    nb = -(-L // tile)
    pad = np.zeros((S, nb * tile), dtype=bool)
    pad[:, :L] = m
    live = pad.reshape(S, nb, tile).any(-1)
    live[~live.any(-1)] = True
    return live.astype(np.uint8)


def segment_tables(live):
    """live uint8 [S, nb] -> (keep [S, nb], tile_off int32 [S * nb], tile_src int32 [S * nb], count_rows).  keep: tiles
    0 .. last live tile of the segment (all nb when none is live).  tile_off: index of a kept tile in the packed order, -1 for
    a dropped one; tile_src: its inverse, -1 past the end; count_rows = 64 x #kept."""
    live = np.asarray(live).astype(bool)
    S, nb = live.shape
    keep = np.zeros((S, nb), dtype=np.uint8)
    for s in range(S):
        nz = np.flatnonzero(live[s])
        f = int(nz.max()) + 1 if len(nz) else nb
        keep[s, :f] = 1
    flat = keep.reshape(-1).astype(bool)
    off = np.where(flat, np.cumsum(flat) - 1, -1).astype(np.int32)
    src = np.full(S * nb, -1, dtype=np.int32)
    src[: int(flat.sum())] = np.flatnonzero(flat).astype(np.int32)
    return keep, off, src, TILE * int(flat.sum())
