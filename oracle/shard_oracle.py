"""numpy statement of the sharded optimizer's layout (atlas_b200/sharded.py): the flat buffer, its partition over W ranks,
the per-rank segments (a parameter intersected with a shard) and the consolidation of per-rank state into the
per-parameter state of `AdamWFP32Copy`.

  * Flat buffer: the parameters in optimizer order, back to back, padded with zeros to a multiple of W * ALIGN elements.
  * Shards: rank r owns the contiguous elements [r * S, (r + 1) * S), S = padded / W.
  * Segments: (parameter index, begin, end) in flat-buffer elements, the non-empty intersections of each parameter with
    the rank's shard, in parameter order.  They tile the shard except for the padding at the end of the last shards.
"""
import numpy as np

ALIGN = 64


def partition(numels, world):
    """(offsets [n], padded total, shard size S) for parameters of `numels` elements over `world` ranks."""
    numels = np.asarray(numels, dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(numels)[:-1]]).astype(np.int64) if len(numels) else np.zeros(0, np.int64)
    total = int(numels.sum())
    unit = world * ALIGN
    padded = -(-total // unit) * unit
    return offsets, padded, padded // world


def segments(numels, world, rank):
    """[(parameter index, begin, end)] of rank `rank`, flat-buffer element coordinates."""
    offsets, _, shard = partition(numels, world)
    lo, hi = rank * shard, (rank + 1) * shard
    out = []
    for i, (o, n) in enumerate(zip(offsets.tolist(), np.asarray(numels).tolist())):
        a, b = max(o, lo), min(o + n, hi)
        if a < b:
            out.append((i, a, b))
    return out


def flatten(tensors, world):
    """The padded flat buffer of a list of arrays (one dtype)."""
    numels = [t.size for t in tensors]
    offsets, padded, _ = partition(numels, world)
    flat = np.zeros(padded, dtype=tensors[0].dtype if tensors else np.float32)
    for t, o in zip(tensors, offsets.tolist()):
        flat[o:o + t.size] = t.reshape(-1)
    return flat


def shard(tensors, world):
    """Per-rank shards [W][S] of the flat buffer of `tensors`."""
    flat = flatten(tensors, world)
    s = flat.size // world
    return [flat[r * s:(r + 1) * s].copy() for r in range(world)]


def consolidate(shards, shapes):
    """Per-parameter arrays from the per-rank shards (what `OSS.consolidate_state_dict` gathers)."""
    flat = np.concatenate(shards)
    numels = [int(np.prod(s, dtype=np.int64)) for s in shapes]
    offsets, padded, _ = partition(numels, len(shards))
    assert flat.size == padded, (flat.size, padded)
    return [flat[o:o + n].reshape(s) for o, n, s in zip(offsets.tolist(), numels, shapes)]
