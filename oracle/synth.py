"""Seeded synthetic inputs shared by the oracle, the golden generator, the tests and bench.py.

TEST/BENCH INFRASTRUCTURE (numpy only, no reference code).  Everything is generated with
`numpy.random.default_rng` (PCG64, stream-stable across numpy versions) so the container
that writes `tests/golden/` and the GPU box that replays them build bit-identical inputs;
each fixture also stores a sha256 of the generated arrays.

Distributions:
  * "grid"  : clamp(round(8*N(0,1))/8, -4, 4).  Every product is a multiple of 2^-6 and every
              partial sum of 768 products fits in 18 bits, so fp32 accumulation is exact in ANY
              order -> the fp16-rounded score matrix is identical on CPU BLAS, cuBLAS and
              wgmma.  This is the bit-exact gate.
  * "gauss" : N(0,1)/sqrt(768)-scaled passages and unit-scale queries ("realistic"); scores may
              differ by 1 fp16 ulp between accumulation orders -> tolerance gate, tie-aware ids.
"""
import hashlib

import numpy as np

EMBEDDINGS_DIM = 768  # reference: src/retrievers.py:13


def _grid(rng, shape):
    x = rng.standard_normal(shape, dtype=np.float32)
    return np.clip(np.round(x * 8.0) / 8.0, -4.0, 4.0).astype(np.float16)


def _gauss(rng, shape, scale):
    return (rng.standard_normal(shape, dtype=np.float32) * scale).astype(np.float16)


def make_bank(n, dim=EMBEDDINGS_DIM, seed=1234, dist="grid", chunk=1 << 16):
    """Passage bank, row-major [n, dim] fp16 (row = passage).  The reference's logical layout is
    the transpose, `[dim, n]` (src/index.py:51)."""
    rng = np.random.default_rng(seed)
    out = np.empty((n, dim), dtype=np.float16)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        if dist == "grid":
            out[s:e] = _grid(rng, (e - s, dim))
        elif dist == "gauss":
            out[s:e] = _gauss(rng, (e - s, dim), 1.0 / np.sqrt(dim))
        else:
            raise ValueError(dist)
    return out


def make_queries(nq, dim=EMBEDDINGS_DIM, seed=4321, dist="grid"):
    """Query embeddings [nq, dim] float32 (the reference's live retriever emits fp32; search_knn
    casts with `.half()`, src/index.py:117).  Values are chosen fp16-representable for "grid"."""
    rng = np.random.default_rng(seed)
    if dist == "grid":
        return _grid(rng, (nq, dim)).astype(np.float32)
    if dist == "gauss":
        return rng.standard_normal((nq, dim), dtype=np.float32)
    raise ValueError(dist)


def make_passages(n, rank=0, world_size=1):
    """Synthetic passage dicts for the shard held by `rank` under the reference's round-robin
    rule `line % world_size == rank` (src/index_io.py:41).  Local index l <-> global line
    g = l*world_size + rank."""
    return [
        {"id": str(g), "title": f"t{g}", "text": f"passage {g}"}
        for g in range(rank, n, world_size)
    ]


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()
