"""Generate `tests/golden/mips_*.npz` by running the UNMODIFIED reference index
(`/root/reference/src/index.py`, `DistributedIndex`) on seeded synthetic inputs.

Run in the build container only (`python oracle/make_golden.py`); `/root/reference` is not
present on the GPU box.  The fixtures hold OUTPUTS only (plus a sha256 of the inputs, which are
regenerated from `oracle/synth.py` by whoever replays them).

For every case we record
  ref_scores   [nq,k] fp16  - values returned by the reference `search_knn` (src/index.py:154-155)
  ref_ids      [nq,k] int64 - the reference's own pick (global line numbers read back from the
                              returned passage dicts); tie order is torch.topk's, i.e. unspecified
  canon_ids    [nq,k] int64 - canonical pick: reference fp16 score matrix
                              (`torch.matmul(q.half(), E)`, src/index.py:117) + stable sort by
                              (score desc, global id asc)           
Multi-rank cases run the reference under a real `torch.distributed` gloo group on CPU
(`Tensor.cuda` patched to a no-op: the reference hard-codes `.cuda()` at src/index.py:35).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import synth  # noqa: E402
import mips_oracle  # noqa: E402

GOLDEN_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")

# name, n, nq per rank, k, dist, bank seed, query seed
CASES = [
    ("c1_grid", 10000, [64], 40, "grid", 1234, 4321),      # BASELINE.json configs[0]
    ("c1_gauss", 10000, [64], 40, "gauss", 1234, 4321),
    ("c1_grid_k80", 10000, [64], 80, "grid", 1234, 4321),  # filtering_overretrieve_ratio=2 (atlas.py:112)
    ("ragged_k5", 257, [3], 5, "grid", 7, 8),
    ("k_equals_n", 40, [2], 40, "grid", 9, 10),
    ("w2_grid", 1003, [3, 5], 7, "grid", 11, 12),
    ("w4_grid_empty_rank", 2050, [3, 0, 5, 2], 40, "grid", 13, 14),  # a rank with 0 queries
    ("w4_gauss", 2050, [4, 4, 4, 4], 40, "gauss", 15, 16),
]


def _split_queries(q, sizes):
    off = np.cumsum([0] + list(sizes))
    return [q[off[i]:off[i + 1]] for i in range(len(sizes))]


def _run_rank(rank, world, case, port, ret):
    import torch
    import ref_shims

    ref_shims.install()
    name, n, nq_per_rank, k, dist, bseed, qseed = case
    torch.set_num_threads(2)
    torch.Tensor.cuda = lambda self, *a, **kw: self  # CPU box; reference hard-codes .cuda()
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        torch.distributed.init_process_group("gloo", rank=rank, world_size=world)
    from src.index import DistributedIndex

    bank = synth.make_bank(n, seed=bseed, dist=dist)
    queries = _split_queries(synth.make_queries(sum(nq_per_rank), seed=qseed, dist=dist), nq_per_rank)
    rows = mips_oracle.shard_rows(n, rank, world)
    index = DistributedIndex()
    index.is_in_gpu = False
    index.init_embeddings(synth.make_passages(n, rank, world))
    index.embeddings[:] = torch.from_numpy(bank[rows]).T  # reference layout [768, n_local]
    q = torch.from_numpy(queries[rank])
    docs, scores = index.search_knn(q, k)
    ids = np.array([[int(d["id"]) for d in row] for row in docs], dtype=np.int64).reshape(len(docs), k)
    vals = np.array(scores, dtype=np.float32).reshape(len(docs), k).astype(np.float16)
    # the reference's own fp16 score matrix for this rank's queries against the FULL bank
    full = torch.matmul(q.half(), torch.from_numpy(bank).T).numpy()
    ret[rank] = (vals, ids, full)
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


def main():
    import torch.multiprocessing as mp

    os.makedirs(GOLDEN_DIR, exist_ok=True)
    port = 29650
    for case in CASES:
        name, n, nq_per_rank, k, dist, bseed, qseed = case
        world = len(nq_per_rank)
        mgr = mp.Manager()
        ret = mgr.dict()
        if world == 1:
            _run_rank(0, 1, case, port, ret)
        else:
            port += 1
            mp.spawn(_run_rank, args=(world, case, port, ret), nprocs=world, join=True)
        bank = synth.make_bank(n, seed=bseed, dist=dist)
        q = synth.make_queries(sum(nq_per_rank), seed=qseed, dist=dist)
        ref_scores = np.concatenate([ret[r][0] for r in range(world)])
        ref_ids = np.concatenate([ret[r][1] for r in range(world)])
        full = np.concatenate([ret[r][2] for r in range(world)])
        canon_v, canon_i = mips_oracle.canonical_topk(full, k)
        # sanity: reference values are the canonical values (tie-independent), and the numpy
        # restatement reproduces the reference matrix bit-for-bit on the exact grid
        assert np.array_equal(ref_scores.view(np.uint16), canon_v.view(np.uint16)), name
        mine = mips_oracle.scores_fp16(q, bank)
        n_diff = int((mine.view(np.uint16) != full.view(np.uint16)).sum())
        if dist == "grid":
            assert n_diff == 0, (name, n_diff)
        np.savez_compressed(
            os.path.join(GOLDEN_DIR, f"mips_{name}.npz"),
            n=n, nq_per_rank=np.array(nq_per_rank), k=k, dist=dist, bank_seed=bseed, query_seed=qseed,
            inputs_sha256=synth.sha256(bank, q),
            ref_scores=ref_scores, ref_ids=ref_ids, canon_ids=canon_i,
            oracle_matrix_mismatches=n_diff,
        )
        agree = float((ref_ids == canon_i).mean())
        print(f"{name}: n={n} nq={nq_per_rank} k={k} dist={dist} world={world} "
              f"ref==canonical ids {agree:.3f}; numpy-vs-reference matrix mismatches {n_diff}")


if __name__ == "__main__":
    main()
