"""CPU checks of the product-quantized index: oracle/pq_oracle.py on hand-written cases with answers known by construction,
and the HOST logic of `atlas_b200.index.DistributedFAISSIndex` (constructor, training state, query exchange, merge,
passage lookup, index files) over gloo with the device kernels replaced by the oracle in this test only."""
import os
import shutil
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from conftest import ROOT

import pq_oracle


# ----------------------------------------------------------------------------------------------- oracle hand cases
def _axis_codebooks(M, dsub):
    """cb[m][j] = j * e_0 of the sub-space: <q_m, cb[m][j]> = j * q[m * dsub]."""
    cb = np.zeros((M, 256, dsub), np.float32)
    cb[:, :, 0] = np.arange(256, dtype=np.float32)[None, :]
    return cb


def test_adc_scores_known_sums():
    cb = _axis_codebooks(2, 2)
    q = np.array([[1, 0, 1, 0], [2, 0, -1, 0]], np.float32)
    codes = np.array([[3, 5], [255, 0], [0, 0]], np.uint8)
    s = pq_oracle.adc_scores(q, codes, cb)
    assert s.dtype == np.float16
    assert s.tolist() == [[8, 255, 0], [6 - 5, 510, 0]]


def test_adc_scores_round_once_to_fp16():
    # 2048 + 1 + 1 = 2050 exactly in fp32; rounding every partial sum to fp16 (ulp 2 above 2048) would give 2048 + 1
    # -> 2048 (tie to even), + 1 -> 2048.
    cb = np.zeros((3, 256, 8), np.float32)
    cb[0, 1, 0], cb[1, 1, 0], cb[2, 1, 0] = 2048, 1, 1
    q = np.zeros((1, 24), np.float32)
    q[0, [0, 8, 16]] = 1
    s = pq_oracle.adc_scores(q, np.ones((1, 3), np.uint8), cb)
    assert float(s[0, 0]) == 2050.0


def test_adc_scores_ivf_adds_the_rows_own_list():
    cb = _axis_codebooks(2, 2)
    coarse = np.array([[0, 0, 0, 0], [10, 0, 0, 0], [0, 0, 100, 0]], np.float32)
    q = np.array([[1, 0, 1, 0]], np.float32)
    codes = np.array([[1, 1], [1, 1], [1, 1]], np.uint8)
    s = pq_oracle.adc_scores(q, codes, cb, coarse, np.array([0, 1, 2]))
    assert s.tolist() == [[2, 12, 102]]


def test_queries_are_rounded_to_fp16_first():
    cb = _axis_codebooks(1, 8)
    q = np.zeros((1, 8), np.float32)
    q[0, 0] = 1 + 2 ** -12                      # rounds to 1.0 in fp16
    assert pq_oracle.lut(q, cb)[0, 0, 3] == 3.0


def test_encode_nearest_and_lowest_index_on_ties():
    cb = np.zeros((2, 256, 2), np.float32)
    cb[0, :, 0] = np.arange(256)                 # sub-space 0: points (j, 0)
    cb[1, :, 1] = np.arange(256) % 128           # sub-space 1: j and j + 128 coincide -> the lower one wins
    x = np.array([[3.2, 0, 0, 7.0], [254.6, 0, 0, 127.9]], np.float32)
    codes, lists = pq_oracle.encode(x, cb)
    assert lists is None
    assert codes.tolist() == [[3, 7], [255, 127]]


def test_encode_ivf_residual_and_ip_assignment():
    cb = np.zeros((1, 256, 8), np.float32)
    cb[0, :, 0] = np.arange(256) - 128.0
    coarse = np.zeros((2, 8), np.float32)
    coarse[0, 1], coarse[1, 0] = 1.0, 100.0      # IP picks list 1 for x[0] > 0.01 x[1]
    x = np.zeros((2, 8), np.float32)
    x[0, 0], x[1, 1] = 103.0, 5.0
    codes, lists = pq_oracle.encode(x, cb, coarse)
    assert lists.tolist() == [1, 0]
    assert codes[:, 0].tolist() == [3 + 128, 128]   # residual 3 -> centroid 3; residual 0 in dim 0 -> centroid 0


def test_kmeans_recovers_separated_clusters():
    rng = np.random.default_rng(0)
    centers = np.array([[0, 0], [10, 0], [0, 10], [10, 10]], np.float32)
    x = np.concatenate([c + 0.1 * rng.standard_normal((50, 2)) for c in centers]).astype(np.float32)
    c = pq_oracle.kmeans(x, 4, iters=10, init=[0, 50, 100, 150])     # one seed per cluster: the means are the answer
    got = sorted(map(tuple, np.round(c).astype(int).tolist()))
    assert got == [(0, 0), (0, 10), (10, 0), (10, 10)]


def test_canonical_topk_is_the_flat_rule():
    import mips_oracle

    assert pq_oracle.canonical_topk is mips_oracle.canonical_topk


# ----------------------------------------------------------------------------------------------- module host logic
N_ROWS, M_TEST, K_TEST = 1200, 8, 10


def _make_cpu_faiss_class():
    import mips_oracle
    from atlas_b200.index import DistributedFAISSIndex

    class OracleBackedFAISSIndex(DistributedFAISSIndex):
        """Host logic of the product class; training, encoding and the code scan swapped for the oracle (test only)."""
        trainings = 0

        @staticmethod
        def _device():
            return torch.device("cpu")

        def _train_and_encode(self, rows, n):
            type(self).trainings += 1
            x = rows.float().numpy()
            cb, coarse = pq_oracle.train(x, self.code_size, self.n_list(n), iters=3, seed=self._id_base)
            codes, lists = pq_oracle.encode(x, cb, coarse)
            t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a))
            return dict(codebooks=t(cb), coarse=t(coarse), codes=t(codes), list_ids=t(lists), n_list=self.n_list(n))

        def _local_search(self, allqueries, topk, exhaustive=False):
            p = self._trained()
            s = pq_oracle.adc_scores(allqueries.float().numpy(), p["codes"].numpy(), p["codebooks"].numpy(),
                                     None if p["coarse"] is None else p["coarse"].numpy(),
                                     None if p["list_ids"] is None else p["list_ids"].numpy())
            v, local = mips_oracle.canonical_topk(s, topk)
            return (torch.from_numpy(v), torch.from_numpy(self._id_base + self._id_stride * local),
                    torch.zeros(1, dtype=torch.int32))

        def _merge(self, blob_all, ids_off, world, nq_total, topk, q_begin, nq_out):
            nb = nq_total * topk
            vs = torch.stack([blob_all[w, : nb * 2].view(torch.float16).view(nq_total, topk) for w in range(world)])
            ids = torch.stack([blob_all[w, ids_off:ids_off + nb * 8].view(torch.int64).view(nq_total, topk)
                               for w in range(world)])
            out_v = np.empty((nq_out, topk), np.float16)
            out_i = np.empty((nq_out, topk), np.int64)
            for j in range(nq_out):
                cv = vs[:, q_begin + j].reshape(-1).numpy()
                ci = ids[:, q_begin + j].reshape(-1).numpy()
                order = np.lexsort((ci, -(cv.astype(np.float32) + 0.0)))[:topk]
                out_v[j], out_i[j] = cv[order], ci[order]
            return torch.from_numpy(out_v), torch.from_numpy(out_i)

    return OracleBackedFAISSIndex


def _bank_and_queries(world):
    rng = np.random.default_rng(5)
    bank = (rng.standard_normal((N_ROWS, 768)) / 16).astype(np.float16)
    q = (rng.standard_normal((3 * world + 1, 768)) / 16).astype(np.float16)
    nq = [3] * world
    nq[-1] += 1
    nq[0] = 0 if world > 2 else nq[0]              # one rank without queries
    return bank, q[: sum(nq)], nq


def _expected(kind, bank, q, nq, world):
    """The oracle's merge of the per-shard lists (each shard trained on its own rows, like the ranks)."""
    import mips_oracle

    cls = _make_cpu_faiss_class()
    per_shard = []
    for r in range(world):
        rows = mips_oracle.shard_rows(N_ROWS, r, world)
        idx = cls(kind, M_TEST)
        idx._id_base, idx._id_stride = r, world
        p = idx._train_and_encode(torch.from_numpy(bank[rows]), len(rows))
        s = pq_oracle.adc_scores(q, p["codes"].numpy(), p["codebooks"].numpy(),
                                 None if p["coarse"] is None else p["coarse"].numpy(),
                                 None if p["list_ids"] is None else p["list_ids"].numpy())
        v, local = mips_oracle.canonical_topk(s, K_TEST)
        per_shard.append((v, rows[local]))
    cat_v = np.concatenate([v for v, _ in per_shard], 1)
    cat_i = np.concatenate([i for _, i in per_shard], 1)
    out_v, out_i = [], []
    for row in range(len(q)):
        order = np.lexsort((cat_i[row], -(cat_v[row].astype(np.float32) + 0.0)))[:K_TEST]
        out_v.append(cat_v[row, order])
        out_i.append(cat_i[row, order])
    return np.array(out_v), np.array(out_i)


def _worker(rank, world, kind, port, tmpdir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mips_oracle
    import synth

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      ATLAS_B200_PASSAGE_STORE="shm")
    torch.distributed.init_process_group("gloo", rank=rank, world_size=world)
    try:
        bank, q, nq = _bank_and_queries(world)
        off = np.cumsum([0] + nq)
        want_v, want_i = _expected(kind, bank, q, nq, world)
        Index = _make_cpu_faiss_class()
        index = Index(kind, M_TEST)
        index.init_embeddings(synth.make_passages(N_ROWS, rank, world))
        rows = mips_oracle.shard_rows(N_ROWS, rank, world)
        index.embeddings[:, : len(rows)] = torch.from_numpy(bank[rows]).T
        assert not index.is_index_trained()
        index.train_index()
        assert index.is_index_trained()
        docs, scores = index.search_knn(torch.from_numpy(q[off[rank]:off[rank + 1]]), K_TEST)
        got_i = np.array([[int(d["id"]) for d in row] for row in docs], np.int64).reshape(-1, K_TEST)
        got_v = np.array(scores, np.float32).reshape(-1, K_TEST).astype(np.float16)
        assert np.array_equal(got_i, want_i[off[rank]:off[rank + 1]])
        assert np.array_equal(got_v.view(np.uint16), want_v[off[rank]:off[rank + 1]].view(np.uint16))
        for row in docs:
            for d in row:
                assert d["title"] == f"t{d['id']}"
        # save -> load with the same world size: no retraining, identical results
        index.save_index(tmpdir, 2 * world)
        torch.distributed.barrier()
        before = Index.trainings
        index2 = Index(kind, M_TEST)
        index2.load_index(tmpdir, 2 * world)
        assert Index.trainings == before and index2.is_index_trained()
        assert torch.equal(index2.embeddings, index.embeddings)
        docs2, scores2 = index2.search_knn(torch.from_numpy(q[off[rank]:off[rank + 1]]), K_TEST)
        assert scores2 == scores
        index._reset_store()
        index2._reset_store()
    finally:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


@pytest.mark.parametrize("kind,world", [("pq", 2), ("ivfpq", 2), ("ivfpq", 4)])
def test_faiss_index_host_logic_gloo(kind, world):
    port = 29790 + world + (5 if kind == "ivfpq" else 0)
    with tempfile.TemporaryDirectory() as tmp:
        mp.spawn(_worker, args=(world, kind, port, tmp), nprocs=world, join=True)


def _single(kind="ivfpq", M=M_TEST, n=N_ROWS, seed=5):
    import synth

    Index = _make_cpu_faiss_class()
    index = Index(kind, M)
    index.init_embeddings(synth.make_passages(n))
    rng = np.random.default_rng(seed)
    index.embeddings[:, :] = torch.from_numpy((rng.standard_normal((n, 768)) / 16).astype(np.float16)).T
    return Index, index


def test_index_file_name_and_round_trip():
    Index, index = _single()
    assert not index.is_index_trained()
    index.train_index()
    with tempfile.TemporaryDirectory() as tmp:
        index.save_index(tmp, 1)
        assert sorted(os.listdir(tmp)) == ["embeddings.0.pt", f"indexivfpq_{M_TEST}_rank_0.atlas_b200.pt", "passages.0.pt"]
        assert torch.load(os.path.join(tmp, "embeddings.0.pt")).shape == (768, N_ROWS)
        before = Index.trainings
        index2 = Index("ivfpq", M_TEST)
        index2.load_index(tmp, 1)
        assert Index.trainings == before
        for key in ("codebooks", "coarse", "codes", "list_ids"):
            assert torch.equal(index2._pq[key], index._pq[key])


def test_load_retrains_on_mismatched_code_size_or_rows():
    Index, index = _single()
    index.train_index()
    _, other = _single(n=N_ROWS - 100)
    with tempfile.TemporaryDirectory() as a, tempfile.TemporaryDirectory() as b:
        index.save_index(a, 1)
        other.save_index(b, 1)          # untrained: shards only
        # row count differs: index file of `index` next to the shards of `other`
        shutil.copy(os.path.join(a, f"indexivfpq_{M_TEST}_rank_0.atlas_b200.pt"), b)
        before = Index.trainings
        loaded = Index("ivfpq", M_TEST)
        loaded.load_index(b, 1)
        assert Index.trainings == before + 1 and loaded._pq["codes"].shape == (N_ROWS - 100, M_TEST)
        # code size differs: the M = 8 file under the M = 16 name
        shutil.copy(os.path.join(a, f"indexivfpq_{M_TEST}_rank_0.atlas_b200.pt"), os.path.join(a, "indexivfpq_16_rank_0.atlas_b200.pt"))
        loaded = Index("ivfpq", 16)
        loaded.load_index(a, 1)
        assert Index.trainings == before + 2 and loaded._pq["codes"].shape == (N_ROWS, 16)


def test_training_state_and_untrained_search():
    from atlas_b200._lib import AtlasB200Error

    _, index = _single("pq")
    with pytest.raises(AtlasB200Error):
        index.search_knn(torch.zeros(2, 768), 3)
    index.train_index()
    assert index.is_index_trained()
    index.embeddings = index.embeddings.clone()     # new rows: stale again
    assert not index.is_index_trained()
    _, small = _single("pq", n=255)
    with pytest.raises(AtlasB200Error):
        small.train_index()


def test_constructor_errors():
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.index import DistributedFAISSIndex

    for kind in ("flat", "ivfflat", "ivfsq"):
        with pytest.raises(AtlasB200Error, match="--index_mode flat"):
            DistributedFAISSIndex(kind, 16)
    with pytest.raises(AtlasB200Error, match="code_size"):
        DistributedFAISSIndex("pq", None)
    for bad in (0, 5, 128, 192, 768):
        with pytest.raises(AtlasB200Error, match="not supported"):
            DistributedFAISSIndex("ivfpq", bad)
    if not torch.cuda.is_available():
        with pytest.raises(AtlasB200Error):
            DistributedFAISSIndex("pq", 16)
