"""CPU checks of the exact re-ranking of product-quantized candidates (`DistributedFAISSIndex(refine_factor > 1)`):
oracle/pq_refine_oracle.py on hand-written cases with answers known by construction, and the HOST logic of the refined
search (candidate count, ids, the refine_factor = 1 path, the distributed merge over gloo, index files, Atlas's option)
with the candidate search and the refine kernel replaced by the oracles in this test only."""
import os
import sys
import tempfile
import types

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from conftest import ROOT

import mips_oracle
import pq_oracle
import pq_refine_oracle

DIM = 768


# ----------------------------------------------------------------------------------------------- oracle hand cases
def _rows(*pairs, n=None):
    """fp16 rows [n, 768] with row r = sum of v * e_d over its (d, v) pairs."""
    rows = np.zeros((n or len(pairs), DIM), np.float16)
    for r, pr in enumerate(pairs):
        for d, v in pr:
            rows[r, d] = v
    return rows


def test_refine_known_sums_and_global_ids():
    rows = _rows([(0, 1), (1, 2)], [(0, 3)], [(1, -1), (5, 4)], [(0, 0.5), (1, 0.5)])
    q = np.zeros((1, DIM), np.float32)
    q[0, :2] = [2, 1]                                  # scores: 4, 6, -1, 1.5
    v, i = pq_refine_oracle.refine_topk(q, rows, np.array([[0, 1, 2, 3]]), 3, id_base=7, id_stride=10)
    assert v.dtype == np.float16 and i.dtype == np.int64
    assert v.tolist() == [[6, 4, 1.5]]
    assert i.tolist() == [[17, 7, 37]]
    # only the candidates are scored: row 1 (the best) is not among them
    v, i = pq_refine_oracle.refine_topk(q, rows, np.array([[3, 2, 0]]), 2)
    assert v.tolist() == [[4, 1.5]] and i.tolist() == [[0, 3]]


def test_refine_rounds_once_to_fp16():
    # 2048 + 1 + 1 = 2050 exactly in fp32; rounding each partial sum to fp16 (ulp 2 above 2048) would give 2048
    rows = _rows([(0, 2048), (1, 1), (2, 1)])
    q = np.zeros((1, DIM), np.float32)
    q[0, :3] = 1
    v, _ = pq_refine_oracle.refine_topk(q, rows, np.array([[0]]), 1)
    assert float(v[0, 0]) == 2050.0
    # the query is rounded to fp16 first: 1 + 2^-12 -> 1
    q[0, 0] = 1 + 2 ** -12
    v, _ = pq_refine_oracle.refine_topk(q, _rows([(0, 1)]), np.array([[0]]), 1)
    assert float(v[0, 0]) == 1.0


def test_refine_ties_resolved_by_global_id():
    rows = _rows([(0, 1)], [(0, 2)], [(0, 1)], [(0, 2)], [(0, 1)])
    q = np.zeros((1, DIM), np.float32)
    q[0, 0] = 1
    v, i = pq_refine_oracle.refine_topk(q, rows, np.array([[4, 2, 3, 0, 1]]), 4, id_base=1, id_stride=2)
    assert v.tolist() == [[2, 2, 1, 1]]
    assert i.tolist() == [[3, 7, 1, 5]]              # rows 1, 3 then rows 0, 2 (global 1 + 2 * row)


def test_refine_skips_invalid_candidates():
    rows = _rows([(0, 1)], [(0, 2)])
    q = np.zeros((1, DIM), np.float32)
    q[0, 0] = 1
    v, i = pq_refine_oracle.refine_topk(q, rows, np.array([[-1, 1, 5]]), 3)
    assert i.tolist() == [[1, -1, -1]]
    assert float(v[0, 0]) == 2 and np.isneginf(v[0, 1:].astype(np.float32)).all()


def test_refine_over_every_row_is_the_flat_topk():
    rng = np.random.default_rng(3)
    rows = (rng.standard_normal((500, DIM)) / 16).astype(np.float16)
    q = (rng.standard_normal((6, DIM)) / 16).astype(np.float16)
    cand = np.stack([rng.permutation(500) for _ in range(6)])
    v, i = pq_refine_oracle.refine_topk(q, rows, cand, 40)
    want_v, want_i = mips_oracle.canonical_topk(mips_oracle.scores_fp16(q, rows), 40)
    assert np.array_equal(v.view(np.uint16), want_v.view(np.uint16))
    assert np.array_equal(i, want_i)


# ----------------------------------------------------------------------------------------------- module host logic
N_ROWS, M_TEST, K_TEST, R_TEST = 1200, 8, 10, 4


def _make_cpu_refine_class():
    from atlas_b200.index import DistributedFAISSIndex

    class OracleRefineIndex(DistributedFAISSIndex):
        """Host logic of the product class; training, encoding, the candidate search and the refine step swapped for
        the oracles (test only).  Records every candidate search and refine call."""
        trainings = 0

        @staticmethod
        def _device():
            return torch.device("cpu")

        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.calls = []

        def _train_and_encode(self, rows, n):
            type(self).trainings += 1
            x = rows.float().numpy()
            cb, coarse = pq_oracle.train(x, self.code_size, self.n_list(n), iters=3, seed=self._id_base)
            codes, lists = pq_oracle.encode(x, cb, coarse)
            t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a))
            return dict(codebooks=t(cb), coarse=t(coarse), codes=t(codes), list_ids=t(lists), n_list=self.n_list(n))

        def _candidate_search(self, allqueries, k, id_base, id_stride, exhaustive):
            self.calls.append(("search", k, id_base, id_stride, exhaustive))
            v, local = _pq_topk(self._trained(), allqueries.float().numpy(), k)
            return torch.from_numpy(v), torch.from_numpy(id_base + id_stride * local), torch.zeros(1, dtype=torch.int32)

        def _refine(self, allqueries, cand_local, topk):
            self.calls.append(("refine", tuple(cand_local.shape), topk))
            v, i = pq_refine_oracle.refine_topk(allqueries.float().numpy(), self._bank.numpy(), cand_local.numpy(), topk,
                                                self._id_base, self._id_stride)
            return torch.from_numpy(v), torch.from_numpy(i)

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

    return OracleRefineIndex


def _pq_topk(p, q, k):
    s = pq_oracle.adc_scores(q, p["codes"].numpy(), p["codebooks"].numpy(),
                             None if p["coarse"] is None else p["coarse"].numpy(),
                             None if p["list_ids"] is None else p["list_ids"].numpy())
    return mips_oracle.canonical_topk(s, k)


def _single(kind="ivfpq", n=N_ROWS, seed=5, refine_factor=R_TEST):
    import synth

    Index = _make_cpu_refine_class()
    index = Index(kind, M_TEST, refine_factor=refine_factor)
    index.init_embeddings(synth.make_passages(n))
    rng = np.random.default_rng(seed)
    index.embeddings[:, :] = torch.from_numpy((rng.standard_normal((n, DIM)) / 16).astype(np.float16)).T
    index.train_index()
    return Index, index


def _queries(nq, seed=9):
    return torch.from_numpy((np.random.default_rng(seed).standard_normal((nq, DIM)) / 16).astype(np.float16))


def test_constructor_keyword_attribute_and_positional_form():
    from atlas_b200._lib import AtlasB200Error

    Index = _make_cpu_refine_class()
    assert Index("ivfpq", 16).refine_factor == 1                  # src/index_io.py's two positional arguments
    assert Index("pq", 16, refine_factor=3).refine_factor == 3
    for bad in (0, -2, 1.5, True):
        with pytest.raises(AtlasB200Error, match="refine_factor"):
            Index("pq", 16, refine_factor=bad)
    _, index = _single(refine_factor=1)
    index.refine_factor = 0                                       # set after construction: checked at search time
    with pytest.raises(AtlasB200Error, match="refine_factor"):
        index.search_knn(_queries(2), K_TEST)


def test_refine_factor_one_is_the_plain_candidate_search():
    _, index = _single(refine_factor=1)
    index._id_base, index._id_stride = 2, 5
    q = _queries(3)
    s, i = index.search_device(q, K_TEST)
    assert index.calls == [("search", K_TEST, 2, 5, False)]
    v, local = _pq_topk(index._pq, q.float().numpy(), K_TEST)
    assert np.array_equal(s.numpy().view(np.uint16), v.view(np.uint16))
    assert np.array_equal(i.numpy(), 2 + 5 * local)


def test_refined_search_candidates_ids_and_scores():
    _, index = _single()
    index._id_base, index._id_stride = 1, 3                       # local row l -> global id 1 + 3 l
    q = _queries(5)
    s, i = index.search_device(q, K_TEST)
    k_cand = K_TEST * R_TEST
    assert index.calls == [("search", k_cand, 0, 1, False), ("refine", (5, k_cand), K_TEST)]
    _, cand = _pq_topk(index._pq, q.float().numpy(), k_cand)
    want_v, want_i = pq_refine_oracle.refine_topk(q.numpy(), index._bank.numpy(), cand, K_TEST, 1, 3)
    assert np.array_equal(s.numpy().view(np.uint16), want_v.view(np.uint16))
    assert np.array_equal(i.numpy(), want_i)
    assert ((i.numpy() - 1) % 3 == 0).all()
    # the scores are exact inner products of the returned rows, not PQ scores
    exact = mips_oracle.scores_fp16(q.numpy(), index._bank.numpy())
    assert np.array_equal(np.take_along_axis(exact, (i.numpy() - 1) // 3, 1).view(np.uint16), s.numpy().view(np.uint16))


def test_candidate_count_is_clamped_to_the_local_rows():
    _, index = _single(kind="pq", n=300, refine_factor=50)         # 10 x 50 = 500 > 300 rows
    q = _queries(2)
    s, i = index.search_device(q, K_TEST)
    assert index.calls[0] == ("search", 300, 0, 1, False) and index.calls[1] == ("refine", (2, 300), K_TEST)
    # every row is a candidate: the result is the exact flat top-k
    want_v, want_i = mips_oracle.canonical_topk(mips_oracle.scores_fp16(q.numpy(), index._bank.numpy()), K_TEST)
    assert np.array_equal(s.numpy().view(np.uint16), want_v.view(np.uint16)) and np.array_equal(i.numpy(), want_i)


def test_too_many_candidates_raise_naming_the_factor_and_topk():
    from atlas_b200._lib import MAX_TOPK, AtlasB200Error

    _, index = _single(refine_factor=MAX_TOPK // K_TEST + 1)      # 1030 candidates of 1200 rows
    with pytest.raises(AtlasB200Error, match=r"refine_factor=103.*topk=10"):
        index.search_device(_queries(2), K_TEST)
    assert index.calls == []
    index.refine_factor = MAX_TOPK // K_TEST                      # 1020 candidates: fine
    index.search_device(_queries(2), K_TEST)
    assert index.calls[0][1] == 1020


def test_exhaustive_retry_refines_too():
    _, index = _single()
    index.search_device(_queries(2), K_TEST, exhaustive=True)
    assert index.calls == [("search", K_TEST * R_TEST, 0, 1, True), ("refine", (2, K_TEST * R_TEST), K_TEST)]


def test_loaded_index_refines_like_the_saved_one():
    Index, index = _single()
    q = _queries(4)
    docs, scores = index.search_knn(q, K_TEST)
    with tempfile.TemporaryDirectory() as tmp:
        index.save_index(tmp, 1)
        saved = sorted(os.listdir(tmp))
        before = Index.trainings
        index2 = Index("ivfpq", M_TEST)
        index2.load_index(tmp, 1)
        assert Index.trainings == before and saved == sorted(os.listdir(tmp))
        index2.refine_factor = R_TEST
        docs2, scores2 = index2.search_knn(q, K_TEST)
    assert scores2 == scores and docs2 == docs
    index._reset_store()
    index2._reset_store()


# ----------------------------------------------------------------------------------------------- gloo
def _bank_and_queries(world):
    rng = np.random.default_rng(15)
    bank = (rng.standard_normal((N_ROWS, DIM)) / 16).astype(np.float16)
    nq = [3] * world
    nq[-1] += 1
    if world > 2:
        nq[1] = 0                                  # one rank without queries
    q = (rng.standard_normal((sum(nq), DIM)) / 16).astype(np.float16)
    return bank, q, nq


def _expected(kind, bank, q, world):
    """Per shard: the PQ top-k' candidates, refined by the oracle; then the canonical merge of the shards' lists."""
    cls = _make_cpu_refine_class()
    per_shard = []
    for r in range(world):
        rows = mips_oracle.shard_rows(N_ROWS, r, world)
        idx = cls(kind, M_TEST)
        idx._id_base, idx._id_stride = r, world
        p = idx._train_and_encode(torch.from_numpy(bank[rows]), len(rows))
        _, cand = _pq_topk(p, q, K_TEST * R_TEST)
        per_shard.append(pq_refine_oracle.refine_topk(q, bank[rows], cand, K_TEST, r, world))
    cat_v = np.concatenate([v for v, _ in per_shard], 1)
    cat_i = np.concatenate([i for _, i in per_shard], 1)
    out_v, out_i = [], []
    for row in range(len(q)):
        order = np.lexsort((cat_i[row], -(cat_v[row].astype(np.float32) + 0.0)))[:K_TEST]
        out_v.append(cat_v[row, order])
        out_i.append(cat_i[row, order])
    return np.array(out_v), np.array(out_i)


def _worker(rank, world, kind, port):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import synth

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      ATLAS_B200_PASSAGE_STORE="shm")
    torch.distributed.init_process_group("gloo", rank=rank, world_size=world)
    try:
        bank, q, nq = _bank_and_queries(world)
        off = np.cumsum([0] + nq)
        want_v, want_i = _expected(kind, bank, q, world)
        index = _make_cpu_refine_class()(kind, M_TEST, refine_factor=R_TEST)
        index.init_embeddings(synth.make_passages(N_ROWS, rank, world))
        rows = mips_oracle.shard_rows(N_ROWS, rank, world)
        index.embeddings[:, : len(rows)] = torch.from_numpy(bank[rows]).T
        index.train_index()
        docs, scores = index.search_knn(torch.from_numpy(q[off[rank]:off[rank + 1]]), K_TEST)
        got_i = np.array([[int(d["id"]) for d in row] for row in docs], np.int64).reshape(-1, K_TEST)
        got_v = np.array(scores, np.float32).reshape(-1, K_TEST).astype(np.float16)
        assert np.array_equal(got_i, want_i[off[rank]:off[rank + 1]])
        assert np.array_equal(got_v.view(np.uint16), want_v[off[rank]:off[rank + 1]].view(np.uint16))
        # every rank refined all gathered queries, its own and the others'
        assert index.calls[-1] == ("refine", (sum(nq), K_TEST * R_TEST), K_TEST)
        index._reset_store()
    finally:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


@pytest.mark.parametrize("kind,world", [("pq", 2), ("ivfpq", 4)])
def test_refined_search_gloo(kind, world):
    port = 29830 + world + (5 if kind == "ivfpq" else 0)
    mp.spawn(_worker, args=(world, kind, port), nprocs=world, join=True)


# ----------------------------------------------------------------------------------------------- Atlas option
def test_atlas_retrieve_sets_the_refine_factor_from_opt():
    from atlas_b200.atlas import Atlas

    class Retriever:
        def eval(self):
            return self

        def __call__(self, ids, mask, is_passages=False):
            return torch.zeros(len(ids), DIM)

    class Index:
        def search_knn(self, q, k):
            self.seen = getattr(self, "refine_factor", None)
            return [[{}] * k for _ in range(len(q))], [[0.0] * k for _ in range(len(q))]

    def run(index, **opt):
        model = types.SimpleNamespace(retriever=Retriever(), training=False, opt=types.SimpleNamespace(**opt))
        Atlas._retrieve(model, index, 2, ["a", "b"], [[1], [2]], None)
        return index

    faiss_like = Index()
    faiss_like.refine_factor = 1
    assert run(faiss_like, faiss_refine_factor=4).seen == 4
    assert run(faiss_like).seen == 4                               # an options object without the field: untouched
    assert run(faiss_like, faiss_refine_factor=None).seen == 4
    flat_like = run(Index(), faiss_refine_factor=4)                 # the flat index has no such attribute: ignored
    assert flat_like.seen is None and not hasattr(flat_like, "refine_factor")
