"""GPU checks of the IVF-SQ index (csrc/pq.cu, csrc/ivfsq.cu, DistributedFAISSIndex("ivfsq")) against the numpy
restatement oracle/sq_oracle.py: the register-A wgmma code scan + exact top-k on hand-built states, the slot layout,
training and encoding, the module and Atlas.build_index."""
import os
import tempfile

import numpy as np
import pytest
import torch

import sq_oracle

pytestmark = pytest.mark.gpu

DIM = 768


def _ulp16(v):
    a = np.abs(np.asarray(v, dtype=np.float32)).astype(np.float16)
    return (np.nextafter(a, np.float16(np.inf)) - a).astype(np.float32)


def _state(rng, sizes, scale=0.05, grid=False):
    """A hand-built index: list l holds sizes[l] rows (in random row order), random codes, coarse and ranges."""
    sizes = list(sizes)
    n, n_list = sum(sizes), len(sizes)
    lists = rng.permutation(np.repeat(np.arange(n_list), sizes)).astype(np.int64)
    codes = rng.integers(0, 16, (n, DIM)).astype(np.uint8)
    if grid:
        coarse = rng.integers(-2, 3, (n_list, DIM)).astype(np.float32)
        vmin = rng.integers(-4, 4, DIM).astype(np.float32) / 4
        vdiff = np.full(DIM, 15 / 8, np.float32)                      # vdiff / 15 = 1 / 8
    else:
        coarse = (rng.standard_normal((n_list, DIM)) * scale).astype(np.float32)
        vmin = (-rng.uniform(0.5, 1.5, DIM) * scale).astype(np.float32)
        vdiff = (rng.uniform(1.0, 3.0, DIM) * scale).astype(np.float32)
    return dict(codes=codes, lists=lists, coarse=coarse, vmin=vmin, vdiff=vdiff, n_list=n_list)


def _device(st):
    from atlas_b200 import ops

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    codes, slot_rows, tile_lists = ops.ivfsq_import(t(sq_oracle.pack(st["codes"])), t(st["lists"].astype(np.int32)),
                                                    st["n_list"])
    return dict(codes=codes, slot_rows=slot_rows, tile_lists=tile_lists, coarse=t(st["coarse"]), vmin=t(st["vmin"]),
                vdiff=t(st["vdiff"]), n=len(st["lists"]))


def _search(d, q, k, exhaustive=False, id_base=0, id_stride=1):
    from atlas_b200 import ops

    s, i, stat = ops.ivfsq_topk(d["codes"], d["slot_rows"], d["tile_lists"], d["n"], d["coarse"], d["vmin"], d["vdiff"],
                                torch.from_numpy(q).cuda(), k, id_base, id_stride, exhaustive=exhaustive)
    return s.cpu().numpy(), i.cpu().numpy(), int(stat.item())


def _oracle(st, q):
    return sq_oracle.contract_scores(q, st["codes"], st["vmin"], st["vdiff"], st["coarse"], st["lists"]).astype(np.float32)


def _check_parity(st, q, s, ids, k, all_rows=False):
    """all_rows: k is (about) every row, so the low scores are compared too; their fp32 accumulation error is an
    absolute one, on the scale of the query's largest score, so the tolerance is one fp16 ulp of that score."""
    n = len(st["lists"])
    ref = _oracle(st, q)
    s = s.astype(np.float32)
    assert (ids >= 0).all() and (ids < n).all()
    assert all(len(set(r)) == k for r in ids.tolist())
    got_ref = np.take_along_axis(ref, ids, 1)
    # one ulp of the larger of the two: a value just below a power of two may round up into the next binade
    tol = np.maximum(_ulp16(got_ref), _ulp16(s))
    if all_rows:
        tol = np.maximum(tol, _ulp16(np.abs(ref).max(1, keepdims=True)))
    assert (np.abs(s - got_ref) <= tol).all(), float(np.abs(s - got_ref).max())
    assert (np.diff(s, axis=1) <= 0).all()
    kth = -np.partition(-ref, k - 1, axis=1)[:, k - 1:k]
    tol = 2 * _ulp16(kth)
    assert (got_ref >= kth - tol).all()
    for r in range(len(q)):
        must = np.flatnonzero(ref[r] > kth[r, 0] + tol[r, 0])
        assert np.isin(must, ids[r]).all(), r


SCAN_CASES = [(300, 1, 1), (5000, 8, 40), (20000, 13, 100), (60000, 64, 40), (40000, 130, 7), (100000, 256, 40),
              (30000, 300, 1024)]


@pytest.mark.parametrize("n,nq,k", SCAN_CASES)
def test_scan_parity_given_state(n, nq, k):
    """fp16 scores within 1 ulp of the contract; the top-k holds every row above the oracle's k-th score by more than
    2 ulp and nothing below it by more than 2 ulp."""
    rng = np.random.default_rng(n + nq)
    n_list = max(1, int(np.sqrt(n)))
    st = _state(rng, np.bincount(rng.integers(0, n_list, n), minlength=n_list))
    q = rng.standard_normal((nq, DIM)).astype(np.float16)
    d = _device(st)
    s, ids, stat = _search(d, q, k)
    if stat:
        s, ids, _ = _search(d, q, k, exhaustive=True)
    _check_parity(st, q, s, ids, k)


@pytest.mark.parametrize("nq", [3, 40, 200])
def test_exact_grid_bit_exact(nq):
    """vdiff / 15 a power of two, small-integer coarse terms and sparse small-integer queries: every sum is exact, so
    scores and canonical ids (ties by id) match bitwise."""
    rng = np.random.default_rng(7 + nq)
    n, k = 70000, 64
    st = _state(rng, np.bincount(rng.integers(0, 264, n), minlength=264), grid=True)
    q = np.zeros((nq, DIM), np.float16)
    for r in range(nq):
        q[r, rng.choice(DIM, 6, replace=False)] = rng.integers(-2, 3, 6)
    d = _device(st)
    s, ids, stat = _search(d, q, k)
    if stat:
        s, ids, _ = _search(d, q, k, exhaustive=True)
    want_v, want_i = sq_oracle.canonical_topk(_oracle(st, q).astype(np.float16), k)
    assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16))
    assert np.array_equal(ids, want_i)
    s2, i2, _ = _search(d, q, k, id_base=3, id_stride=5)
    assert np.array_equal(s2.view(np.uint16), want_v.view(np.uint16)) and np.array_equal(i2, 3 + 5 * want_i)


def test_sampled_and_exhaustive_paths_agree():
    rng = np.random.default_rng(11)
    n = 200000
    st = _state(rng, np.bincount(rng.integers(0, 447, n), minlength=447))
    q = rng.standard_normal((100, DIM)).astype(np.float16)
    d = _device(st)
    s1, i1, stat = _search(d, q, 40)
    s2, i2, _ = _search(d, q, 40, exhaustive=True)
    assert stat == 0
    assert np.array_equal(s1.view(np.uint16), s2.view(np.uint16)) and np.array_equal(i1, i2)


def test_all_equal_scores_raise_status_and_exhaustive_returns_first_ids():
    rng = np.random.default_rng(12)
    n, k = 100000, 40
    st = _state(rng, [n // 3, n - n // 3])
    st["coarse"][:] = 0
    st["vdiff"][:] = 0
    q = rng.standard_normal((3, DIM)).astype(np.float16)
    d = _device(st)
    _, _, stat = _search(d, q, k)
    assert stat == 1
    s, ids, _ = _search(d, q, k, exhaustive=True)
    ref = _oracle(st, q)
    assert (s.astype(np.float32) == ref[:, :1]).all() and np.array_equal(ids, np.tile(np.arange(k), (3, 1)))


@pytest.mark.parametrize("sizes", [[0, 1, 63, 64, 65, 0, 200], [5000], [0, 0, 777, 0], [1], [2], [3], [2, 3], [1, 1, 1, 1, 1]])
def test_layout_edges(sizes):
    """Empty lists, lists of 1, 63, 64 and 65 rows, one list holding everything, n of 1, 2, 3 and 5: padding slots are
    never returned and the layout round-trips."""
    from atlas_b200 import ops

    rng = np.random.default_rng(sum(sizes) + len(sizes))
    st = _state(rng, sizes)
    n = len(st["lists"])
    d = _device(st)
    counts = np.array(sizes)
    assert d["codes"].shape[0] == int(((counts + 63) // 64 * 64).sum())
    assert int((d["slot_rows"] >= 0).sum()) == n
    codes, lists = ops.ivfsq_export(d["codes"], d["slot_rows"], d["tile_lists"], n)
    assert np.array_equal(codes.cpu().numpy(), sq_oracle.pack(st["codes"]))
    assert np.array_equal(lists.cpu().numpy(), st["lists"])
    q = rng.standard_normal((9, DIM)).astype(np.float16)
    for k in sorted({1, min(n, 4), min(n, 1024)}):
        for ex in (False, True):
            s, ids, stat = _search(d, q, k, exhaustive=ex)
            assert stat == 0
            _check_parity(st, q, s, ids, k, all_rows=k > 4)


def _clustered(rng, n, centers=64, spread=0.3):
    c = rng.standard_normal((centers, DIM)).astype(np.float32)
    x = c[rng.integers(0, centers, n)] + spread * rng.standard_normal((n, DIM)).astype(np.float32)
    return (x / np.sqrt(DIM)).astype(np.float16)


def _index(x, kind="ivfsq", code_size=None, **kw):
    import synth
    from atlas_b200.index import DistributedFAISSIndex

    index = DistributedFAISSIndex(kind, code_size, **kw)
    index.init_embeddings(synth.make_passages(len(x)))
    index.embeddings[:, :] = torch.from_numpy(x).T
    return index


def _export(index):
    from atlas_b200 import ops

    p = index._pq
    codes, lists = ops.ivfsq_export(p["codes"], p["slot_rows"], p["tile_lists"], int(index._bank.shape[0]))
    return (codes.cpu().numpy(), lists.cpu().numpy().astype(np.int64), p["coarse"].cpu().numpy(), p["vmin"].cpu().numpy(),
            p["vdiff"].cpu().numpy())


@pytest.mark.parametrize("n", [6000, 120000])
def test_encode_and_ranges(n):
    """Given the device's list ids, coarse centroids and ranges, codes are bit-identical to sq_oracle.encode; the list is
    within 2e-3 of the best inner product; vmin / vdiff are numpy's min / max of the sample's fp32 residuals."""
    from atlas_b200.index import DistributedFAISSIndex

    rng = np.random.default_rng(21)
    x = _clustered(rng, n)
    index = _index(x)
    index.train_index()
    codes, lists, coarse, vmin, vdiff = _export(index)
    r = sq_oracle.residuals(x, coarse, lists)
    assert np.array_equal(codes, sq_oracle.encode(r, vmin, vdiff))
    ip = x.astype(np.float32) @ coarse.T
    best = ip.max(1)
    assert (ip[np.arange(n), lists] >= best - 2e-3 * (1 + np.abs(best))).all()
    sample = np.random.default_rng(DistributedFAISSIndex.TRAIN_SEED).permutation(n)[:min(n, 100000)]
    want_min, want_diff = sq_oracle.train_range(r[sample])
    assert np.array_equal(vmin, want_min) and np.array_equal(vdiff, want_diff)


def test_training_is_deterministic_and_works_from_one_row():
    rng = np.random.default_rng(31)
    index = _index(_clustered(rng, 30000))
    index.train_index()
    a = {k: (v.cpu().clone() if torch.is_tensor(v) else v) for k, v in index._pq.items()}
    index.train_index()
    for key in ("coarse", "vmin", "vdiff", "codes", "slot_rows", "tile_lists"):
        assert torch.equal(a[key].view(torch.uint8), index._pq[key].cpu().view(torch.uint8)), key
    for n in (1, 2, 3, 5):
        small = _index(_clustered(rng, n))
        small.train_index()
        docs, _ = small.search_knn(torch.from_numpy(_clustered(rng, 4)).cuda(), n)
        assert all(sorted(int(d["id"]) for d in row) == list(range(n)) for row in docs)


def test_module_search_save_load_memory_and_refine(monkeypatch):
    from atlas_b200 import ops
    from atlas_b200.index import DistributedFAISSIndex

    rng = np.random.default_rng(51)
    n, k = 200000, 40
    x = _clustered(rng, n)
    q = torch.from_numpy(_clustered(rng, 50)).cuda()
    index = _index(x, code_size=4)
    assert not index.is_index_trained() and index.is_in_gpu is False
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    index.train_index()
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    n_list = index.n_list()
    budget = n * (384 + 4) + n_list * 63 * 388 + (n_list + 2) * DIM * 4 + (1 << 20)
    assert grown <= budget, (grown, budget)
    assert grown < n * DIM * 2 // 3

    docs, scores = index.search_knn(q, k)
    p = index._pq
    s, i, _ = ops.ivfsq_topk(p["codes"], p["slot_rows"], p["tile_lists"], n, p["coarse"], p["vmin"], p["vdiff"], q, k)
    assert [[int(d["id"]) for d in row] for row in docs] == i.cpu().tolist()
    assert np.array_equal(np.array(scores, np.float32), s.float().cpu().numpy())

    # refine_factor = 4: the top 4k by SQ score re-ranked by pq_refine_topk
    index.refine_factor = 4
    docs_r, scores_r = index.search_knn(q, k)
    _, cand, _ = ops.ivfsq_topk(p["codes"], p["slot_rows"], p["tile_lists"], n, p["coarse"], p["vmin"], p["vdiff"], q, 4 * k)
    rs, ri = ops.pq_refine_topk(index._bank, q, cand, k)
    assert [[int(d["id"]) for d in row] for row in docs_r] == ri.cpu().tolist()
    assert np.array_equal(np.array(scores_r, np.float32), rs.float().cpu().numpy())
    index.refine_factor = 1

    with tempfile.TemporaryDirectory() as tmp:
        index.save_index(tmp, 1)
        f = os.path.join(tmp, "indexivfsq_4_rank_0.atlas_b200.pt")
        assert os.path.exists(f)
        saved = torch.load(f)
        codes, lists, *_ = _export(index)
        assert np.array_equal(saved["codes"].numpy(), codes) and np.array_equal(saved["list_ids"].numpy(), lists)
        real = monkeypatch.context()
        with real as m:
            m.setattr(ops, "ivfsq_train", lambda *a, **kw: (_ for _ in ()).throw(AssertionError("retrained")))
            index2 = DistributedFAISSIndex("ivfsq", 4)
            index2.load_index(tmp, 1)
            assert index2.is_index_trained() and not index2._bank.is_cuda
            for key in ("codes", "slot_rows", "tile_lists"):
                assert torch.equal(index2._pq[key], index._pq[key]), key
            docs2, scores2 = index2.search_knn(q, k)
            assert scores2 == scores and docs2 == docs
        # a file that does not match (another n_list) is ignored and the index retrained
        saved["n_list"] += 1
        torch.save(saved, f)
        calls = []
        train = ops.ivfsq_train
        monkeypatch.setattr(ops, "ivfsq_train", lambda *a, **kw: calls.append(1) or train(*a, **kw))
        index3 = DistributedFAISSIndex("ivfsq", 4)
        index3.load_index(tmp, 1)
        assert calls == [1] and index3.is_index_trained()
        assert index3.search_knn(q, k) == (docs, scores)


def test_quality_vs_oracle_pipeline_and_ivfpq():
    """Device recall@40 against the exact flat search is at least the oracle pipeline's minus 0.02, and at least 0.25
    above ivfpq with M = 16 on the same rows."""
    import mips_oracle
    import pq_oracle

    rng = np.random.default_rng(41)
    n, k = 8000, 40
    x = _clustered(rng, n)
    q = _clustered(rng, 64)
    _, exact = mips_oracle.canonical_topk(mips_oracle.scores_fp16(q, x), k)
    recall = lambda ids: np.mean([len(set(a) & set(b)) / k for a, b in zip(ids.tolist(), exact.tolist())])

    index = _index(x)
    index.train_index()
    docs, _ = index.search_knn(torch.from_numpy(q).cuda(), k)
    got = recall(np.array([[int(d["id"]) for d in row] for row in docs]))

    coarse = pq_oracle.kmeans(x, index.n_list(), 10, seed=5, inner_product=True)
    lists = sq_oracle.assign_lists(x, coarse)
    r = sq_oracle.residuals(x, coarse, lists)
    vmin, vdiff = sq_oracle.train_range(r)
    codes = sq_oracle.quantize(r, vmin, vdiff)
    _, ref_ids = sq_oracle.canonical_topk(sq_oracle.contract_scores(q, codes, vmin, vdiff, coarse, lists), k)
    assert got >= recall(ref_ids) - 0.02, (got, recall(ref_ids))

    pq_index = _index(x, "ivfpq", 16)
    pq_index.train_index()
    docs, _ = pq_index.search_knn(torch.from_numpy(q).cuda(), k)
    pq_recall = recall(np.array([[int(d["id"]) for d in row] for row in docs]))
    assert got >= pq_recall + 0.25, (got, pq_recall)


def test_build_index_with_host_rows():
    """Atlas.build_index into an ivfsq index: host rows bit-identical to the flat bank of the same build, one training,
    then retrieval end to end."""
    import atlas_synth
    import model_synth
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.index import DistributedFAISSIndex, DistributedIndex
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    dev = torch.device("cuda:0")
    opt = atlas_synth.make_opt()
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    reader = FiD(T5ConfigLite(**{k: v for k, v in model_synth.T5_CFG.items()
                                 if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}))
    reader.load_state_dict(model_synth.fill_state_dict(reader.state_dict(), seed=202)[0])
    contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    contriever.load_state_dict(model_synth.fill_state_dict(contriever.state_dict(), seed=101)[0])
    retriever = DualEncoderRetriever(opt, contriever.to(dev)).eval()
    model = Atlas(opt, reader.to(dev).eval(), retriever, reader_tok, retriever_tok).eval()
    passages = []
    for seed in (77, 78, 79, 80):
        for p in atlas_synth.make_corpus(seed):
            passages.append(dict(p, id=str(len(passages))))
    flat = DistributedIndex()
    flat.init_embeddings(passages)
    model.build_index(flat, passages, opt.per_gpu_embedder_batch_size)
    index = DistributedFAISSIndex("ivfsq", None)
    index.init_embeddings(passages)
    calls = []
    train = index.train_index
    index.train_index = lambda: calls.append(1) or train()
    model.build_index(index, passages, opt.per_gpu_embedder_batch_size)
    assert calls == [1] and index.is_index_trained()
    assert torch.equal(index.embeddings.cpu().view(torch.int16), flat.embeddings.cpu().view(torch.int16))
    query, _ = atlas_synth.make_batch()
    enc = model.retriever_tokenize(query)
    ps, sc, _ = model._retrieve(index, atlas_synth.TOPK, query, enc["input_ids"], enc["attention_mask"])
    assert len(ps) == len(query) and all(len(r) == atlas_synth.TOPK for r in ps)
    assert (np.diff(np.array(sc, np.float32), axis=1) <= 0).all()
