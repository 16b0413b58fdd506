"""GPU checks of the product-quantized index (csrc/pq.cu, atlas_b200.index.DistributedFAISSIndex) against the numpy
restatement oracle/pq_oracle.py: the code scan + exact top-k, the encoder, the k-means training, the module and
Atlas.build_index with host-resident rows."""
import os
import tempfile

import numpy as np
import pytest
import torch

import pq_oracle

pytestmark = pytest.mark.gpu

DIM = 768


def _ulp16(v):
    """fp16 ulp at |v| (vectorised)."""
    a = np.abs(np.asarray(v, dtype=np.float32)).astype(np.float16)
    return (np.nextafter(a, np.float16(np.inf)) - a).astype(np.float32)


def _random_index(rng, kind, M, n, n_list=None, scale=0.05):
    cb = (rng.standard_normal((M, 256, DIM // M)) * scale).astype(np.float32)
    codes = rng.integers(0, 256, (n, M), dtype=np.uint8)
    coarse = lists = None
    if kind == "ivfpq":
        n_list = n_list or max(1, int(np.sqrt(n)))
        coarse = (rng.standard_normal((n_list, DIM)) * scale).astype(np.float32)
        lists = rng.integers(0, n_list, n).astype(np.uint16)
    return cb, codes, coarse, lists


def _to_dev(cb, codes, coarse, lists):
    dev = torch.device("cuda")
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)
    return t(cb), t(codes), t(coarse), t(lists)


def _search(cb, codes, coarse, lists, q, k, exhaustive=False):
    from atlas_b200 import ops

    d = _to_dev(cb, codes, coarse, lists)
    s, i, st = ops.pq_topk(d[1], d[3], d[0], d[2], torch.from_numpy(q).cuda(), k, exhaustive=exhaustive)
    return s.cpu().numpy(), i.cpu().numpy(), int(st.item())


SCAN_CASES = [
    ("pq", 8, 300, 1, 1),
    ("ivfpq", 8, 300, 7, 300),
    ("pq", 16, 5000, 37, 40),
    ("ivfpq", 16, 300000, 256, 40),
    ("pq", 32, 300000, 300, 100),
    ("ivfpq", 64, 120000, 300, 1024),
    ("pq", 96, 20000, 5, 500),
    ("ivfpq", 96, 50000, 130, 7),
    ("pq", 64, 40000, 64, 1024),
]


@pytest.mark.parametrize("kind,M,n,nq,k", SCAN_CASES)
def test_scan_parity_given_codebooks(kind, M, n, nq, k):
    """fp16 scores within 1 ulp of the oracle's; the top-k holds every row that beats the oracle's k-th score by more
    than 2 ulp and nothing below it by more than 2 ulp."""
    rng = np.random.default_rng(1000 + M + n % 997)
    cb, codes, coarse, lists = _random_index(rng, kind, M, n)
    q = rng.standard_normal((nq, DIM)).astype(np.float16)
    s, ids, st = _search(cb, codes, coarse, lists, q, k)
    if st:
        s, ids, _ = _search(cb, codes, coarse, lists, q, k, exhaustive=True)
    ref = pq_oracle.adc_scores(q, codes, cb, coarse, lists).astype(np.float32)
    s = s.astype(np.float32)
    assert (ids >= 0).all() and (ids < n).all()
    assert all(len(set(r)) == k for r in ids.tolist())
    got_ref = np.take_along_axis(ref, ids, 1)
    assert (np.abs(s - got_ref) <= _ulp16(got_ref)).all()
    assert (np.diff(s, axis=1) <= 0).all()
    kth = -np.partition(-ref, k - 1, axis=1)[:, k - 1:k]
    tol = 2 * _ulp16(kth)
    assert (got_ref >= kth - tol).all()
    for r in range(nq):
        must = np.flatnonzero(ref[r] > kth[r, 0] + tol[r, 0])
        assert np.isin(must, ids[r]).all(), r


@pytest.mark.parametrize("kind", ["pq", "ivfpq"])
def test_scan_exact_grid_bit_exact(kind):
    """Small-integer LUT values and coarse terms: every fp32 sum is exact, so scores and canonical ids match bitwise."""
    rng = np.random.default_rng(7)
    M, n, nq, k = 16, 70000, 40, 64
    cb = rng.integers(-2, 3, (M, 256, DIM // M)).astype(np.float32)
    codes = rng.integers(0, 256, (n, M), dtype=np.uint8)
    coarse = lists = None
    if kind == "ivfpq":
        coarse = rng.integers(-2, 3, (264, DIM)).astype(np.float32)
        lists = rng.integers(0, 264, n).astype(np.uint16)
    q = np.zeros((nq, DIM), np.float16)
    for r in range(nq):
        q[r, rng.choice(DIM, 6, replace=False)] = rng.integers(-1, 2, 6)
    s, ids, st = _search(cb, codes, coarse, lists, q, k)
    if st:
        s, ids, _ = _search(cb, codes, coarse, lists, q, k, exhaustive=True)
    want_v, want_i = pq_oracle.canonical_topk(pq_oracle.adc_scores(q, codes, cb, coarse, lists), k)
    assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16))
    assert np.array_equal(ids, want_i)


def test_sampled_and_exhaustive_paths_agree():
    rng = np.random.default_rng(11)
    cb, codes, coarse, lists = _random_index(rng, "ivfpq", 16, 200000)
    q = rng.standard_normal((100, DIM)).astype(np.float16)
    s1, i1, st = _search(cb, codes, coarse, lists, q, 40)
    s2, i2, _ = _search(cb, codes, coarse, lists, q, 40, exhaustive=True)
    assert st == 0
    assert np.array_equal(s1.view(np.uint16), s2.view(np.uint16)) and np.array_equal(i1, i2)


def test_all_equal_scores_raise_status_and_exhaustive_returns_first_ids():
    rng = np.random.default_rng(12)
    n, k = 100000, 40
    cb = np.zeros((8, 256, 96), np.float32)
    codes = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    q = rng.standard_normal((3, DIM)).astype(np.float16)
    _, _, st = _search(cb, codes, None, None, q, k)
    assert st == 1
    s, ids, _ = _search(cb, codes, None, None, q, k, exhaustive=True)
    assert (s == 0).all() and np.array_equal(ids, np.tile(np.arange(k), (3, 1)))


def _clustered(rng, n, centers=64, spread=0.3):
    c = rng.standard_normal((centers, DIM)).astype(np.float32)
    x = c[rng.integers(0, centers, n)] + spread * rng.standard_normal((n, DIM)).astype(np.float32)
    return (x / np.sqrt(DIM)).astype(np.float16)


@pytest.mark.parametrize("kind,M", [("pq", 16), ("ivfpq", 32), ("pq", 96)])
def test_encode_is_nearest_centroid(kind, M):
    from atlas_b200 import ops

    rng = np.random.default_rng(21)
    x = _clustered(rng, 6000)
    cb, _, coarse, _ = _random_index(rng, kind, M, 10, n_list=40, scale=0.02)
    d = _to_dev(cb, None, coarse, None)
    codes = torch.empty((len(x), M), dtype=torch.uint8, device="cuda")
    lists = torch.empty(len(x), dtype=torch.uint16, device="cuda") if coarse is not None else None
    ops.pq_encode(torch.from_numpy(x).cuda(), d[0], d[2], codes, lists)
    codes = codes.cpu().numpy()
    r = x.astype(np.float32)
    if coarse is not None:
        lists = lists.cpu().numpy().astype(np.int64)
        ip = r @ coarse.T
        best = ip.max(1)
        assert (ip[np.arange(len(x)), lists] >= best - 2e-3 * (1 + np.abs(best))).all()
        r = r - coarse[lists]
    dist = pq_oracle.sub_distances(r, cb)
    got = np.take_along_axis(dist, codes.astype(np.int64)[:, :, None], 2)[:, :, 0]
    dmin = dist.min(2)
    assert (got <= dmin + 1e-5 * (1 + dmin)).all(), float((got - dmin).max())


def _faiss_index(kind, M, x):
    import synth
    from atlas_b200.index import DistributedFAISSIndex

    index = DistributedFAISSIndex(kind, M)
    index.init_embeddings(synth.make_passages(len(x)))
    index.embeddings[:, :] = torch.from_numpy(x).T
    return index


def test_training_is_deterministic():
    rng = np.random.default_rng(31)
    x = _clustered(rng, 30000)
    index = _faiss_index("ivfpq", 16, x)
    index.train_index()
    a = {k: (v.cpu().clone() if torch.is_tensor(v) else v) for k, v in index._pq.items()}
    index.train_index()
    for key in ("codebooks", "coarse", "codes", "list_ids"):
        assert torch.equal(a[key].view(torch.uint8), index._pq[key].cpu().view(torch.uint8)), key


@pytest.mark.parametrize("kind,M", [("pq", 16), ("ivfpq", 16)])
def test_training_quality_vs_oracle_lloyd(kind, M):
    """Quantization MSE within 5 % of the oracle's plain Lloyd pipeline, recall@40 within 0.02 of the oracle's (both
    against the exact fp16 flat search of the same rows)."""
    import mips_oracle

    rng = np.random.default_rng(41)
    n, k = 8000, 40
    x = _clustered(rng, n)
    q = _clustered(rng, 64)
    index = _faiss_index(kind, M, x)
    index.train_index()
    p = index._pq
    cb = p["codebooks"].cpu().numpy()
    coarse = None if p["coarse"] is None else p["coarse"].cpu().numpy()
    lists = None if p["list_ids"] is None else p["list_ids"].cpu().numpy().astype(np.int64)
    codes = p["codes"].cpu().numpy()
    mse_gpu = pq_oracle.quantization_mse(x, codes, cb, coarse, lists)
    ocb, ocoarse = pq_oracle.train(x, M, index.n_list(), iters=25, seed=5)
    ocodes, olists = pq_oracle.encode(x, ocb, ocoarse)
    mse_ref = pq_oracle.quantization_mse(x, ocodes, ocb, ocoarse, olists)
    assert mse_gpu <= 1.05 * mse_ref, (mse_gpu, mse_ref)

    _, exact = mips_oracle.canonical_topk(mips_oracle.scores_fp16(q, x), k)
    docs, _ = index.search_knn(torch.from_numpy(q).cuda(), k)
    got = np.array([[int(d["id"]) for d in row] for row in docs])
    _, ref_ids = pq_oracle.canonical_topk(pq_oracle.adc_scores(q, ocodes, ocb, ocoarse, olists), k)
    recall = lambda ids: np.mean([len(set(a) & set(b)) / k for a, b in zip(ids.tolist(), exact.tolist())])
    assert recall(got) >= recall(ref_ids) - 0.02, (recall(got), recall(ref_ids))


@pytest.mark.parametrize("kind", ["pq", "ivfpq"])
def test_module_search_save_load_and_memory(kind, monkeypatch):
    from atlas_b200 import ops

    rng = np.random.default_rng(51)
    n, M, k = 200000, 16, 40
    x = _clustered(rng, n)
    q = torch.from_numpy(_clustered(rng, 50)).cuda()
    index = _faiss_index(kind, M, x)
    assert not index.is_index_trained() and index.is_in_gpu is False
    assert not index._bank.is_cuda and index.embeddings.shape == (DIM, n)
    from atlas_b200._lib import AtlasB200Error

    with pytest.raises(AtlasB200Error):
        index.search_knn(q, k)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    index.train_index()
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    list_bytes = 2 if kind == "ivfpq" else 0
    assert grown <= n * (M + list_bytes) + (8 << 20), grown
    assert grown < n * DIM * 2 // 10
    assert index.is_index_trained()

    docs, scores = index.search_knn(q, k)
    p = index._pq
    s, i, _ = ops.pq_topk(p["codes"], p["list_ids"], p["codebooks"], p["coarse"], q, k)
    assert [[int(d["id"]) for d in row] for row in docs] == i.cpu().tolist()
    assert np.array_equal(np.array(scores, np.float32), s.float().cpu().numpy())

    with tempfile.TemporaryDirectory() as tmp:
        index.save_index(tmp, 1)
        assert os.path.exists(os.path.join(tmp, f"index{kind}_{M}_rank_0.atlas_b200.pt"))
        from atlas_b200.index import DistributedFAISSIndex

        monkeypatch.setattr(ops, "pq_train", lambda *a, **kw: (_ for _ in ()).throw(AssertionError("retrained")))
        index2 = DistributedFAISSIndex(kind, M)
        index2.load_index(tmp, 1)
        assert index2.is_index_trained() and not index2._bank.is_cuda
        assert torch.equal(index2.embeddings, index.embeddings)
        docs2, scores2 = index2.search_knn(q, k)
        assert scores2 == scores and docs2 == docs


def test_build_index_with_host_rows():
    """Atlas.build_index into a DistributedFAISSIndex: host rows bit-identical to the flat bank of the same build, then
    the index is retrained and retrieval runs end to end."""
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
    index = DistributedFAISSIndex("ivfpq", 16)
    index.init_embeddings(passages)
    index.train_index = _counting(index.train_index)
    model.build_index(index, passages, opt.per_gpu_embedder_batch_size)
    assert index.train_index.calls == 1 and index.is_index_trained()
    assert torch.equal(index.embeddings.cpu().view(torch.int16), flat.embeddings.cpu().view(torch.int16))
    query, _ = atlas_synth.make_batch()
    enc = model.retriever_tokenize(query)
    ps, sc, _ = model._retrieve(index, atlas_synth.TOPK, query, enc["input_ids"], enc["attention_mask"])
    assert len(ps) == len(query) and all(len(r) == atlas_synth.TOPK for r in ps)
    assert (np.diff(np.array(sc, np.float32), axis=1) <= 0).all()


def _counting(fn):
    def wrapped():
        wrapped.calls += 1
        return fn()

    wrapped.calls = 0
    return wrapped
