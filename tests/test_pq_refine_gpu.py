"""GPU checks of the exact re-ranking of product-quantized candidates (csrc/pq_refine.cu, `ops.pq_refine_topk`,
`DistributedFAISSIndex(refine_factor > 1)`) against oracle/pq_refine_oracle.py, the exact flat search and the unrefined
PQ search."""
import numpy as np
import pytest
import torch

import mips_oracle
import pq_refine_oracle

pytestmark = pytest.mark.gpu

DIM = 768


def _ulp16(v):
    a = np.abs(np.asarray(v, dtype=np.float32)).astype(np.float16)
    return (np.nextafter(a, np.float16(np.inf)) - a).astype(np.float32)


def _pinned(x):
    return torch.from_numpy(np.ascontiguousarray(x)).pin_memory()


def _grid_rows(rng, n):
    """Halves in [-2, 2] and queries of small integers: every fp32 partial sum of a score is exact."""
    return (rng.integers(-4, 5, (n, DIM)) / 2).astype(np.float16)


def _grid_queries(rng, nq):
    return rng.integers(-2, 3, (nq, DIM)).astype(np.float16)


def _candidates(rng, nq, n, k_cand):
    return np.argsort(rng.random((nq, n)), axis=1)[:, :k_cand].astype(np.int64)


def _refine(rows, q, cand, k, id_base=0, id_stride=1):
    from atlas_b200 import ops

    rows_t = rows if torch.is_tensor(rows) else _pinned(rows)
    s, i = ops.pq_refine_topk(rows_t, torch.from_numpy(q).cuda(), torch.from_numpy(cand).cuda(), k, id_base, id_stride)
    assert s.is_cuda and i.is_cuda and s.dtype == torch.float16 and i.dtype == torch.int64
    return s.cpu().numpy(), i.cpu().numpy()


def _separated(v_sorted, k):
    """Positions p < k whose score differs by more than 2 fp16 ulp from its neighbours in the full sorted list."""
    v = v_sorted.astype(np.float32)
    tol = 2 * _ulp16(v)
    sep = np.ones(v.shape, bool)
    sep[:, 1:] &= (v[:, :-1] - v[:, 1:]) > tol[:, 1:]
    sep[:, :-1] &= (v[:, :-1] - v[:, 1:]) > tol[:, :-1]
    return sep[:, :k]


def _check_close(s, ids, q, rows, cand, k, id_base=0, id_stride=1):
    """Scores within one fp16 ulp of the oracle's score of the same row, descending, ids among the candidates, and
    equal to the oracle's wherever the oracle's neighbouring scores are not tied within 2 ulp."""
    nq = len(q)
    assert s.shape == (nq, k) and ids.shape == (nq, k)
    if nq == 0:
        return
    exact = mips_oracle.scores_fp16(q, rows).astype(np.float32)
    local = (ids - id_base) // id_stride
    assert (local >= 0).all()
    for r in range(nq):
        assert np.isin(local[r], cand[r]).all() and len(set(local[r].tolist())) == k
    got_ref = np.take_along_axis(exact, local, 1)
    assert (np.abs(s.astype(np.float32) - got_ref) <= _ulp16(got_ref)).all()
    assert (np.diff(s.astype(np.float32), axis=1) <= 0).all()
    all_v, all_i = pq_refine_oracle.refine_topk(q, rows, cand, cand.shape[1], id_base, id_stride)
    sep = _separated(all_v, k)
    assert np.array_equal(ids[sep], all_i[:, :k][sep])


KERNEL_CASES = [   # nq, k, k'
    (0, 10, 40),
    (1, 1, 1),
    (1, 40, 160),
    (7, 100, 100),
    (3, 1024, 1024),
    (256, 40, 160),
    (256, 40, 1024),
    (300, 64, 200),
]


@pytest.mark.parametrize("nq,k,k_cand", KERNEL_CASES)
def test_kernel_bit_exact_on_grid(nq, k, k_cand):
    rng = np.random.default_rng(100 + nq + k_cand)
    n = 3000
    rows = _grid_rows(rng, n)
    q = _grid_queries(rng, nq)
    cand = _candidates(rng, nq, n, k_cand)
    s, ids = _refine(rows, q, cand, k, id_base=3, id_stride=7)
    want_v, want_i = pq_refine_oracle.refine_topk(q, rows, cand, k, 3, 7)
    assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16))
    assert np.array_equal(ids, want_i)


@pytest.mark.parametrize("nq,k,k_cand", KERNEL_CASES)
def test_kernel_within_one_ulp_on_gaussian(nq, k, k_cand):
    rng = np.random.default_rng(200 + nq + k_cand)
    n = 5000
    rows = (rng.standard_normal((n, DIM)) / 16).astype(np.float16)
    q = rng.standard_normal((nq, DIM)).astype(np.float16)
    cand = _candidates(rng, nq, n, k_cand)
    s, ids = _refine(rows, q, cand, k, id_base=1, id_stride=2)
    _check_close(s, ids, q, rows, cand, k, 1, 2)
    s2, ids2 = _refine(rows, q, cand, k, id_base=1, id_stride=2)
    assert np.array_equal(s.view(np.uint16), s2.view(np.uint16)) and np.array_equal(ids, ids2)   # deterministic


def test_kernel_skips_out_of_range_candidates_and_reads_row_slices():
    rng = np.random.default_rng(5)
    n = 2000
    base = _pinned(_grid_rows(rng, n + 100))
    rows_t = base[100:]                          # a pinned slice: its pointer is inside the pinned allocation
    rows = rows_t.numpy()
    q = _grid_queries(rng, 9)
    cand = _candidates(rng, 9, n, 50)
    cand[0, :45] = -1
    cand[1, 3] = n
    cand[2, :] = -1
    s, ids = _refine(rows_t, q, cand, 8)
    want_v, want_i = pq_refine_oracle.refine_topk(q, rows, cand, 8)
    assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16)) and np.array_equal(ids, want_i)
    assert (ids[0, 5:] == -1).all() and (ids[2] == -1).all()


def test_argument_errors():
    from atlas_b200 import ops
    from atlas_b200._lib import MAX_TOPK, AtlasB200Error

    rows = _pinned(np.zeros((100, DIM), np.float16))
    q = torch.zeros(2, DIM, device="cuda")
    cand = torch.zeros(2, 10, dtype=torch.int64, device="cuda")
    with pytest.raises(AtlasB200Error, match="pinned"):
        ops.pq_refine_topk(torch.zeros(100, DIM, dtype=torch.float16), q, cand, 5)
    with pytest.raises(AtlasB200Error, match="CPU fp16"):
        ops.pq_refine_topk(rows.cuda(), q, cand, 5)
    with pytest.raises(AtlasB200Error, match="k <= k'"):
        ops.pq_refine_topk(rows, q, cand, 11)
    with pytest.raises(AtlasB200Error, match="MAX_TOPK"):
        ops.pq_refine_topk(rows, q, torch.zeros(2, MAX_TOPK + 1, dtype=torch.int64, device="cuda"), 5)
    with pytest.raises(AtlasB200Error, match="int64"):
        ops.pq_refine_topk(rows, q, cand.int(), 5)


# ----------------------------------------------------------------------------------------------- the module
def _faiss_index(kind, M, x, refine_factor=1):
    import synth
    from atlas_b200.index import DistributedFAISSIndex

    index = DistributedFAISSIndex(kind, M, refine_factor=refine_factor)
    index.init_embeddings(synth.make_passages(len(x)))
    index.embeddings[:, :] = torch.from_numpy(x).T
    index.train_index()
    return index


def _clustered(rng, n, centers=64, spread=0.3):
    c = rng.standard_normal((centers, DIM)).astype(np.float32)
    x = c[rng.integers(0, centers, n)] + spread * rng.standard_normal((n, DIM)).astype(np.float32)
    return (x / np.sqrt(DIM)).astype(np.float16)


@pytest.mark.parametrize("kind", ["pq", "ivfpq"])
def test_refined_search_over_every_row_is_the_flat_search_on_grid(kind):
    from atlas_b200 import ops

    rng = np.random.default_rng(61)
    n, k = 1000, 40
    x = _grid_rows(rng, n)
    q = torch.from_numpy(_grid_queries(rng, 50)).cuda()
    index = _faiss_index(kind, 16, x, refine_factor=25)         # 40 x 25 = 1000 candidates = every row
    s, i = index.search_device(q, k)
    fs, fi, st = ops.mips_topk(torch.from_numpy(x).cuda(), q, k)
    assert int(st.item()) == 0
    assert torch.equal(s.view(torch.int16), fs.view(torch.int16)) and torch.equal(i, fi)


@pytest.mark.parametrize("kind", ["pq", "ivfpq"])
def test_refined_search_over_every_row_is_the_flat_search_on_gaussian(kind):
    from atlas_b200 import ops

    rng = np.random.default_rng(62)
    n, k = 1000, 32
    x = _clustered(rng, n)
    qn = _clustered(rng, 40)
    index = _faiss_index(kind, 16, x, refine_factor=40)         # 1280 > 1000: clamped to every row
    s, i = index.search_device(torch.from_numpy(qn).cuda(), k)
    fs, fi, _ = ops.mips_topk(torch.from_numpy(x).cuda(), torch.from_numpy(qn).cuda(), k)
    s, i, fs, fi = s.cpu().numpy(), i.cpu().numpy(), fs.cpu().numpy(), fi.cpu().numpy()
    assert (np.abs(s.astype(np.float32) - fs.astype(np.float32)) <= _ulp16(fs)).all()
    _check_close(s, i, qn, x, np.tile(np.arange(n), (len(qn), 1)), k)
    all_v, _ = mips_oracle.canonical_topk(mips_oracle.scores_fp16(qn, x), n)
    sep = _separated(all_v, k)
    assert np.array_equal(i[sep], fi[sep])


def test_refine_factor_one_is_bit_identical_to_pq_topk():
    from atlas_b200 import ops

    rng = np.random.default_rng(63)
    x = _clustered(rng, 20000)
    q = torch.from_numpy(_clustered(rng, 77)).cuda()
    index = _faiss_index("ivfpq", 16, x)
    assert index.refine_factor == 1
    s, i = index.search_device(q, 40)
    p = index._pq
    ws, wi, st = ops.pq_topk(p["codes"], p["list_ids"], p["codebooks"], p["coarse"], q, 40)
    assert int(st.item()) == 0
    assert torch.equal(s.view(torch.int16), ws.view(torch.int16)) and torch.equal(i, wi)


def test_refined_recall_is_at_least_unrefined():
    from atlas_b200 import ops

    rng = np.random.default_rng(64)
    n, k = 8192, 40
    x = _clustered(rng, n)
    q = torch.from_numpy(_clustered(rng, 128)).cuda()
    _, exact, _ = ops.mips_topk(torch.from_numpy(x).cuda(), q, k)
    exact = exact.cpu().tolist()
    index = _faiss_index("ivfpq", 16, x)
    recall = lambda ids: np.mean([len(set(a) & set(b)) / k for a, b in zip(ids.cpu().tolist(), exact)])
    _, plain = index.search_device(q, k)
    index.refine_factor = 4
    s, refined = index.search_device(q, k)
    assert recall(refined) >= recall(plain), (recall(refined), recall(plain))
    # the refined scores are the exact scores of the rows returned
    ref = mips_oracle.scores_fp16(q.cpu().numpy(), x).astype(np.float32)
    got = np.take_along_axis(ref, refined.cpu().numpy(), 1)
    assert (np.abs(s.float().cpu().numpy() - got) <= _ulp16(got)).all()


def test_exhaustive_retry_refines_too(monkeypatch):
    from atlas_b200 import ops

    rng = np.random.default_rng(65)
    n, k, R = 40000, 40, 4
    x = np.tile(rng.standard_normal((1, DIM)).astype(np.float16) / 16, (n, 1))     # every row equal: PQ scores tie
    q = torch.from_numpy(rng.standard_normal((3, DIM)).astype(np.float16)).cuda()
    index = _faiss_index("pq", 8, x, refine_factor=R)
    _, _, status = index.search_device(q, k, return_status=True)
    assert int(status.item()) == 1
    calls = []
    real = ops.pq_refine_topk
    monkeypatch.setattr(ops, "pq_refine_topk", lambda *a, **kw: calls.append(a[2].shape) or real(*a, **kw))
    s, i = index.search_device(q, k)
    assert calls == [(3, k * R), (3, k * R)]                     # the fast path, then the exhaustive retry
    assert torch.equal(i.cpu(), torch.arange(k).repeat(3, 1))
    want = mips_oracle.scores_fp16(q.cpu().numpy(), x[:1]).astype(np.float32)
    assert (np.abs(s.float().cpu().numpy() - want) <= _ulp16(want)).all()


def test_unpinned_rows_raise():
    from atlas_b200._lib import AtlasB200Error

    rng = np.random.default_rng(66)
    index = _faiss_index("pq", 16, _clustered(rng, 2000), refine_factor=2)
    index._bank = torch.empty_like(index._bank, pin_memory=False).copy_(index._bank)     # a pageable copy
    assert not index._bank.is_pinned()
    with pytest.raises(AtlasB200Error, match="pinned"):
        index.search_device(torch.zeros(2, DIM, device="cuda"), 10)


def test_device_memory_does_not_grow_with_rows():
    """Refinement adds no per-passage device memory: after a refined search, the device holds the unrefined index plus
    scratch whose size depends on the queries and k' (and sqrt(k' n) for the candidate search), never a copy of rows."""
    from atlas_b200 import ops
    from atlas_b200._lib import lib

    rng = np.random.default_rng(67)
    n, M, k, R = 200000, 16, 40, 4
    index = _faiss_index("ivfpq", M, _clustered(rng, n))
    q = torch.from_numpy(_clustered(rng, 64)).cuda()
    index.search_device(q, k)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    index.refine_factor = R
    torch.cuda.reset_peak_memory_stats()
    index.search_device(q, k)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    peak = torch.cuda.max_memory_allocated() - before
    n_list = index._pq["n_list"]
    bound = (lib().atlas_b200_pq_workspace_bytes(ops.PQ_OP_SEARCH, n, M, n_list, k * R)
             + lib().atlas_b200_pq_refine_workspace_bytes(64, k * R) + 64 * k * R * 16 + (2 << 20))
    assert grown <= bound and peak <= bound + (1 << 20), (grown, peak, bound)
    assert peak < n * DIM * 2 // 10


def test_build_index_then_refined_search_sees_the_new_rows():
    """Atlas.build_index writes the host rows; a refined search over every row afterwards returns what the flat index
    built from the same passages returns (every passage, scores within one fp16 ulp, the same order wherever the
    scores are not tied within 2 ulp)."""
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
    model.build_index(index, passages, opt.per_gpu_embedder_batch_size)
    query, _ = atlas_synth.make_batch()
    enc = model.retriever_tokenize(query)
    n = len(passages)
    model.opt.faiss_refine_factor = 2                              # k' = min(2 n, n): every row is a candidate
    ps, sc, _ = model._retrieve(index, n, query, enc["input_ids"], enc["attention_mask"])
    assert index.refine_factor == 2
    fps, fsc, _ = model._retrieve(flat, n, query, enc["input_ids"], enc["attention_mask"])
    assert not hasattr(flat, "refine_factor")
    ids = np.array([[int(p["id"]) for p in r] for r in ps])
    fids = np.array([[int(p["id"]) for p in r] for r in fps])
    sc, fsc = np.array(sc, np.float32), np.array(fsc, np.float32)
    assert (np.sort(ids, 1) == np.arange(n)).all()
    by_id = np.empty_like(fsc)
    np.put_along_axis(by_id, fids, fsc, 1)
    assert (np.abs(sc - np.take_along_axis(by_id, ids, 1)) <= _ulp16(sc)).all()
    sep = _separated(fsc.astype(np.float16), n)
    assert np.array_equal(ids[sep], fids[sep])
