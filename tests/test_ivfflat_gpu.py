"""GPU checks of the IVF-Flat passage index (`DistributedFAISSIndex("ivfflat")` / ("flat"), csrc/ivfflat.cu): exact grid
states bit for bit against the numpy restatement (tests/test_ivfflat_cpu.flat_probed_topk), the full scan against the flat
index (`ops.mips_topk`), Gaussian probed states, the search's properties (batch independence, monotonicity in nprobe, the
small-shard extension, the sampled and exhaustive paths, CUDA-graph replay) and the module."""
import os
import tempfile
import types

import numpy as np
import pytest
import torch

import ivf_probe_oracle
import mips_oracle
from test_ivfflat_cpu import flat_probed_topk

pytestmark = pytest.mark.gpu

DIM = 768


def _ulp16(v):
    a = np.abs(np.asarray(v, dtype=np.float32)).astype(np.float16)
    return (np.nextafter(a, np.float16(np.inf)) - a).astype(np.float32)


# ------------------------------------------------------------------ states
def _state(rng, sizes, grid=False, scale=0.05):
    """list l holds sizes[l] rows in random row order; small-integer rows, centroids (exact sums) when grid."""
    sizes = list(sizes)
    n, n_list = sum(sizes), len(sizes)
    lists = rng.permutation(np.repeat(np.arange(n_list), sizes)).astype(np.int64)
    if grid:
        rows = rng.integers(-2, 3, (n, DIM)).astype(np.float16)
        coarse = rng.integers(-2, 3, (n_list, DIM)).astype(np.float32)
    else:
        rows = (rng.standard_normal((n, DIM)) * scale).astype(np.float16)
        coarse = (rng.standard_normal((n_list, DIM)) * scale).astype(np.float32)
    return dict(rows=rows, coarse=coarse, lists=lists, n=n, n_list=n_list)


def _grid_queries(rng, nq):
    q = np.zeros((nq, DIM), np.float16)
    for r in range(nq):
        q[r, rng.choice(DIM, 6, replace=False)] = rng.integers(-2, 3, 6)
    return q


def _device(st):
    from atlas_b200 import ops

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    slot_rows, tile_lists, row_slot = ops.ivfsq_layout(t(st["lists"].astype(np.int32)), st["n_list"])
    rows = torch.zeros((slot_rows.numel(), DIM), dtype=torch.float16, device="cuda")
    rows[row_slot.to(torch.int64)] = t(st["rows"])
    d = dict(n=st["n"], n_list=st["n_list"], coarse=t(st["coarse"]), rows=rows, slot_rows=slot_rows, tile_lists=tile_lists,
             bank=t(st["rows"]))
    d["list_tile_off"], d["list_rows"] = ops.ivfsq_list_tables(slot_rows, tile_lists, st["n_list"])
    return d


def _search_dev(d, q, k, nprobe=None, exhaustive=False, id_base=0, id_stride=1, tables=True, workspace=None):
    from atlas_b200 import ops

    qd = q if torch.is_tensor(q) else torch.from_numpy(q).cuda()
    tb = dict(list_tile_off=d["list_tile_off"], list_rows=d["list_rows"]) if tables else {}
    return ops.ivfflat_topk(d["rows"], d["slot_rows"], d["tile_lists"], d["n"], d["coarse"], qd, k, id_base, id_stride,
                            workspace, exhaustive=exhaustive, nprobe=nprobe, **tb)


def _search(d, q, k, nprobe=None, exhaustive=False, id_base=0, id_stride=1, retry=True):
    s, i, stat = _search_dev(d, q, k, nprobe, exhaustive, id_base, id_stride)
    stat = int(stat.item())
    if stat and retry and not exhaustive:
        s, i, _ = _search_dev(d, q, k, nprobe, True, id_base, id_stride)
    return s.cpu().numpy(), i.cpu().numpy(), stat


def _flat(d, q, k):
    from atlas_b200 import ops

    s, i, stat = ops.mips_topk(d["bank"], torch.from_numpy(q).cuda(), k)
    if int(stat.item()):
        s, i, _ = ops.mips_topk(d["bank"], torch.from_numpy(q).cuda(), k, exhaustive=True)
    return s.cpu().numpy(), i.cpu().numpy()


def _sizes(st):
    return np.bincount(st["lists"], minlength=st["n_list"])


_GRID = {}


def _grid_state():
    if not _GRID:
        rng = np.random.default_rng(7)
        n_list = 141
        sizes = np.bincount(rng.integers(0, n_list, 20000), minlength=n_list)
        sizes[:5] = [0, 1, 63, 64, 65]             # list lengths around the 64-slot tile
        st = _state(rng, sizes, grid=True)
        _GRID["st"], _GRID["d"] = st, _device(st)
    return _GRID["st"], _GRID["d"]


# ------------------------------------------------------------------ 1. exact grid states
@pytest.mark.parametrize("nq", [1, 3, 40, 129, 256, 300])
@pytest.mark.parametrize("nprobe", [1, 2, 7, None])
def test_grid_bit_exact(nprobe, nq):
    """Small-integer rows, centroids and sparse queries: T and every score are exact and full of ties, so scores and
    canonical ids match the oracle over the probed rows bitwise, with a non-zero id_base / id_stride."""
    st, d = _grid_state()
    rng = np.random.default_rng(100 * nq + (nprobe or 0))
    q = _grid_queries(rng, nq)
    for k in (1, 40, 1024):
        want_v, want_i, _ = flat_probed_topk(q, st["rows"], st["coarse"], st["lists"], nprobe, k)
        s, ids, _ = _search(d, q, k, nprobe, id_base=7, id_stride=3)
        assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16)), k
        assert np.array_equal(ids, 7 + 3 * want_i), k


# ------------------------------------------------------------------ 2. the full scan is the flat index
def test_full_scan_grid_is_the_flat_index_bitwise():
    st, d = _grid_state()
    rng = np.random.default_rng(11)
    for nq in (5, 256, 300):
        q = _grid_queries(rng, nq)
        for k in (1, 40, 1024):
            want_s, want_i = _flat(d, q, k)
            for nprobe in (None, st["n_list"], st["n_list"] + 9):
                s, ids, _ = _search(d, q, k, nprobe)
                assert np.array_equal(s.view(np.uint16), want_s.view(np.uint16)) and np.array_equal(ids, want_i), (nq, k)


def test_full_scan_gaussian_matches_the_flat_index():
    """Scores within one fp16 ulp of the flat index's, ids identical wherever its scores are separated by > 2 ulp."""
    rng = np.random.default_rng(13)
    st = _state(rng, np.bincount(rng.integers(0, 300, 90000), minlength=300), scale=1.0)
    d = _device(st)
    for nq, k in ((8, 40), (256, 100)):
        q = rng.standard_normal((nq, DIM)).astype(np.float16)
        ref_s, ref_i = _flat(d, q, k)
        ref = ref_s.astype(np.float32)
        ulp = _ulp16(ref)
        for nprobe in (None, st["n_list"]):
            s, ids, _ = _search(d, q, k, nprobe)
            assert np.all(np.abs(s.astype(np.float32) - ref) <= ulp)
            for r in range(nq):
                for p in range(k - 1):
                    hi = ref[r, p - 1] if p > 0 else np.inf
                    if ref[r, p] - ref[r, p + 1] > 2 * ulp[r, p] and hi - ref[r, p] > 2 * ulp[r, p]:
                        assert ids[r, p] == ref_i[r, p], (r, p)


# ------------------------------------------------------------------ 3. Gaussian probed states
@pytest.mark.parametrize("nprobe", [1, 8])
def test_gaussian_probed_parity(nprobe):
    """Parity within one fp16 ulp against the oracle restricted to its probe sets; queries whose last probed and first
    unprobed coarse terms lie within 1e-5 of the largest |T| (where fp32 summation order could swap them) are skipped,
    and most queries must be kept."""
    rng = np.random.default_rng(17 + nprobe)
    n, n_list, nq, k = 60000, 244, 64, 40
    st = _state(rng, np.bincount(rng.integers(0, n_list, n), minlength=n_list))
    q = rng.standard_normal((nq, DIM)).astype(np.float16)
    d = _device(st)
    s, ids, _ = _search(d, q, k, nprobe)
    T = ivf_probe_oracle.sq_coarse_terms(q, st["coarse"])
    probed = ivf_probe_oracle.probe_lists(T, nprobe, _sizes(st), k)
    ref = mips_oracle.scores_fp16(q, st["rows"]).astype(np.float32)
    kept = 0
    for r in range(nq):
        ts = np.sort(T[r])[::-1]
        p = int(probed[r].sum())
        if p < n_list and ts[p - 1] - ts[p] <= 1e-5 * float(np.abs(T[r]).max()):
            continue
        kept += 1
        rows = np.flatnonzero(probed[r][st["lists"]])
        assert np.isin(ids[r], rows).all() and len(set(ids[r].tolist())) == k, r
        got_ref = ref[r, ids[r]]
        sv = s[r].astype(np.float32)
        assert (np.abs(sv - got_ref) <= np.maximum(_ulp16(got_ref), _ulp16(sv))).all(), r
        assert (np.diff(sv) <= 0).all()
        sub = ref[r, rows]
        kth = -np.partition(-sub, k - 1)[k - 1]
        tol = 2 * _ulp16(kth)
        assert (got_ref >= kth - tol).all(), r
        assert np.isin(rows[sub > kth + tol], ids[r]).all(), r
    assert kept >= 0.9 * nq, kept


# ------------------------------------------------------------------ 4. properties
def test_batch_independence():
    rng = np.random.default_rng(29)
    st = _state(rng, np.bincount(rng.integers(0, 200, 40000), minlength=200))
    d = _device(st)
    q = rng.standard_normal((300, DIM)).astype(np.float16)
    for nprobe in (4, None):
        s, ids, _ = _search(d, q, 40, nprobe)
        for r in list(range(0, 300, 37)) + [129, 255, 256, 299]:
            s1, i1, _ = _search(d, q[r:r + 1], 40, nprobe)
            assert np.array_equal(s1[0].view(np.uint16), s[r].view(np.uint16)) and np.array_equal(i1[0], ids[r]), r
        s2, i2, _ = _search(d, q[100:], 40, nprobe)
        assert np.array_equal(s2.view(np.uint16), s[100:].view(np.uint16)) and np.array_equal(i2, ids[100:])


def test_monotone_in_nprobe():
    rng = np.random.default_rng(31)
    st = _state(rng, np.bincount(rng.integers(0, 200, 40000), minlength=200))
    d = _device(st)
    q = rng.standard_normal((50, DIM)).astype(np.float16)
    prev = None
    for nprobe in (1, 4, 16, st["n_list"]):
        s, _, _ = _search(d, q, 40, nprobe)
        s = s.astype(np.float32)
        if prev is not None:
            assert (s >= prev).all(), nprobe
        prev = s


def test_extension_on_a_small_shard():
    """About 300 rows in 17 lists, nprobe = 1, k = 40: the best list alone holds fewer than 40 rows, the probe set is
    extended and 40 valid ids come back, equal to the oracle's."""
    rng = np.random.default_rng(37)
    st = _state(rng, np.bincount(rng.integers(0, 17, 300), minlength=17), grid=True)
    d = _device(st)
    q = _grid_queries(rng, 9)
    s, ids, _ = _search(d, q, 40, 1)
    want_v, want_i, probed = flat_probed_topk(q, st["rows"], st["coarse"], st["lists"], 1, 40)
    assert (probed.sum(1) > 1).all()
    assert (ids >= 0).all()
    assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16)) and np.array_equal(ids, want_i)


def test_sampled_and_exhaustive_agree():
    rng = np.random.default_rng(41)
    st = _state(rng, np.bincount(rng.integers(0, 447, 200000), minlength=447))
    d = _device(st)
    q = rng.standard_normal((100, DIM)).astype(np.float16)
    for nprobe in (3, 40, None):
        s1, i1, stat = _search(d, q, 40, nprobe, retry=False)
        s2, i2, _ = _search(d, q, 40, nprobe, exhaustive=True)
        assert stat == 0
        assert np.array_equal(s1.view(np.uint16), s2.view(np.uint16)) and np.array_equal(i1, i2), nprobe


def test_all_equal_scores_raise_status_and_exhaustive_returns_lowest_probed_ids():
    """Every row scores the same: the probe sets are the lowest list ids (ties by list id), their 25 lists hold more rows
    than the candidate lists, so status is set, and the exhaustive path returns the lowest row ids of the probed lists."""
    rng = np.random.default_rng(43)
    n, n_list, k = 100000, 50, 40
    st = _state(rng, np.bincount(rng.integers(0, n_list, n), minlength=n_list))
    st["rows"][:] = 0
    st["coarse"][:] = 0
    d = _device(st)
    q = rng.standard_normal((3, DIM)).astype(np.float16)
    _, _, stat = _search(d, q, k, 25, retry=False)
    assert stat == 1
    s, ids, _ = _search(d, q, k, 25, exhaustive=True)
    probed = ivf_probe_oracle.probe_lists(ivf_probe_oracle.sq_coarse_terms(q, st["coarse"]), 25, _sizes(st), k)
    assert (probed[:, :25].all(1) & ~probed[:, 25:].any(1)).all()
    for r in range(3):
        rows = np.flatnonzero(probed[r][st["lists"]])
        assert np.array_equal(ids[r], rows[:k]), r
        assert (s[r] == s[r, 0]).all()


def test_probed_search_replays_in_a_cuda_graph():
    from atlas_b200 import ops

    rng = np.random.default_rng(47)
    st = _state(rng, np.bincount(rng.integers(0, 200, 40000), minlength=200))
    d = _device(st)
    q = torch.from_numpy(rng.standard_normal((300, DIM)).astype(np.float16)).cuda()
    ws = ops.Workspace()
    want = [t.clone() for t in _search_dev(d, q, 40, 5, workspace=ws)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _search_dev(d, q, 40, 5, workspace=ws)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = _search_dev(d, q, 40, 5, workspace=ws)
    for t in out:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, want):
        assert torch.equal(a, b)


def test_argument_errors():
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    rng = np.random.default_rng(49)
    st = _state(rng, np.bincount(rng.integers(0, 10, 500), minlength=10))
    d = _device(st)
    q = torch.from_numpy(rng.standard_normal((4, DIM)).astype(np.float16)).cuda()
    with pytest.raises(AtlasB200Error, match="out of range"):
        _search_dev(d, q, 501)
    with pytest.raises(AtlasB200Error, match="list_tile_off"):
        ops.ivfflat_topk(d["rows"], d["slot_rows"], d["tile_lists"], d["n"], d["coarse"], q, 5, nprobe=2,
                         list_tile_off=d["list_tile_off"][:-1], list_rows=d["list_rows"])
    shifted = torch.zeros(128 * DIM + 4, dtype=torch.float16, device="cuda")[4:].view(128, DIM)     # 8-byte aligned
    with pytest.raises(AtlasB200Error, match="aligned"):
        ops.ivfflat_topk(shifted, d["slot_rows"][:128], d["tile_lists"][:2], 1, None, q, 1)
    with pytest.raises(AtlasB200Error, match="flat has none"):
        ops.ivfflat_topk(d["rows"], d["slot_rows"], d["tile_lists"], d["n"], None, q, 5, nprobe=2)


# ------------------------------------------------------------------ 5. the module
def _clustered(rng, n, centers=64, spread=0.3):
    c = rng.standard_normal((centers, DIM)).astype(np.float32)
    x = c[rng.integers(0, centers, n)] + spread * rng.standard_normal((n, DIM)).astype(np.float32)
    return (x / np.sqrt(DIM)).astype(np.float16)


def _index(x, kind, code_size=None, **kw):
    import synth
    from atlas_b200.index import DistributedFAISSIndex

    index = DistributedFAISSIndex(kind, code_size, **kw)
    index.init_embeddings(synth.make_passages(len(x)))
    index.embeddings[:, :] = torch.from_numpy(x).T
    return index


def _ids(docs):
    return [[int(doc["id"]) for doc in row] for row in docs]


def test_module_search_save_load_stale_and_memory(monkeypatch):
    from atlas_b200 import ops
    from atlas_b200.index import DistributedFAISSIndex

    rng = np.random.default_rng(53)
    n, k = 30000, 40
    x = _clustered(rng, n)
    q = torch.from_numpy(_clustered(rng, 20)).cuda()
    index = _index(x, "ivfflat", nprobe=4)
    assert not index.is_index_trained() and index.is_in_gpu is False and not index._bank.is_cuda
    assert index._bank.is_pinned() and tuple(index.embeddings.shape) == (DIM, n)
    index.train_index()
    p = index._pq
    n_list = int(np.floor(np.sqrt(n)))
    assert p["n_list"] == n_list and p["rows"].dtype == torch.float16
    # device bytes per passage: 1536 of row and 4 of row id per slot, and at most 63 padding slots per list
    slots = p["rows"].shape[0]
    assert p["rows"].numel() * 2 + p["slot_rows"].numel() * 4 == slots * (1536 + 4)
    assert n <= slots <= n + 63 * n_list and slots % 64 == 0

    docs, scores = index.search_knn(q, k)
    assert "list_tile_off" in p
    s, i, _ = ops.ivfflat_topk(p["rows"], p["slot_rows"], p["tile_lists"], n, p["coarse"], q, k, nprobe=4)
    assert _ids(docs) == i.cpu().tolist()
    assert np.array_equal(np.array(scores, np.float32), s.float().cpu().numpy())
    # the scores are the exact ones: refine_factor is accepted and ignored
    index.refine_factor = 3
    assert index.search_knn(q, k) == (docs, scores)
    index.refine_factor = 1

    with tempfile.TemporaryDirectory() as tmp:
        index.save_index(tmp, 1)
        assert os.path.exists(os.path.join(tmp, "indexivfflat_rank_0.atlas_b200.pt"))
        index2 = DistributedFAISSIndex("ivfflat", nprobe=4)
        monkeypatch.setattr(index2, "train_index", lambda: pytest.fail("load_index retrained"))
        index2.load_index(tmp, 1)
        assert index2.is_index_trained()
        for key in ("rows", "slot_rows", "tile_lists", "coarse"):
            assert torch.equal(index2._pq[key], p[key]), key
        assert index2.search_knn(q, k) == (docs, scores)
        index2.nprobe = None
        index.nprobe = None
        assert index2.search_knn(q, k) == index.search_knn(q, k)

    # writing rows makes the index stale; retraining drops the probe tables
    index.embeddings = torch.from_numpy(x).T
    assert not index.is_index_trained()
    index.train_index()
    assert "list_tile_off" not in index._pq
    index.mark_stale()
    assert not index.is_index_trained()


def test_training_is_deterministic_matches_ivfsq_and_works_from_one_row():
    from atlas_b200 import ops

    rng = np.random.default_rng(57)
    x = _clustered(rng, 20000)
    a, b = _index(x, "ivfflat"), _index(x, "ivfflat")
    a.train_index()
    b.train_index()
    for key in ("coarse", "rows", "slot_rows", "tile_lists"):
        assert torch.equal(a._pq[key], b._pq[key]), key
    sq = _index(x, "ivfsq")
    sq.train_index()
    assert torch.equal(a._pq["coarse"], sq._pq["coarse"])
    _, sq_lists = ops.ivfsq_export(sq._pq["codes"], sq._pq["slot_rows"], sq._pq["tile_lists"], len(x))
    assert torch.equal(a._flat_list_ids(a._pq, len(x)), sq_lists)
    assert torch.equal(a._pq["slot_rows"], sq._pq["slot_rows"]) and torch.equal(a._pq["tile_lists"], sq._pq["tile_lists"])
    one = _index(x[:1], "ivfflat")
    one.train_index()
    docs, scores = one.search_knn(torch.from_numpy(x[:2]).cuda(), 1)
    assert _ids(docs) == [[0], [0]]


def test_flat_type_is_the_flat_index():
    import synth
    from atlas_b200.index import DistributedIndex

    rng = np.random.default_rng(59)
    x = _clustered(rng, 9001)
    q = torch.from_numpy(_clustered(rng, 33)).cuda()
    flat = DistributedIndex()
    flat.init_embeddings(synth.make_passages(len(x)))
    flat.embeddings[:, :] = torch.from_numpy(x).T.cuda()
    index = _index(x, "flat")
    index.train_index()
    assert index._pq["n_list"] == 1 and index._pq["coarse"] is None
    assert index._pq["slot_rows"].tolist() == list(range(len(x))) + [-1] * (64 * ((len(x) + 63) // 64) - len(x))
    for k in (1, 40, 500):
        assert index.search_knn(q, k) == flat.search_knn(q, k), k
    with tempfile.TemporaryDirectory() as tmp:
        index.save_index(tmp, 1)
        from atlas_b200.index import DistributedFAISSIndex

        index2 = DistributedFAISSIndex("flat")
        index2.load_index(tmp, 1)
        assert index2.search_knn(q, 40) == flat.search_knn(q, 40)


def test_atlas_retrieve_passes_faiss_nprobe():
    from atlas_b200.atlas import Atlas

    rng = np.random.default_rng(61)
    index = _index(_clustered(rng, 5000), "ivfflat")
    index.train_index()
    emb = torch.from_numpy(_clustered(rng, 3)).cuda()

    class Retriever:
        def eval(self):
            return self

        def __call__(self, ids, mask, is_passages=False):
            return emb

    fake = types.SimpleNamespace(opt=types.SimpleNamespace(faiss_nprobe=3, faiss_refine_factor=2), retriever=Retriever(),
                                 training=False)
    passages, scores, _ = Atlas._retrieve(fake, index, 10, ["a", "b", "c"], None, None)
    assert index.nprobe == 3 and index.refine_factor == 2
    want = index.search_knn(emb, 10)
    assert (passages, scores) == want
    index.refine_factor = 1
    assert index.search_knn(emb, 10) == want
