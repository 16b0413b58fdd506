"""GPU checks of the probed IVF search (`nprobe`, csrc/ivf_probe.cu with the ivfpq and ivfsq scans) against the numpy
restatement oracle/ivf_probe_oracle.py: exact grid states bit for bit, Gaussian states within the indexes' tolerances,
the no-op values, batch independence, monotonicity in nprobe, the extension on small shards, the sampled and exhaustive
paths, CUDA-graph capture (no host synchronisation) and the module."""
import os
import tempfile
import types

import numpy as np
import pytest
import torch

import ivf_probe_oracle
import pq_oracle
import sq_oracle

pytestmark = pytest.mark.gpu

DIM = 768
M_PQ = 16
KINDS = ["ivfpq", "ivfsq"]


def _ulp16(v):
    a = np.abs(np.asarray(v, dtype=np.float32)).astype(np.float16)
    return (np.nextafter(a, np.float16(np.inf)) - a).astype(np.float32)


# ------------------------------------------------------------------ hand-built states
def _state(kind, rng, sizes, grid=False, scale=0.05):
    """list l holds sizes[l] rows in random row order; random codes; small-integer parameters when grid (exact sums)."""
    sizes = list(sizes)
    n, n_list = sum(sizes), len(sizes)
    lists = rng.permutation(np.repeat(np.arange(n_list), sizes)).astype(np.int64)
    st = dict(kind=kind, lists=lists, n_list=n_list, n=n)
    if grid:
        st["coarse"] = rng.integers(-2, 3, (n_list, DIM)).astype(np.float32)
    else:
        st["coarse"] = (rng.standard_normal((n_list, DIM)) * scale).astype(np.float32)
    if kind == "ivfsq":
        st["codes"] = rng.integers(0, 16, (n, DIM)).astype(np.uint8)
        if grid:
            st["vmin"] = rng.integers(-4, 4, DIM).astype(np.float32) / 4
            st["vdiff"] = np.full(DIM, 15 / 8, np.float32)
        else:
            st["vmin"] = (-rng.uniform(0.5, 1.5, DIM) * scale).astype(np.float32)
            st["vdiff"] = (rng.uniform(1.0, 3.0, DIM) * scale).astype(np.float32)
    else:
        st["codes"] = rng.integers(0, 256, (n, M_PQ), dtype=np.uint8)
        if grid:
            st["codebooks"] = rng.integers(-2, 3, (M_PQ, 256, DIM // M_PQ)).astype(np.float32)
        else:
            st["codebooks"] = (rng.standard_normal((M_PQ, 256, DIM // M_PQ)) * scale).astype(np.float32)
    return st


def _grid_queries(rng, nq):
    q = np.zeros((nq, DIM), np.float16)
    for r in range(nq):
        q[r, rng.choice(DIM, 6, replace=False)] = rng.integers(-2, 3, 6)
    return q


def _device(st):
    from atlas_b200 import ops

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d = dict(kind=st["kind"], n=st["n"], n_list=st["n_list"], coarse=t(st["coarse"]))
    if st["kind"] == "ivfsq":
        d["codes"], d["slot_rows"], d["tile_lists"] = ops.ivfsq_import(t(sq_oracle.pack(st["codes"])),
                                                                       t(st["lists"].astype(np.int32)), st["n_list"])
        d["vmin"], d["vdiff"] = t(st["vmin"]), t(st["vdiff"])
        d["list_tile_off"], d["list_rows"] = ops.ivfsq_list_tables(d["slot_rows"], d["tile_lists"], st["n_list"])
    else:
        d["codes"], d["codebooks"] = t(st["codes"]), t(st["codebooks"])
        d["list_ids"] = t(st["lists"].astype(np.uint16))
        d["list_order"], d["list_offsets"] = ops.ivfpq_list_tables(d["list_ids"], st["n_list"])
    return d


def _search_dev(d, q, k, nprobe=None, exhaustive=False, id_base=0, id_stride=1, tables=True, workspace=None):
    """Device tensors (scores, ids, status) of one ops-level search."""
    from atlas_b200 import ops

    qd = q if torch.is_tensor(q) else torch.from_numpy(q).cuda()
    if d["kind"] == "ivfsq":
        tb = dict(list_tile_off=d["list_tile_off"], list_rows=d["list_rows"]) if tables else {}
        return ops.ivfsq_topk(d["codes"], d["slot_rows"], d["tile_lists"], d["n"], d["coarse"], d["vmin"], d["vdiff"], qd,
                              k, id_base, id_stride, workspace, exhaustive=exhaustive, nprobe=nprobe, **tb)
    tb = dict(list_order=d["list_order"], list_offsets=d["list_offsets"]) if tables else {}
    return ops.pq_topk(d["codes"], d["list_ids"], d["codebooks"], d["coarse"], qd, k, id_base, id_stride, workspace,
                       exhaustive=exhaustive, nprobe=nprobe, **tb)


def _search(d, q, k, nprobe=None, exhaustive=False, id_base=0, id_stride=1, retry=True):
    s, i, stat = _search_dev(d, q, k, nprobe, exhaustive, id_base, id_stride)
    stat = int(stat.item())
    if stat and retry and not exhaustive:
        s, i, _ = _search_dev(d, q, k, nprobe, True, id_base, id_stride)
    return s.cpu().numpy(), i.cpu().numpy(), stat


def _oracle_scores(st, q):
    if st["kind"] == "ivfsq":
        return sq_oracle.contract_scores(q, st["codes"], st["vmin"], st["vdiff"], st["coarse"], st["lists"])
    return pq_oracle.adc_scores(q, st["codes"], st["codebooks"], st["coarse"], st["lists"])


def _oracle_T(st, q):
    if st["kind"] == "ivfsq":
        return ivf_probe_oracle.sq_coarse_terms(q, st["coarse"])
    return ivf_probe_oracle.pq_coarse_terms(q, st["coarse"])


def _sizes(st):
    return np.bincount(st["lists"], minlength=st["n_list"])


_GRID = {}


def _grid_state(kind):
    if kind not in _GRID:
        rng = np.random.default_rng(5 if kind == "ivfsq" else 6)
        n, n_list = 20000, 141
        st = _state(kind, rng, np.bincount(rng.integers(0, n_list, n), minlength=n_list), grid=True)
        _GRID[kind] = (st, _device(st))
    return _GRID[kind]


# ------------------------------------------------------------------ 1. exact grid states
@pytest.mark.parametrize("nq", [1, 3, 40, 129, 256, 300])
@pytest.mark.parametrize("nprobe", [1, 2, 7, -1])
@pytest.mark.parametrize("kind", KINDS)
def test_grid_bit_exact(kind, nprobe, nq):
    """Small-integer coarse terms, codes and sparse queries: T and every score are exact and full of ties, so scores and
    canonical ids match the oracle over the probed rows bitwise; nprobe -1 stands for n_list - 1."""
    st, d = _grid_state(kind)
    nprobe = st["n_list"] - 1 if nprobe < 0 else nprobe
    rng = np.random.default_rng(100 * nq + nprobe)
    q = _grid_queries(rng, nq)
    scores = _oracle_scores(st, q)
    probed = ivf_probe_oracle.probe_lists(_oracle_T(st, q), nprobe, _sizes(st), 1024)
    for k in (1, 40, 1024):
        pk = probed if k == 1024 else ivf_probe_oracle.probe_lists(_oracle_T(st, q), nprobe, _sizes(st), k)
        want_v, want_i = ivf_probe_oracle.restricted_topk(scores, st["lists"], pk, k)
        s, ids, _ = _search(d, q, k, nprobe, id_base=7, id_stride=3)
        assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16)), k
        assert np.array_equal(ids, 7 + 3 * want_i), k


# ------------------------------------------------------------------ 2. Gaussian states
@pytest.mark.parametrize("nprobe", [1, 8])
@pytest.mark.parametrize("kind", KINDS)
def test_gaussian_parity(kind, nprobe):
    """Parity within one fp16 ulp against the oracle restricted to its probe sets; queries whose last probed and first
    unprobed coarse scores lie within 1e-5 of the largest |T| (where fp32 summation order could swap them) are skipped,
    and most queries must be kept."""
    rng = np.random.default_rng(17 + nprobe)
    n, n_list, nq, k = 60000, 244, 64, 40
    st = _state(kind, rng, np.bincount(rng.integers(0, n_list, n), minlength=n_list))
    q = rng.standard_normal((nq, DIM)).astype(np.float16)
    d = _device(st)
    s, ids, _ = _search(d, q, k, nprobe)
    T = _oracle_T(st, q)
    probed = ivf_probe_oracle.probe_lists(T, nprobe, _sizes(st), k)
    ref = _oracle_scores(st, q).astype(np.float32)
    kept = 0
    for r in range(nq):
        ts = np.sort(T[r])[::-1]
        p = int(probed[r].sum())
        margin = 1e-5 * float(np.abs(T[r]).max())
        if p < n_list and ts[p - 1] - ts[p] <= margin:
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


# ------------------------------------------------------------------ 3. no-op values
@pytest.mark.parametrize("kind", KINDS)
def test_noop_values_are_the_full_scan(kind):
    rng = np.random.default_rng(23)
    st = _state(kind, rng, np.bincount(rng.integers(0, 90, 8000), minlength=90))
    d = _device(st)
    q = rng.standard_normal((37, DIM)).astype(np.float16)
    for k in (1, 40):
        base = [t.cpu().numpy() for t in _search_dev(d, q, k)]
        for nprobe in (None, st["n_list"], st["n_list"] + 5):
            got = [t.cpu().numpy() for t in _search_dev(d, q, k, nprobe)]
            assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(base, got)), nprobe


# ------------------------------------------------------------------ 4. batch independence
@pytest.mark.parametrize("kind", KINDS)
def test_batch_independence(kind):
    rng = np.random.default_rng(29)
    st = _state(kind, rng, np.bincount(rng.integers(0, 200, 40000), minlength=200))
    d = _device(st)
    q = rng.standard_normal((300, DIM)).astype(np.float16)
    s, ids, _ = _search(d, q, 40, 4)
    for r in list(range(0, 300, 37)) + [129, 255, 256, 299]:
        s1, i1, _ = _search(d, q[r:r + 1], 40, 4)
        assert np.array_equal(s1[0].view(np.uint16), s[r].view(np.uint16)) and np.array_equal(i1[0], ids[r]), r
    s2, i2, _ = _search(d, q[100:], 40, 4)
    assert np.array_equal(s2.view(np.uint16), s[100:].view(np.uint16)) and np.array_equal(i2, ids[100:])


# ------------------------------------------------------------------ 5. monotonicity
@pytest.mark.parametrize("kind", KINDS)
def test_monotone_in_nprobe(kind):
    rng = np.random.default_rng(31)
    st = _state(kind, rng, np.bincount(rng.integers(0, 200, 40000), minlength=200))
    d = _device(st)
    q = rng.standard_normal((50, DIM)).astype(np.float16)
    prev = None
    for nprobe in (1, 4, 16, st["n_list"]):
        s, _, _ = _search(d, q, 40, nprobe)
        s = s.astype(np.float32)
        if prev is not None:
            assert (s >= prev).all(), nprobe
        prev = s


# ------------------------------------------------------------------ 6. extension on small shards
@pytest.mark.parametrize("kind", KINDS)
def test_extension_on_a_small_shard(kind):
    """About 300 rows in 17 lists, nprobe = 1, k = 40: the best list alone holds fewer than 40 rows, the probe set is
    extended and 40 valid ids come back, equal to the oracle's."""
    rng = np.random.default_rng(37)
    st = _state(kind, rng, np.bincount(rng.integers(0, 17, 300), minlength=17), grid=True)
    d = _device(st)
    q = _grid_queries(rng, 9)
    s, ids, _ = _search(d, q, 40, 1)
    probed = ivf_probe_oracle.probe_lists(_oracle_T(st, q), 1, _sizes(st), 40)
    assert (probed.sum(1) > 1).all()
    want_v, want_i = ivf_probe_oracle.restricted_topk(_oracle_scores(st, q), st["lists"], probed, 40)
    assert (ids >= 0).all()
    assert np.array_equal(s.view(np.uint16), want_v.view(np.uint16)) and np.array_equal(ids, want_i)


# ------------------------------------------------------------------ 7. sampled and exhaustive paths
@pytest.mark.parametrize("kind", KINDS)
def test_large_probe_sets_do_not_overflow(kind):
    """256 queries, each probing about 45 k rows - more than a query's candidate list holds (32768 here) - and the probe
    sets of the block covering nearly every list: every query's sampled bound comes from its own probed rows, so the
    fast path does not overflow, and it agrees with the exhaustive path."""
    rng = np.random.default_rng(45)
    n, n_list, k, nprobe = 200000, 447, 40, 100
    st = _state(kind, rng, np.bincount(rng.integers(0, n_list, n), minlength=n_list))
    d = _device(st)
    q = rng.standard_normal((256, DIM)).astype(np.float16)
    probed = ivf_probe_oracle.probe_lists(_oracle_T(st, q), nprobe, _sizes(st), k)
    assert (probed.astype(np.int64) @ _sizes(st) > 32768).all()
    s1, i1, stat = _search(d, q, k, nprobe, retry=False)
    assert stat == 0
    s2, i2, _ = _search(d, q, k, nprobe, exhaustive=True)
    assert np.array_equal(s1.view(np.uint16), s2.view(np.uint16)) and np.array_equal(i1, i2)


@pytest.mark.parametrize("kind", KINDS)
def test_sampled_and_exhaustive_agree(kind):
    rng = np.random.default_rng(41)
    st = _state(kind, rng, np.bincount(rng.integers(0, 447, 200000), minlength=447))
    d = _device(st)
    q = rng.standard_normal((100, DIM)).astype(np.float16)
    for nprobe in (3, 40):
        s1, i1, stat = _search(d, q, 40, nprobe, retry=False)
        s2, i2, _ = _search(d, q, 40, nprobe, exhaustive=True)
        assert stat == 0
        assert np.array_equal(s1.view(np.uint16), s2.view(np.uint16)) and np.array_equal(i1, i2), nprobe


@pytest.mark.parametrize("kind", KINDS)
def test_all_equal_scores_raise_status_and_exhaustive_returns_lowest_probed_ids(kind):
    """Every row of every list scores the same: the probe sets are the lowest list ids (ties by list id), their 25 lists
    hold more rows than the candidate lists, so status is set, and the exhaustive path returns the lowest row ids among
    the rows of the probed lists."""
    rng = np.random.default_rng(43)
    n, n_list, k = 100000, 50, 40
    st = _state(kind, rng, np.bincount(rng.integers(0, n_list, n), minlength=n_list))
    if kind == "ivfsq":
        st["vdiff"][:] = 0
    else:
        st["codebooks"][:] = 0
    st["coarse"][:] = 0
    d = _device(st)
    q = rng.standard_normal((3, DIM)).astype(np.float16)
    _, _, stat = _search(d, q, k, 25, retry=False)
    assert stat == 1
    s, ids, _ = _search(d, q, k, 25, exhaustive=True)
    probed = ivf_probe_oracle.probe_lists(_oracle_T(st, q), 25, _sizes(st), k)
    assert (probed[:, :25].all(1) & ~probed[:, 25:].any(1)).all()
    for r in range(3):
        rows = np.flatnonzero(probed[r][st["lists"]])
        assert np.array_equal(ids[r], rows[:k]), r
        assert (s[r] == s[r, 0]).all()


# ------------------------------------------------------------------ 8. CUDA graph capture (no host synchronisation)
@pytest.mark.parametrize("kind", KINDS)
def test_probed_search_replays_in_a_cuda_graph(kind):
    from atlas_b200 import ops

    rng = np.random.default_rng(47)
    st = _state(kind, rng, np.bincount(rng.integers(0, 200, 40000), minlength=200))
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


# ------------------------------------------------------------------ 9. the module
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


@pytest.mark.parametrize("kind,code_size", [("ivfpq", 16), ("ivfsq", None)])
def test_module_search_refine_save_load_and_tables(kind, code_size):
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.index import DistributedFAISSIndex

    rng = np.random.default_rng(53)
    n, k = 30000, 40
    x = _clustered(rng, n)
    q = torch.from_numpy(_clustered(rng, 20)).cuda()
    index = _index(x, kind, code_size, nprobe=4)
    index.train_index()
    p = index._pq
    clean = tempfile.TemporaryDirectory()
    index.save_index(clean.name, 1)       # before any probed search: no list tables exist yet
    table = "list_tile_off" if kind == "ivfsq" else "list_order"
    assert table not in p

    docs, scores = index.search_knn(q, k)
    assert table in p
    if kind == "ivfsq":
        s, i, _ = ops.ivfsq_topk(p["codes"], p["slot_rows"], p["tile_lists"], n, p["coarse"], p["vmin"], p["vdiff"], q, k,
                                 nprobe=4)
    else:
        s, i, _ = ops.pq_topk(p["codes"], p["list_ids"], p["codebooks"], p["coarse"], q, k, nprobe=4)
    assert _ids(docs) == i.cpu().tolist()
    assert np.array_equal(np.array(scores, np.float32), s.float().cpu().numpy())

    # refinement composes: the probed search supplies the k' candidates
    index.refine_factor = 3
    docs_r, scores_r = index.search_knn(q, k)
    if kind == "ivfsq":
        _, cand, _ = ops.ivfsq_topk(p["codes"], p["slot_rows"], p["tile_lists"], n, p["coarse"], p["vmin"], p["vdiff"], q,
                                    3 * k, nprobe=4)
    else:
        _, cand, _ = ops.pq_topk(p["codes"], p["list_ids"], p["codebooks"], p["coarse"], q, 3 * k, nprobe=4)
    rs, ri = ops.pq_refine_topk(index._bank, q, cand, k)
    assert _ids(docs_r) == ri.cpu().tolist()
    assert np.array_equal(np.array(scores_r, np.float32), rs.float().cpu().numpy())
    index.refine_factor = 1

    # neither nprobe nor the list tables (present now) reach the index file: files saved with nprobe = 4 after probed
    # searches and with nprobe = None are byte-identical to the files saved before any probed search
    with clean, tempfile.TemporaryDirectory() as a, tempfile.TemporaryDirectory() as b:
        assert table in p
        index.save_index(a, 1)
        index.nprobe = None
        index.save_index(b, 1)
        names = sorted(os.listdir(clean.name))
        for d in (a, b):
            assert names == sorted(os.listdir(d))
            for f in names:
                with open(os.path.join(clean.name, f), "rb") as fc, open(os.path.join(d, f), "rb") as fd:
                    assert fc.read() == fd.read(), f
        index2 = DistributedFAISSIndex(kind, code_size, nprobe=4)
        index2.load_index(a, 1)
        assert index2.search_knn(q, k) == (docs, scores)

    # the tables go with the trained index
    index.train_index()
    assert table not in index._pq
    index.nprobe = 4
    index.search_knn(q, k)
    assert table in index._pq
    for bad in (0, True, 2.0):
        index.nprobe = bad
        with pytest.raises(AtlasB200Error):
            index.search_knn(q, k)
    index.nprobe = 4
    index.mark_stale()
    assert index._pq is None


def test_pq_with_nprobe_raises():
    from atlas_b200._lib import AtlasB200Error

    rng = np.random.default_rng(59)
    with pytest.raises(AtlasB200Error):
        _index(_clustered(rng, 1000), "pq", 16, nprobe=2)
    index = _index(_clustered(rng, 1000), "pq", 16)
    index.train_index()
    index.nprobe = 2
    with pytest.raises(AtlasB200Error):
        index.search_knn(torch.from_numpy(_clustered(rng, 2)).cuda(), 5)


def test_atlas_retrieve_passes_faiss_nprobe():
    from atlas_b200.atlas import Atlas

    rng = np.random.default_rng(61)
    index = _index(_clustered(rng, 5000), "ivfsq")
    index.train_index()
    emb = torch.from_numpy(_clustered(rng, 3)).cuda()

    class Retriever:
        def eval(self):
            return self

        def __call__(self, ids, mask, is_passages=False):
            return emb

    fake = types.SimpleNamespace(opt=types.SimpleNamespace(faiss_nprobe=3), retriever=Retriever(), training=False)
    passages, scores, _ = Atlas._retrieve(fake, index, 10, ["a", "b", "c"], None, None)
    assert index.nprobe == 3
    want = index.search_knn(emb, 10)
    assert (passages, scores) == want
