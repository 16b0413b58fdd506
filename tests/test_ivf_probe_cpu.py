"""CPU checks of the probed IVF search (`nprobe`): the probe rule of oracle/ivf_probe_oracle.py on hand cases, the
validation of `DistributedFAISSIndex.nprobe`, the Atlas option plumbing with stub indexes, and the C ABI declarations."""
import os
import re
import types

import numpy as np
import pytest

import ivf_probe_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sets(probed):
    return [sorted(np.flatnonzero(r).tolist()) for r in probed]


def test_ties_go_to_the_lower_list_id():
    T = np.array([[1.0, 3.0, 3.0, 2.0, 3.0]], np.float32)
    sizes = [10, 10, 10, 10, 10]
    assert _sets(ivf_probe_oracle.probe_lists(T, 1, sizes, 1)) == [[1]]
    assert _sets(ivf_probe_oracle.probe_lists(T, 2, sizes, 1)) == [[1, 2]]
    assert _sets(ivf_probe_oracle.probe_lists(T, 3, sizes, 1)) == [[1, 2, 4]]
    assert _sets(ivf_probe_oracle.probe_lists(T, 4, sizes, 1)) == [[1, 2, 3, 4]]
    # -0 and +0 are equal coarse terms
    T0 = np.array([[-0.0, 0.0, -1.0]], np.float32)
    assert _sets(ivf_probe_oracle.probe_lists(T0, 1, [1, 1, 1], 1)) == [[0]]


def test_empty_lists_count_toward_nprobe():
    T = np.array([[5.0, 4.0, 3.0, 2.0]], np.float32)
    sizes = [0, 7, 0, 9]
    assert _sets(ivf_probe_oracle.probe_lists(T, 2, sizes, 3)) == [[0, 1]]
    assert _sets(ivf_probe_oracle.probe_lists(T, 3, sizes, 3)) == [[0, 1, 2]]


def test_extension_until_k_rows():
    T = np.array([[5.0, 4.0, 3.0, 2.0], [2.0, 3.0, 4.0, 5.0]], np.float32)
    sizes = [3, 0, 4, 20]
    # nprobe 1 holds 3 rows (query 0) / 20 rows (query 1); k = 5 extends query 0 by the next lists, an empty one included
    assert _sets(ivf_probe_oracle.probe_lists(T, 1, sizes, 5)) == [[0, 1, 2], [3]]
    assert _sets(ivf_probe_oracle.probe_lists(T, 1, sizes, 27)) == [[0, 1, 2, 3], [0, 1, 2, 3]]
    with pytest.raises(ValueError):
        ivf_probe_oracle.probe_lists(T, 1, sizes, 28)


def test_nprobe_at_least_n_list_gives_every_list():
    rng = np.random.default_rng(1)
    T = rng.standard_normal((6, 9)).astype(np.float32)
    for nprobe in (9, 10, 1000):
        assert ivf_probe_oracle.probe_lists(T, nprobe, np.ones(9), 1).all()


def test_probe_sets_nest_in_nprobe():
    rng = np.random.default_rng(2)
    T = rng.integers(-3, 4, (20, 30)).astype(np.float32)      # many ties
    sizes = rng.integers(0, 5, 30)
    prev = None
    for nprobe in range(1, 32):
        cur = ivf_probe_oracle.probe_lists(T, nprobe, sizes, 6)
        assert (cur.sum(1) >= min(nprobe, 30)).all()
        if prev is not None:
            assert (cur >= prev).all()
        prev = cur


def test_restricted_topk_keeps_probed_rows_only():
    scores = np.array([[5, 4, 3, 2, 1, 0]], np.float16)
    lists = np.array([0, 1, 0, 1, 2, 2])
    probed = np.array([[False, True, True]])
    v, i = ivf_probe_oracle.restricted_topk(scores, lists, probed, 3)
    assert i.tolist() == [[1, 3, 4]] and v.astype(np.float32).tolist() == [[4, 2, 1]]


# ------------------------------------------------------------------ module validation (no GPU needed)
def _stub(index_type, nprobe=None):
    from atlas_b200.index import DistributedFAISSIndex

    index = DistributedFAISSIndex.__new__(DistributedFAISSIndex)
    index.index_type = index_type
    index.nprobe = nprobe
    index.refine_factor = 1
    return index


@pytest.mark.parametrize("bad", [0, -1, True, False, 2.0, "4", [4]])
def test_nprobe_validation(bad):
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.index import DistributedFAISSIndex

    with pytest.raises(AtlasB200Error):
        DistributedFAISSIndex("ivfpq", 16, nprobe=bad)
    with pytest.raises(AtlasB200Error):
        _stub("ivfsq", bad)._local_search(None, 1)


def test_nprobe_valid_values_and_pq():
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.index import DistributedFAISSIndex

    for kind in ("ivfpq", "ivfsq"):
        for ok in (None, 1, 7, 10 ** 9):
            assert _stub(kind, ok)._nprobe() == ok
    assert _stub("pq", None)._nprobe() is None
    with pytest.raises(AtlasB200Error):
        _stub("pq", 4)._nprobe()
    with pytest.raises(AtlasB200Error):
        DistributedFAISSIndex("pq", 16, nprobe=4)


# ------------------------------------------------------------------ Atlas option plumbing
def _retrieve(index, opt):
    import torch

    from atlas_b200.atlas import Atlas

    class Retriever:
        def eval(self):
            return self

        def __call__(self, ids, mask, is_passages=False):
            return torch.zeros((2, 768))

    fake = types.SimpleNamespace(opt=opt, retriever=Retriever(), training=False)
    return Atlas._retrieve(fake, index, 3, ["a", "b"], None, None)


def test_atlas_sets_nprobe_on_faiss_indexes_only():
    from atlas_b200.index import DistributedFAISSIndex, DistributedIndex

    seen = []

    class FaissStub(DistributedFAISSIndex):
        def __init__(self):
            self.nprobe = 99

        def search_knn(self, q, k):
            seen.append(self.nprobe)
            return [[]] * 2, [[]] * 2

    class FlatStub(DistributedIndex):
        def __init__(self):
            pass

        def search_knn(self, q, k):
            seen.append(getattr(self, "nprobe", "unset"))
            return [[]] * 2, [[]] * 2

    _retrieve(FaissStub(), types.SimpleNamespace(faiss_nprobe=8))
    _retrieve(FaissStub(), types.SimpleNamespace(faiss_nprobe=None))
    _retrieve(FaissStub(), types.SimpleNamespace())
    _retrieve(FlatStub(), types.SimpleNamespace(faiss_nprobe=8))
    assert seen == [8, None, None, "unset"]


# ------------------------------------------------------------------ C ABI declarations
NEW = ["atlas_b200_pq_topk_probed", "atlas_b200_pq_topk_probed_exhaustive", "atlas_b200_ivfsq_topk_probed",
       "atlas_b200_ivfsq_topk_probed_exhaustive"]


def test_header_and_argtypes():
    from atlas_b200 import _lib

    header = open(os.path.join(ROOT, "include", "atlas_b200.h")).read()
    assert "#define ATLAS_B200_PQ_OP_SEARCH_PROBED 3" in header
    counts = {}
    for name in NEW:
        m = re.search(r"\b" + name + r"\(([^)]*)\)", header)
        assert m, name
        counts[name] = len(m.group(1).split(","))
        assert name in _lib.EXPORTED_SYMBOLS
    # the existing entry point plus list tables and nprobe
    assert counts["atlas_b200_pq_topk_probed"] == 18 + 3
    assert counts["atlas_b200_pq_topk_probed_exhaustive"] == 17 + 3
    assert counts["atlas_b200_ivfsq_topk_probed"] == 20 + 3
    assert counts["atlas_b200_ivfsq_topk_probed_exhaustive"] == 19 + 3
    src = open(os.path.join(ROOT, "atlas_b200", "_lib.py")).read()
    for name in NEW:
        m = re.search(r"L\." + name + r"\.argtypes = \[([^\]]*)\]", src)
        assert m and len(m.group(1).split(",")) == counts[name], name
