"""CPU checks of the IVF-Flat passage index (`DistributedFAISSIndex("ivfflat")` / ("flat"), csrc/ivfflat.cu): the numpy
restatement of its probed search on hand cases, and the constructor contract.

`flat_probed_topk` below is the restatement tests/test_ivfflat_gpu.py checks the device against.  It composes the
existing oracles and states no rule of its own: the flat scores of oracle/mips_oracle.py, the coarse terms T of the ivfsq
index (oracle/ivf_probe_oracle.sq_coarse_terms), the probe sets P(q) of ivf_probe_oracle.probe_lists and the canonical
top-k over the probed rows of ivf_probe_oracle.restricted_topk."""
import numpy as np
import pytest
import torch

import ivf_probe_oracle
import mips_oracle


def flat_probed_topk(queries, rows, coarse, lists, nprobe, k):
    """(scores fp16 [nq, k], ids [nq, k], probed bool [nq, n_list]) of the IVF-Flat search of fp16 `rows` [n, 768] in
    lists `lists` [n] with coarse centroids `coarse` [n_list, 768]; nprobe None scans every list."""
    lists = np.asarray(lists, np.int64)
    n_list = np.asarray(coarse).shape[0]
    T = ivf_probe_oracle.sq_coarse_terms(queries, coarse)
    if nprobe is None:
        probed = np.ones((T.shape[0], n_list), bool)
    else:
        probed = ivf_probe_oracle.probe_lists(T, nprobe, np.bincount(lists, minlength=n_list), k)
    s = mips_oracle.scores_fp16(queries, np.asarray(rows, np.float16))
    v, i = ivf_probe_oracle.restricted_topk(s, lists, probed, k)
    return v, i, probed


DIM = 768


def _unit(d, v=1.0):
    x = np.zeros(DIM, np.float32)
    x[d] = v
    return x


def test_best_row_in_an_unprobed_list_is_not_returned():
    # list 0's centroid points along dim 0 (the query's), list 1's away from it; the best row sits in list 1
    coarse = np.stack([_unit(0), _unit(0, -1.0)])
    rows = np.stack([_unit(0, 1.0), _unit(0, 2.0), _unit(0, 8.0), _unit(0, 0.5)]).astype(np.float16)
    lists = np.array([0, 0, 1, 1])
    q = _unit(0)[None].astype(np.float16)
    v, i, probed = flat_probed_topk(q, rows, coarse, lists, 1, 2)
    assert probed.tolist() == [[True, False]]
    assert i.tolist() == [[1, 0]] and v.astype(np.float32).tolist() == [[2.0, 1.0]]
    v, i, _ = flat_probed_topk(q, rows, coarse, lists, None, 2)
    assert i.tolist() == [[2, 1]]


def test_probe_set_is_extended_when_the_probed_lists_hold_fewer_than_k_rows():
    coarse = np.stack([_unit(0, 3.0), _unit(0, 2.0), _unit(0, 1.0)])
    rows = np.stack([_unit(0, float(r + 1)) for r in range(6)]).astype(np.float16)
    lists = np.array([2, 0, 1, 1, 2, 2])          # list 0 holds one row
    q = _unit(0)[None].astype(np.float16)
    v, i, probed = flat_probed_topk(q, rows, coarse, lists, 1, 3)
    assert probed.tolist() == [[True, True, False]]
    assert i.tolist() == [[3, 2, 1]]
    v, i, probed = flat_probed_topk(q, rows, coarse, lists, 1, 4)
    assert probed.tolist() == [[True, True, True]]
    assert i.tolist() == [[5, 4, 3, 2]]


def test_empty_lists_count_toward_nprobe_and_return_nothing():
    coarse = np.stack([_unit(0, 5.0), _unit(0, 4.0), _unit(0, 3.0)])
    rows = np.stack([_unit(0, 1.0), _unit(0, 7.0), _unit(0, 2.0)]).astype(np.float16)
    lists = np.array([1, 2, 1])                    # list 0 is empty
    q = _unit(0)[None].astype(np.float16)
    v, i, probed = flat_probed_topk(q, rows, coarse, lists, 2, 2)
    assert probed.tolist() == [[True, True, False]]
    assert i.tolist() == [[2, 0]]


def test_ties_are_broken_by_row_id():
    rng = np.random.default_rng(3)
    coarse = rng.integers(-1, 2, (4, DIM)).astype(np.float32)
    rows = np.zeros((40, DIM), np.float16)
    rows[:, 0] = rng.integers(0, 3, 40)            # three score values, many ties
    lists = rng.integers(0, 4, 40)
    q = _unit(0)[None].astype(np.float16)
    v, i, probed = flat_probed_topk(q, rows, coarse, lists, 2, 10)
    keep = np.flatnonzero(probed[0][lists])
    order = sorted(keep.tolist(), key=lambda r: (-float(rows[r, 0]), r))[:10]
    assert i[0].tolist() == order


def test_every_list_is_the_flat_oracle():
    rng = np.random.default_rng(4)
    n, n_list, nq, k = 500, 9, 7, 25
    rows = rng.standard_normal((n, DIM)).astype(np.float16)
    coarse = rng.standard_normal((n_list, DIM)).astype(np.float32)
    lists = rng.integers(0, n_list, n)
    q = rng.standard_normal((nq, DIM)).astype(np.float16)
    want_v, want_i = mips_oracle.canonical_topk(mips_oracle.scores_fp16(q, rows), k)
    for nprobe in (None, n_list, n_list + 3):
        v, i, probed = flat_probed_topk(q, rows, coarse, lists, nprobe, k)
        assert probed.all()
        assert np.array_equal(v.view(np.uint16), want_v.view(np.uint16)) and np.array_equal(i, want_i), nprobe


def test_constructor_contract():
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.index import DistributedFAISSIndex

    assert {"ivfflat", "flat"} <= set(DistributedFAISSIndex.SUPPORTED_TYPES)
    for kind in ("ivfflat", "flat"):
        for code_size in (4, 8, 16, 64, True):
            with pytest.raises(AtlasB200Error, match="--index_mode flat"):
                DistributedFAISSIndex(kind, code_size)
        for bad in (0, -1, True, False, 2.0, "4"):
            with pytest.raises(AtlasB200Error, match="nprobe"):
                DistributedFAISSIndex(kind, None, nprobe=bad)
    with pytest.raises(AtlasB200Error, match="flat has none"):
        DistributedFAISSIndex("flat", None, nprobe=4)
    if not torch.cuda.is_available():
        for kind in ("ivfflat", "flat"):
            with pytest.raises(AtlasB200Error, match="CUDA"):
                DistributedFAISSIndex(kind)
            with pytest.raises(AtlasB200Error, match="CUDA"):
                DistributedFAISSIndex(kind, None, nprobe=None if kind == "flat" else 4)
