"""CPU checks of the IVF-SQ rules (oracle/sq_oracle.py) on hand cases whose answers are known by construction, the
contract-vs-faiss error bound, the slot permutation and the constructor of DistributedFAISSIndex("ivfsq")."""
import numpy as np
import pytest
import torch

import sq_oracle

DIM = 768


def test_range_endpoints_and_clamping():
    vmin = np.array([-1.0, 0.5, 2.0, -3.0], np.float32)
    vdiff = np.array([2.0, 1.0, 0.0, 0.25], np.float32)
    r = np.stack([vmin, vmin + vdiff, vmin - 5, vmin + vdiff + 5]).astype(np.float32)
    c = sq_oracle.quantize(r, vmin, vdiff)
    assert c[0].tolist() == [0, 0, 0, 0]                     # x = vmin -> 0
    assert c[1].tolist() == [15, 15, 0, 15]                  # x = vmax -> 15; vdiff = 0 -> 0
    assert c[2].tolist() == [0, 0, 0, 0]                     # below the range: clamped to 0
    assert c[3].tolist() == [15, 15, 0, 15]                  # above: clamped to 15


def test_train_range_is_min_and_max_minus_min():
    r = np.array([[1.0, -2.0], [3.0, -1.0], [2.0, -4.0]], np.float32)
    vmin, vdiff = sq_oracle.train_range(r)
    assert vmin.tolist() == [1.0, -4.0] and vdiff.tolist() == [2.0, 3.0]
    assert vmin.dtype == np.float32 and vdiff.dtype == np.float32


def test_nibble_order():
    codes = np.array([[1, 2, 3, 4, 15, 0]], np.uint8)
    packed = sq_oracle.pack(codes)
    assert packed.tolist() == [[0x21, 0x43, 0x0F]]
    assert np.array_equal(sq_oracle.unpack(packed), codes)


def test_code_product_in_double():
    """faiss multiplies the float xi by the double 15.0.  For the multiplier 15 an fp32 product never rounds up onto the
    next integer: the fp32 xi just below m / 15 leaves 15 xi at least half an fp32 ulp of the product below m.  The fp32
    values around every boundary show it; the oracle, like the encode kernel, takes the product in double anyway."""
    xs = []
    for m in range(1, 16):
        x = np.float32(m / 15.0)
        for _ in range(256):
            xs.append(x)
            x = np.nextafter(x, np.float32(0))
        x = np.float32(m / 15.0)
        for _ in range(256):
            xs.append(x)
            x = np.nextafter(x, np.float32(1))
    xs = np.clip(np.array(xs, np.float32), 0, 1)
    in_double = (xs.astype(np.float64) * 15.0).astype(np.int64)
    assert np.array_equal((xs * np.float32(15)).astype(np.int64), in_double)
    vmin, vdiff = np.zeros(1, np.float32), np.ones(1, np.float32)
    assert np.array_equal(sq_oracle.quantize(xs[:, None], vmin, vdiff)[:, 0], in_double)
    below = np.nextafter(np.float32(7 / 15.0), np.float32(0))         # 7 / 15 rounds up in fp32: the one below gives 6
    assert float(below) * 15 < 7 and sq_oracle.quantize(np.array([[below]]), vmin, vdiff)[0, 0] == 6


def test_decode_rule():
    vmin = np.array([-1.0, 2.0], np.float32)
    vdiff = np.array([3.0, 0.0], np.float32)
    x = sq_oracle.decode(np.array([[0, 7], [15, 15]]), vmin, vdiff)
    np.testing.assert_allclose(x, [[-1.0 + 0.5 / 15 * 3, 2.0], [-1.0 + 15.5 / 15 * 3, 2.0]], rtol=1e-6)
    coarse = np.array([[10.0, 20.0]], np.float32)
    x = sq_oracle.decode(np.array([[0, 0]]), vmin, vdiff, coarse, np.array([0]))
    np.testing.assert_allclose(x, [[9.0 + 0.1, 22.0]], rtol=1e-6)


@pytest.mark.parametrize("seed,clustered", [(1, False), (2, True), (3, True)])
def test_contract_within_bound_of_faiss_rule(seed, clustered):
    rng = np.random.default_rng(seed)
    n, nq, n_list = 3000, 24, 16
    if clustered:
        c = rng.standard_normal((64, DIM)).astype(np.float32)
        x = ((c[rng.integers(0, 64, n)] + 0.3 * rng.standard_normal((n, DIM))) / np.sqrt(DIM)).astype(np.float16)
        q = ((c[rng.integers(0, 64, nq)] + 0.3 * rng.standard_normal((nq, DIM))) / np.sqrt(DIM)).astype(np.float16)
    else:
        x = rng.standard_normal((n, DIM)).astype(np.float16)
        q = rng.standard_normal((nq, DIM)).astype(np.float16)
    coarse = x[rng.choice(n, n_list, replace=False)].astype(np.float32)
    lists = sq_oracle.assign_lists(x, coarse)
    r = sq_oracle.residuals(x, coarse, lists)
    vmin, vdiff = sq_oracle.train_range(r)
    codes = sq_oracle.quantize(r, vmin, vdiff)
    ref = sq_oracle.faiss_scores(q, codes, vmin, vdiff, coarse, lists)
    got = sq_oracle.contract_scores(q, codes, vmin, vdiff, coarse, lists).astype(np.float64)
    bound = sq_oracle.contract_error_bound(q, codes, vmin, vdiff, coarse, lists)
    assert (np.abs(got - ref) <= bound).all()
    # the bound is a worst case (every w^ rounding error in the same direction); the gap itself is about one fp16 ulp
    # of the largest score
    top = np.abs(ref).max(1, keepdims=True)
    assert (np.abs(got - ref) <= 2 * sq_oracle._ulp16(top)).all(), float((np.abs(got - ref) / sq_oracle._ulp16(top)).max())


def test_query_operand_range():
    rng = np.random.default_rng(4)
    q = rng.standard_normal((8, DIM)).astype(np.float16) * np.float16(1e-3)
    q[3] = 0
    vdiff = rng.uniform(0, 2, DIM).astype(np.float32)
    w, e = sq_oracle.query_operand(q, vdiff)
    m = np.abs(w.astype(np.float32)).max(1)
    live = np.arange(8) != 3
    assert ((m[live] >= 2 ** 14) & (m[live] <= 2 ** 15)).all()
    assert e[3] == 0 and not w[3].any()


def test_slot_permutation_is_a_bijection_matching_the_fragment():
    from atlas_b200 import ops

    p = ops.sq_nibble_of_dim().numpy()
    assert sorted(p.tolist()) == list(range(DIM))
    # quad lane j of K-block kb, k16 step s: dims 16 s + 2 j + {0, 1} are the low nibbles of bytes 0 and 2 of its word,
    # dims + 8 the high nibbles
    for kb, s, j in [(0, 0, 0), (3, 1, 2), (11, 3, 3)]:
        d = kb * 64 + 16 * s + 2 * j
        word_byte = kb * 32 + j * 8 + (s // 2) * 4 + (s % 2)
        assert p[d] == 2 * word_byte and p[d + 1] == 2 * (word_byte + 2)
        assert p[d + 8] == 2 * word_byte + 1 and p[d + 9] == 2 * (word_byte + 2) + 1


def test_constructor():
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.index import DistributedFAISSIndex

    for bad in (16, 8, 0):
        with pytest.raises(AtlasB200Error, match="4-bit") as e:
            DistributedFAISSIndex("ivfsq", bad)
        assert "None or 4" in str(e.value) and "--index_mode flat" in str(e.value)
    if not torch.cuda.is_available():
        for ok in (None, 4):
            with pytest.raises(AtlasB200Error, match="CUDA device"):
                DistributedFAISSIndex("ivfsq", ok)


def test_index_file_names():
    from atlas_b200.index import DistributedFAISSIndex

    idx = DistributedFAISSIndex.__new__(DistributedFAISSIndex)
    idx.index_type, idx.code_size = "ivfsq", None
    assert idx._get_index_filename("/d").endswith("/indexivfsq_rank_0.atlas_b200.pt")
    assert idx._get_faiss_index_filename("/d").endswith("/indexivfsq_rank_0.faiss")
    idx.code_size = 4
    assert idx._get_index_filename("/d").endswith("/indexivfsq_4_rank_0.atlas_b200.pt")
    idx.index_type, idx.code_size = "ivfpq", 16
    assert idx._get_index_filename("/d").endswith("/indexivfpq_16_rank_0.atlas_b200.pt")
