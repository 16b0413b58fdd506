"""The attention forward kernels against float64 references, at the shapes the models run and with the per-element error
bounds that oracle/attention_fwd_oracle.py derives from the kernels' rounding steps (the style of
tests/test_backward_kernels_gpu.py).  Every assertion on a value is |got - fp64 reference| <= bound, element by element.

Part A: `ops.attention` (attention_kernel of csrc/attention.cu): O and the log-sum-exp.
Part B: the split-KV path: its raw partials, `combine_splits_kernel` on synthetic partials, and the two together.
Part C: the K / V stream kernel (csrc/attention_stream.cu), dense and compacted.
Part D: `ops.attention_packed` on the padding-compacted rows.
Part E: the forward with dropout, against the reference with the kernel's own keep mask.

Inputs are read from NaN-filled wider buffers (q at column 8, V before K in one buffer) and the output is written to a
strided column slice; afterwards the columns around it still hold the NaN bit pattern.  Where a key mask exists each case
runs without and with `key_block_live` and the two results are bit-identical.

A ragged last key block makes the TMA boxes read the rows of the NEXT segment; those keys carry s_mask = -inf, their
probabilities are exactly 0, and 0 x (any finite value) adds nothing.  Non-finite values in a neighbouring segment are not
a supported input (0 x inf): the projections that feed these kernels are finite or clamped (ops.clamp_inf_).

The worst |got - ref| / bound of each part and dtype is printed at the end of the module (run with -s)."""
import pytest
import torch

import attention_fwd_oracle as afo

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
NAN_BITS = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0}
NEG = {torch.float16: -1e4, torch.bfloat16: -1e9}     # invert_attention_mask (transformers 4.18): FiD's cross mask
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    yield torch.device("cuda:0")
    for key in sorted(WORST):
        print(f"\nWORST {key}: {WORST[key]:.4f}", end="")
    print()


def _assert_within(got, ref, bound, what, part, dtype):
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    worst = float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())
    print(f"RATIO {what}: {worst:.4f}")
    key = f"{part} {str(dtype)[6:]}"
    WORST[key] = max(WORST.get(key, 0.0), worst)
    assert worst <= 1.0, f"{what}: max |got - ref| / bound = {worst:.3g}"
    return worst


def _nan_filled(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _assert_sentinels(buf, c0, c1, dtype, what):
    outside = torch.ones(buf.shape[1], dtype=torch.bool, device=buf.device)
    outside[c0:c1] = False
    assert bool((buf.view(torch.int16)[:, outside] == NAN_BITS[dtype]).all()), f"{what}: write outside the heads"
    assert bool(torch.isfinite(buf[:, c0:c1]).all()), f"{what}: non-finite output"


def _inv_keep(p):
    thr = int(p * 65536 + 0.5)
    return float(torch.tensor(65536.0 / (65536 - thr), dtype=torch.float32))


def _length_mask(B, L, seed, full0=True):
    """Encoder self-attention mask (-10000 past each passage's length), lengths in bench's 148..276 of 384 scaled to L."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = max(1, L * 148 // 384), max(2, L * 276 // 384)
    lens = torch.randint(lo, hi + 1, (B,), generator=g)
    if full0:
        lens[0] = L
    return (torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0


def _passage_mask(B, Lk, neg, seed, holes=0.1, dead_passages=None, passage=384):
    """FiD's padded passages with bench's lengths (148..276 live keys of 384), random holes in the live keys, and
    optionally a run of wholly masked passages in batch row B - 1 (whole key chunks dead)."""
    g = torch.Generator().manual_seed(seed)
    j = torch.arange(Lk)
    n_pass = (Lk + passage - 1) // passage
    rows = []
    for b in range(B):
        lens = torch.randint(148 * passage // 384, 276 * passage // 384 + 1, (n_pass,), generator=g)
        live = j % passage < lens[j // passage]
        if holes:
            live &= torch.rand(Lk, generator=g) >= holes
        if dead_passages is not None and b == B - 1:
            live &= ~((j // passage >= dead_passages[0]) & (j // passage < dead_passages[1]))
        live[0] = True
        rows.append(torch.where(live, 0.0, neg))
    return torch.stack(rows)


def _qkv(B, H, Lq, Lk, dtype, seed, qmul, dev, big_v_segment=None):
    """16-bit q, k, v in NaN-filled wider buffers (q at column 8; V at column 8 and K at column H*64 + 24 of one buffer)
    and as the float64 [B, L, H, 64] the oracle reads."""
    g = torch.Generator().manual_seed(seed)
    HD = H * 64
    q16 = (torch.randn(B * Lq, HD, generator=g) * qmul).to(dtype)
    k16 = torch.randn(B * Lk, HD, generator=g).to(dtype)
    v16 = torch.randn(B * Lk, HD, generator=g)
    if big_v_segment is not None:          # +-60000: anything leaking out of a masked neighbour is seen at once
        rows = slice(big_v_segment * Lk, (big_v_segment + 1) * Lk)
        v16[rows] = torch.sign(v16[rows]) * 60000.0
    v16 = v16.to(dtype)
    qbuf = _nan_filled((B * Lq, HD + 72), dtype, dev)
    qbuf[:, 8:8 + HD] = q16.to(dev)
    kvbuf = _nan_filled((B * Lk, 2 * HD + 40), dtype, dev)
    kvbuf[:, 8:8 + HD] = v16.to(dev)
    kvbuf[:, HD + 24:2 * HD + 24] = k16.to(dev)
    Q = q16.double().view(B, Lq, H, 64).to(dev)
    K = k16.double().view(B, Lk, H, 64).to(dev)
    V = v16.double().view(B, Lk, H, 64).to(dev)
    return qbuf, kvbuf, HD + 24, 8, Q, K, V


# ------------------------------------------------------------------------------------------------------------------------
# Part A. ops.attention
# ------------------------------------------------------------------------------------------------------------------------
def _run_attention(dev, dtype, B, H, Lq, Lk, mask, bias, scale, causal, seed, qmul, what, part="A", dropout=None,
                   big_v_segment=None):
    from atlas_b200 import ops

    HD = H * 64
    qbuf, kvbuf, k_col0, v_col0, Q, K, V = _qkv(B, H, Lq, Lk, dtype, seed, qmul, dev, big_v_segment)
    maskd = mask.to(dev) if mask is not None else None
    biasd = bias.to(dev) if bias is not None else None
    keep, inv = None, 1.0
    if dropout is not None:
        keep = ops.attention_dropout_mask(B, H, Lq, Lk, dropout[0], dropout[1], dropout[2], dev)
        inv = _inv_keep(dropout[0])
    O64, lse64, bo, bl = afo.forward_bound(Q, K, V, maskd, biasd, scale, causal, keep, inv, dtype=dtype)
    live = ops.key_block_live(maskd)
    outs = []
    for blk in ((None, live) if live is not None else (None,)):
        obuf = _nan_filled((B * Lq, HD + 64), dtype, dev)
        out, lse = ops.attention(qbuf, 8, kvbuf, k_col0, kvbuf, v_col0, B, H, Lq, Lk, add_mask=maskd, bias_delta=biasd,
                                 scale=scale, causal_value=causal, out=obuf[:, 32:32 + HD], return_lse=True,
                                 dropout=dropout, block_live=blk)
        tag = f"{what} {str(dtype)[6:]} block_live={blk is not None}"
        _assert_sentinels(obuf, 32, 32 + HD, dtype, tag)
        _assert_within(out, O64.reshape(B * Lq, HD), bo.reshape(B * Lq, HD), f"{tag} O", part, dtype)
        _assert_within(lse, lse64, bl, f"{tag} lse", part + "-lse", dtype)
        outs.append((out.clone(), lse.clone()))
    if len(outs) == 2:
        assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16)), f"{what}: O differs with block_live"
        assert torch.equal(outs[0][1], outs[1][1]), f"{what}: lse differs with block_live"
    return outs[0], (O64, lse64, bo, bl)


def _bias(H, Lq, Lk, seed, ramp=0.0):
    g = torch.Generator().manual_seed(seed)
    b = 0.5 * torch.randn(H, Lq + Lk - 1, generator=g)
    return b + ramp * torch.arange(Lq + Lk - 1)[None, :].float() if ramp else b


# (S, H, L, qmul): T5 encoder self-attention, relative-position bias, bench's passage lengths under -10000
T5_ENC = [(40, 12, 384, 0.35), (2, 16, 384, 1.0), (3, 12, 384, 0.12), (1, 32, 384, 0.12), (2, 12, 480, 0.35),
          (5, 8, 320, 0.35)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S,H,L,qmul", T5_ENC, ids=[f"S{c[0]}-H{c[1]}-L{c[2]}" for c in T5_ENC])
def test_t5_encoder_attention(dev, dtype, S, H, L, qmul):
    """FiD encoder at the bench's shape, T5-large heads with |q| ~ 1 (a peaked softmax: few keys carry a row), and the
    small-magnitude near-uniform softmax (and, for S = 3, no key mask at all: the bench's shape); 480 = 7.5 key blocks."""
    _run_attention(dev, dtype, S, H, L, L, _length_mask(S, L, seed=L + S, full0=S < 40), _bias(H, L, L, S), 1.0, 0.0,
                   seed=S * L, qmul=qmul, what=f"t5enc S{S} H{H} L{L}")
    if S == 3:
        _run_attention(dev, dtype, S, H, L, L, None, _bias(H, L, L, S), 1.0, 0.0, seed=S * L + 1, qmul=qmul,
                       what=f"t5enc nomask S{S} H{H} L{L}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,L", [(37, 128), (37, 173), (37, 512), (3, 256), (5, 64), (8, 384)])
def test_contriever_attention(dev, dtype, B, L):
    """Scale 1/8, no bias; 37 segments x 12 heads is more CTAs than SMs.  B = 3 runs without any key mask."""
    mask = _length_mask(B, L, seed=L + 1) if B > 3 else None
    _run_attention(dev, dtype, B, 12, L, L, mask, None, 0.125, 0.0, seed=L, qmul=1.0, what=f"bert B{B} L{L}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [1, 63, 64, 65, 127, 129, 200, 576])
def test_tile_edges(dev, dtype, L):
    """The edges of the 128-row query tile and the 64-key block, and MAX_LK = 576 (9 key blocks).  Three segments: the
    ragged blocks of segments 0 and 1 read the next segment's rows, and segment 1's V is +-60000 everywhere."""
    g = torch.Generator().manual_seed(L)
    lens = torch.randint(max(1, L // 3), L + 1, (3,), generator=g)
    lens[0] = L
    mask = (torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0
    _run_attention(dev, dtype, 3, 4, L, L, mask, _bias(4, L, L, L), 1.0, 0.0, seed=L + 11, qmul=0.35, what=f"edge L{L}",
                   big_v_segment=1)
    _run_attention(dev, dtype, 3, 4, L, L, None, None, 0.125, 0.0, seed=L + 12, qmul=1.0, what=f"edge nomask L{L}",
                   big_v_segment=1)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("T", [1, 32, 64, 130, 200])
def test_decoder_causal_self_attention(dev, dtype, T):
    """Causal -10000 with T5's decoder bias; 130 and 200 put the causal edge across the query tiles and key blocks."""
    _run_attention(dev, dtype, 4, 12, T, T, None, _bias(12, T, T, T), 1.0, -10000.0, seed=T + 7, qmul=0.35,
                   what=f"dec T{T}")
    if T in (32, 200):  # with a key mask on top
        _run_attention(dev, dtype, 2, 4, T, T, _length_mask(2, T, seed=3), _bias(4, T, T, T), 1.0, -10000.0, seed=T + 8,
                       qmul=0.35, what=f"dec masked T{T}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Lq,Lk", [(32, 384), (200, 64), (577, 576), (100, 173)])
def test_rectangular_attention(dev, dtype, Lq, Lk):
    """Lq != Lk with the bias table indexed j - i + Lq - 1 and the causal rule j > i; (577, 576) fills the table
    (Lq + Lk - 1 = 2 MAX_LK)."""
    H = 4
    mask = _length_mask(2, Lk, seed=Lq)
    _run_attention(dev, dtype, 2, H, Lq, Lk, mask, _bias(H, Lq, Lk, Lq + Lk), 1.0, 0.0, seed=Lq + Lk, qmul=0.35,
                   what=f"rect Lq{Lq} Lk{Lk}")
    _run_attention(dev, dtype, 2, H, Lq, Lk, None, _bias(H, Lq, Lk, Lq - Lk), 1.0, -10000.0, seed=Lq * Lk, qmul=0.35,
                   what=f"rect causal Lq{Lq} Lk{Lk}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_bias_ramp_rescales_every_block(dev, dtype):
    """A bias ramp of +0.15 per key offset: every later key block raises the row maximum by ~10 and O is rescaled on
    every block; the exponents reach the hundreds, which the bound's term on their magnitude covers."""
    L, H = 384, 12
    _run_attention(dev, dtype, 2, H, L, L, _length_mask(2, L, seed=1), _bias(H, L, L, 5, ramp=0.15), 1.0, 0.0, seed=17,
                   qmul=0.12, what="ramp")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S,H,L,use_bias", [(7, 3, 384, True), (5, 2, 200, True), (4, 12, 512, False), (3, 1, 512, True)])
def test_masked_segments_and_holes(dev, dtype, S, H, L, use_bias):
    """Lengths from 3 keys to all of them, a hole of one whole masked key block in the middle of segment 3, and a
    segment whose keys are ALL masked: it keeps every block live and is uniform-ish over the masked keys, like the
    reference's softmax."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(S * 100 + L)
    lens = torch.randint(1, L + 1, (S,), generator=g)
    lens[0], lens[1] = L, 3
    mask = (torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0
    if S > 3:
        mask[3, :] = 0.0
        mask[3, 64:140] = -10000.0
    mask[2, :] = -10000.0
    live = ops.key_block_live(mask.to(dev))
    assert live.shape == (S, (L + 63) // 64) and int(live[1].sum()) == 1 and bool(live[0].all()) and bool(live[2].all())
    if S > 3:
        assert int(live[3, 1]) == 0 and int(live[3].sum()) == live.shape[1] - 1
    bias = _bias(H, L, L, L) if use_bias else None
    _run_attention(dev, dtype, S, H, L, L, mask, bias, 1.0, 0.0, seed=S + L, qmul=0.3, what=f"masked S{S} L{L}")


def test_attention_argument_checks(dev):
    """B = 0 is a no-op; the documented limits are errors before any launch."""
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    H = 2
    buf = torch.zeros((1200, 3 * H * 64 + 8), dtype=torch.bfloat16, device=dev)
    out = ops.attention(buf, 0, buf, H * 64, buf, 2 * H * 64, 0, H, 128, 128,
                        out=torch.empty((0, H * 64), dtype=torch.bfloat16, device=dev))
    assert out.shape == (0, H * 64)
    for kw, frag in ((dict(Lq=64, Lk=577), "Lk <= 576"), (dict(Lq=578, Lk=576), "bias table"),
                     (dict(Lq=64, Lk=64, k_col0=H * 64 + 4), "multiples of 8")):
        sentinel = torch.full((1200, H * 64), 3.0, dtype=torch.bfloat16, device=dev)
        with pytest.raises(AtlasB200Error, match=frag):
            ops.attention(buf, 0, buf, kw.get("k_col0", H * 64), buf, 2 * H * 64, 1, H, kw["Lq"], kw["Lk"], out=sentinel)
        assert bool((sentinel == 3.0).all())


# ------------------------------------------------------------------------------------------------------------------------
# Part B. split-KV partials and combine_splits_kernel
# ------------------------------------------------------------------------------------------------------------------------
def _partials_to_oracle_layout(o_part, ml, B, C, Lq, H):
    o = o_part.double().view(B, C, Lq, H, 64)
    mlv = ml.double().view(B, C, Lq, H, 2)
    return o, mlv[..., 0].permute(0, 1, 3, 2), mlv[..., 1].permute(0, 1, 3, 2)


def _assert_partials(o_part, ml, part, B, C, Lq, H, what, key, dtype):
    """Max-invariant comparison of kernel partials (o_c, m_c, l_c) with the oracle's: o_c / l_c, m_c + log l_c, and m_c
    against the chunk maximum."""
    o, m, l = _partials_to_oracle_layout(o_part, ml, B, C, Lq, H)
    assert bool((l >= 0.999).all()), f"{what}: a chunk's row sum is below 1"
    _assert_within(o / l.permute(0, 1, 3, 2)[..., None], part["O"], part["O_bound"], f"{what} partial O", key, dtype)
    _assert_within(m + torch.log(l), part["lse"], part["lse_bound"], f"{what} partial lse", key + "-lse", dtype)
    _assert_within(m, part["m"], part["m_bound"], f"{what} partial max", key + "-lse", dtype)


# (B, H, T, Lk, split)
SPLIT_CASES = [(2, 12, 32, 15 * 384, 384), (1, 12, 100, 4 * 512, 512), (2, 3, 128, 1152, 384), (2, 12, 8, 768, 384)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,T,Lk,split", SPLIT_CASES, ids=[f"B{c[0]}-H{c[1]}-T{c[2]}-Lk{c[3]}" for c in SPLIT_CASES])
def test_split_kv_partials_and_combine(dev, dtype, B, H, T, Lk, split):
    """attention_kernel with q_div = splits: every chunk's partials on their own, then `cross_attention_split` on the
    split path (the stream kernel switched off where it would take the shape).  The last batch row has wholly masked
    passages: chunks whose every key is masked."""
    from atlas_b200 import ops
    from atlas_b200._lib import current_stream_ptr, lib

    HD, C = H * 64, Lk // split
    qbuf, kvbuf, k_col0, v_col0, Q, K, V = _qkv(B, H, T, Lk, dtype, seed=Lk + T, qmul=0.4, dev=dev)
    mask = _passage_mask(B, Lk, NEG[dtype], seed=T, dead_passages=(1, 2), passage=split).to(dev)
    o_part = torch.full((B * C * T, HD), float("nan"), dtype=torch.float32, device=dev)
    ml = torch.full((B * C * T, H, 2), float("nan"), dtype=torch.float32, device=dev)
    dummy = torch.empty((8,), dtype=dtype, device=dev)
    p = ops._ptr
    ops.check(lib().atlas_b200_attention_train(p(qbuf), qbuf.stride(0), 8, p(kvbuf), kvbuf.stride(0), k_col0, p(kvbuf),
                                               kvbuf.stride(0), v_col0, p(dummy), 8, p(mask), None, B * C, H, T, split, 1.0,
                                               0.0, C, p(o_part), p(ml), None, 0.0, 0, 0, None, ops._bf(qbuf),
                                               current_stream_ptr()))
    part = afo.split_partials(Q, K, V, mask, 1.0, split, dtype=dtype)
    tag = f"split B{B} T{T} Lk{Lk} {str(dtype)[6:]}"
    _assert_partials(o_part, ml, part, B, C, T, H, tag, "B-partials", dtype)

    O64, lse64, bo, bl = afo.forward_bound(Q, K, V, mask, None, 1.0, 0.0, dtype=dtype)
    saved = ops._XATTN_STREAM
    ops._XATTN_STREAM = False
    try:
        out, lse = ops.cross_attention_split(qbuf, 8, kvbuf, k_col0, v_col0, B, H, T, Lk, add_mask=mask, split=split,
                                             return_lse=True)
    finally:
        ops._XATTN_STREAM = saved
    _assert_within(out, O64.reshape(B * T, HD), bo.reshape(B * T, HD), f"{tag} O", "B", dtype)
    _assert_within(lse, lse64, bl, f"{tag} lse", "B-lse", dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_combine_kernel_on_synthetic_partials(dev, dtype):
    """combine_splits_kernel alone: row maxima 1e4 apart, a dead chunk exactly as the stream kernel writes one
    (o = 0, m = -inf, l = 0), odd Lq, an output wider than H * 64, and splits = 1."""
    from atlas_b200 import ops
    from atlas_b200._lib import current_stream_ptr, lib

    g = torch.Generator().manual_seed(6)
    B, C, Lq, H = 2, 5, 7, 3
    o = torch.randn(B, C, Lq, H, 64, generator=g) * 3.0
    m = torch.randn(B, C, H, Lq, generator=g) * 4.0
    l = 1.0 + 50.0 * torch.rand(B, C, H, Lq, generator=g)
    o[:, 1], m[:, 1], l[:, 1] = 0.0, float("-inf"), 0.0
    m[:, 2] -= 1e4
    m[0, 3] += 1e4              # batch row 0: chunk 3 alone survives
    for splits in (C, 1):
        oc, mc, lc = (t[:, :splits].contiguous().to(dev) for t in (o, m, l))
        if splits == 1:
            mc = mc + 3.0       # the dead and shifted chunks are gone: a plain finite maximum
        o_part = oc.reshape(B * splits * Lq, H * 64).contiguous()
        ml = torch.stack([mc.permute(0, 1, 3, 2), lc.permute(0, 1, 3, 2)], -1).reshape(B * splits * Lq, H, 2).contiguous()
        obuf = _nan_filled((B * Lq, H * 64 + 64), dtype, dev)
        lse = torch.empty((B, H, Lq), dtype=torch.float32, device=dev)
        p = ops._ptr
        ops.check(lib().atlas_b200_attention_combine_ex(p(o_part), p(ml), B, splits, Lq, H, p(obuf[:, 32:]), obuf.stride(0),
                                                        p(lse), ops._bf(obuf), current_stream_ptr()))
        ref, ref_lse, ob, lb = afo.combine(oc.double(), mc.double(), lc.double(), dtype=dtype)
        tag = f"combine splits={splits} {str(dtype)[6:]}"
        _assert_sentinels(obuf, 32, 32 + H * 64, dtype, tag)
        _assert_within(obuf[:, 32:32 + H * 64], ref.reshape(B * Lq, H * 64), ob.reshape(B * Lq, H * 64), f"{tag} O",
                       "B-combine", dtype)
        _assert_within(lse, ref_lse, lb, f"{tag} lse", "B-combine-lse", dtype)


# ------------------------------------------------------------------------------------------------------------------------
# Part C. the K / V stream kernel
# ------------------------------------------------------------------------------------------------------------------------
# (B, H, T, Lk, dead passages of the last batch row)
STREAM_CASES = [(1, 12, 8, 15360, None), (2, 12, 32, 40 * 384, (20, 40)), (3, 2, 64, 1088, None), (2, 1, 1, 2048, None),
                (2, 3, 32, 4000, (5, 11)), (1, 12, 7, 15360, (3, 9))]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,T,Lk,dead", STREAM_CASES, ids=[f"B{c[0]}-H{c[1]}-T{c[2]}-Lk{c[3]}" for c in STREAM_CASES])
def test_stream_kernel(dev, dtype, B, H, T, Lk, dead):
    """cross_stream_kernel + combine through `cross_attention_split` at its default chunk: FiD-base training shapes, a
    ragged last chunk and tile (1088, 4000), one query, dead passages (chunks without a live tile write (0, -inf, 0)),
    the dead-tile skipping on and off, and every chunk's partials on their own."""
    from atlas_b200 import ops
    from atlas_b200._lib import current_stream_ptr, lib

    assert ops._XATTN_STREAM and ops._SKIP_MASKED
    HD = H * 64
    qbuf, kvbuf, k_col0, v_col0, Q, K, V = _qkv(B, H, T, Lk, dtype, seed=Lk + 3 * T + H, qmul=0.4, dev=dev)
    mask = _passage_mask(B, Lk, NEG[dtype], seed=Lk + T, dead_passages=dead).to(dev)
    O64, lse64, bo, bl = afo.forward_bound(Q, K, V, mask, None, 1.0, 0.0, dtype=dtype)
    tag = f"stream B{B} H{H} T{T} Lk{Lk} {str(dtype)[6:]}"
    out, lse = ops.cross_attention_split(qbuf, 8, kvbuf, k_col0, v_col0, B, H, T, Lk, add_mask=mask, split=Lk, return_lse=True)
    _assert_within(out, O64.reshape(B * T, HD), bo.reshape(B * T, HD), f"{tag} O", "C", dtype)
    _assert_within(lse, lse64, bl, f"{tag} lse", "C-lse", dtype)
    ops._SKIP_MASKED = False
    try:
        full = ops.cross_attention_split(qbuf, 8, kvbuf, k_col0, v_col0, B, H, T, Lk, add_mask=mask, split=Lk)
    finally:
        ops._SKIP_MASKED = True
    assert torch.equal(full.view(torch.int16), out.view(torch.int16)), f"{tag}: differs with the dead tiles skipped"

    chunk = ops._XATTN_CHUNK
    C = (Lk + chunk - 1) // chunk
    live = ops.key_block_live(mask)
    o_part = torch.full((B * C * T, HD), float("nan"), dtype=torch.float32, device=dev)
    ml = torch.full((B * C * T, H, 2), float("nan"), dtype=torch.float32, device=dev)
    p = ops._ptr
    ops.check(lib().atlas_b200_cross_attention_stream(p(qbuf), qbuf.stride(0), 8, p(kvbuf), kvbuf.stride(0), k_col0, v_col0,
                                                      p(mask), p(live), B, H, T, Lk, chunk, 1.0, p(o_part), p(ml),
                                                      ops._bf(qbuf), current_stream_ptr()))
    nt = (Lk + 63) // 64
    dead_chunk = torch.stack([~live[:, c * (chunk // 64):min(nt, (c + 1) * (chunk // 64))].bool().any(1) for c in range(C)], 1)
    o, m, l = _partials_to_oracle_layout(o_part, ml, B, C, T, H)
    if dead is not None and Lk >= 4000:
        assert bool(dead_chunk.any()), "the case has no chunk without a live tile"
    assert bool((o[dead_chunk] == 0).all()) and bool((l[dead_chunk] == 0).all()) and bool((m[dead_chunk] == float("-inf")).all())
    part = afo.split_partials(Q, K, V, mask, 1.0, chunk, dtype=dtype)
    alive = ~dead_chunk
    sel = {n: t[alive] for n, t in part.items()}
    _assert_within((o / l.permute(0, 1, 3, 2)[..., None])[alive], sel["O"], sel["O_bound"], f"{tag} partial O", "C-partials", dtype)
    _assert_within((m + torch.log(l))[alive], sel["lse"], sel["lse_bound"], f"{tag} partial lse", "C-partials-lse", dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_stream_kernel_on_compacted_kv(dev, dtype):
    """The stream kernel reading only the live 64-key tiles, compacted (`compact_live_tiles`): bit-identical to the
    dense run and within the bounds of the oracle."""
    from atlas_b200 import ops

    B, H, T, Lk = 3, 12, 32, 5 * 384
    HD = H * 64
    g = torch.Generator().manual_seed(5)
    q = (torch.randn(B * T, HD, generator=g) * 0.4).to(dtype).to(dev)
    kv = torch.randn(B * Lk, 2 * HD, generator=g).to(dtype).to(dev)
    lens = torch.randint(20, 385, (B, 5), generator=g)
    lens[0, 0], lens[1, 2] = 384, 1
    mask = ((torch.arange(384)[None, None, :] >= lens[..., None]).reshape(B, Lk).float() * NEG[dtype]).to(dev)
    live = ops.key_block_live(mask)
    kv_live, tile_off, _ = ops.compact_live_tiles(kv, live)
    a, lse = ops.cross_attention_stream_compact(q, kv_live, live, tile_off, B, H, T, Lk, mask, return_lse=True)
    b = ops.cross_attention_split(q, 0, kv, 0, HD, B, H, T, Lk, add_mask=mask, split=384, tile_live=live)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    Q = q.double().view(B, T, H, 64)
    K, V = (t.reshape(B, Lk, H, 64) for t in kv.double().split(HD, dim=1))
    O64, lse64, bo, bl = afo.forward_bound(Q, K, V, mask, None, 1.0, 0.0, dtype=dtype)
    _assert_within(a, O64.reshape(B * T, HD), bo.reshape(B * T, HD), f"compact {str(dtype)[6:]} O", "C", dtype)
    _assert_within(lse, lse64, bl, f"compact {str(dtype)[6:]} lse", "C-lse", dtype)


# ------------------------------------------------------------------------------------------------------------------------
# Part D. ops.attention_packed
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S,H,L,use_bias,scale", [(40, 12, 384, True, 1.0), (9, 4, 256, True, 1.0), (6, 12, 192, True, 1.0),
                                                  (11, 2, 128, True, 1.0), (4, 3, 64, False, 1.0), (8, 12, 320, False, 0.125)])
def test_packed_attention(dev, dtype, S, H, L, use_bias, scale):
    """Segment s keeps its first n_s 64-row tiles, stored back to back: each segment's rows against the fp64 attention over
    its kept keys (the dropped tiles hold masked keys only).  Segments keeping one tile, all of them, a dead tile inside
    the kept prefix, and a segment of padding only (keeps every tile)."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(S * 1000 + L)
    HD = H * 64
    qkv16 = torch.randn(S * L, 3 * HD, generator=g)
    qkv16[:, :HD] *= 0.35 if scale == 1.0 else 1.0
    qkv16 = qkv16.to(dtype)
    bias = _bias(H, L, L, S).to(dev) if use_bias else None
    lens = torch.randint(max(1, L * 148 // 384), L * 276 // 384 + 1, (S,), generator=g)
    lens[0], lens[1] = L, 3
    mask = (torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0
    if L >= 192:
        mask[3, :150] = 0.0
        mask[3, 64:140] = -10000.0                                 # block 1 of segment 3 is dead but kept (prefix rule)
    mask[2, :] = -10000.0                                          # no live key at all: keeps every tile
    mask = mask.to(dev)
    keep, off, _, count = ops.segment_tile_scan(ops.key_block_live(mask))
    n_rows = int(count)
    kept = keep.reshape(-1).bool()
    packed = _nan_filled((S * L, 3 * HD), dtype, dev)              # rows past the count must never matter
    packed[:n_rows] = qkv16.to(dev).view(-1, 64, 3 * HD)[kept].reshape(n_rows, -1)
    obuf = _nan_filled((S * L, HD + 64), dtype, dev)
    out = ops.attention_packed(packed, keep, off, S, H, L, mask, bias, scale=scale, out=obuf[:, 32:32 + HD])
    assert bool((obuf.view(torch.int16)[n_rows:] == NAN_BITS[dtype]).all()), "write past the packed rows"
    _assert_sentinels(obuf[:n_rows], 32, 32 + HD, dtype, f"packed S{S} L{L}")
    n_kept = keep.sum(1).tolist()
    assert n_kept[0] == L // 64 and n_kept[1] == 1 and n_kept[2] == L // 64
    refs, bounds = [], []
    q64, k64, v64 = (t.double().view(S, L, H, 64).to(dev) for t in qkv16.split(HD, dim=1))
    for s in range(S):
        n = 64 * n_kept[s]
        bs = bias[:, L - n:L + n - 1] if bias is not None else None       # offsets -(n - 1) .. n - 1 of the [H, 2 L - 1] table
        O64, _, bo, _ = afo.forward_bound(q64[s:s + 1, :n], k64[s:s + 1, :n], v64[s:s + 1, :n], mask[s:s + 1, :n], bs, scale,
                                          0.0, dtype=dtype)
        refs.append(O64.reshape(n, HD))
        bounds.append(bo.reshape(n, HD))
    _assert_within(out[:n_rows], torch.cat(refs), torch.cat(bounds), f"packed S{S} H{H} L{L} {str(dtype)[6:]} O", "D", dtype)


# ------------------------------------------------------------------------------------------------------------------------
# Part E. dropout on the probabilities
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p_drop", [0.1, 0.5])
def test_attention_forward_with_dropout(dev, dtype, p_drop):
    """Encoder shape and the cross shape on the split path, each element against the fp64 forward with the keep mask the
    kernels derive from (seed, offset); the log-sum-exp is that of the run without dropout."""
    from atlas_b200 import ops

    B, H, L = 4, 12, 384
    dkey = (p_drop, 1234, 40)
    (_, lse_d), (_, lse64, _, bl) = _run_attention(dev, dtype, B, H, L, L, _length_mask(B, L, seed=5), _bias(H, L, L, 3), 1.0,
                                                  0.0, seed=11, qmul=0.35, what=f"dropout {p_drop} enc", part="E",
                                                  dropout=dkey)
    (_, lse_0), _ = _run_attention(dev, dtype, B, H, L, L, _length_mask(B, L, seed=5), _bias(H, L, L, 3), 1.0, 0.0, seed=11,
                                   qmul=0.35, what="dropout off enc", part="E")
    assert torch.equal(lse_d, lse_0), "dropout changed the log-sum-exp"

    B, T, Lk, split = 2, 32, 1152, 384
    HD = H * 64
    qbuf, kvbuf, k_col0, v_col0, Q, K, V = _qkv(B, H, T, Lk, dtype, seed=13, qmul=0.4, dev=dev)
    mask = _passage_mask(B, Lk, NEG[dtype], seed=7).to(dev)
    keep = ops.attention_dropout_mask(B, H, T, Lk, p_drop, dkey[1], dkey[2], dev)
    frac = float(keep.float().mean())
    assert abs(frac - (1.0 - p_drop)) < 0.01, frac
    O64, lse64, bo, bl = afo.forward_bound(Q, K, V, mask, None, 1.0, 0.0, keep, _inv_keep(p_drop), dtype=dtype)
    out, lse = ops.cross_attention_split(qbuf, 8, kvbuf, k_col0, v_col0, B, H, T, Lk, add_mask=mask, split=split,
                                         return_lse=True, dropout=dkey)
    tag = f"dropout {p_drop} cross {str(dtype)[6:]}"
    _assert_within(out, O64.reshape(B * T, HD), bo.reshape(B * T, HD), f"{tag} O", "E", dtype)
    _assert_within(lse, lse64, bl, f"{tag} lse", "E-lse", dtype)
