"""The training step's backward kernels against float64 references, at the shapes training runs and with per-element error
bounds derived from the kernels' rounding steps (the style of tests/test_decode_kernels_gpu.py).

Part A: `ops.attention_bwd` (csrc/attention_bwd.cu) against oracle/attention_bwd_oracle.py, which states the bounds: one
16-bit rounding of the output, u sum |terms| for the 16-bit P / dS operands of the MMAs, 2^-25 sum |other factor| for fp16
subnormals, and an fp32 headroom of 2^-16 on the magnitudes that make up S, dP, D and the sums.  Every case also checks
the column-offset sentinels, the dead-block skipping (`block_live`) on and off, exact zeros for masked keys, and the
log-sum-exp the forward kernels hand to the backward.

Part B: the row kernels of csrc/backward.cu, each computed in fp64 the way its header comment states the operation."""
import math

import pytest
import torch

import attention_bwd_oracle as abo

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
NAN_BITS = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0}
NEG = {torch.float16: -1e4, torch.bfloat16: -1e9}     # invert_attention_mask (transformers 4.18): FiD's cross mask
UNIT = abo.UNIT
SUB = abo.SUBNORMAL_HALF_SPACING
F32 = 2.0 ** -22      # the fp32 operation just before an output's 16-bit rounding
P_DROP = 0.1


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _assert_within(got, ref, bound, what):
    worst = float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())
    print(f"RATIO {what}: {worst:.4f}")
    assert worst <= 1.0, f"{what}: max |got - ref| / bound = {worst:.3g}"
    return worst


def _nan_filled(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _inv_keep(p):
    thr = int(p * 65536 + 0.5)
    return float(torch.tensor(65536.0 / (65536 - thr), dtype=torch.float32))


def _key_chunks(B, H, Lq, Lk, sms):
    """The dq kernel's split of the key blocks (atlas_b200_attention_bwd_train)."""
    nkb = (Lk + 63) // 64
    base = B * H * ((Lq + 63) // 64)
    want = (2 * sms + base - 1) // base
    return max(1, min(want, (nkb + 3) // 4))


# ------------------------------------------------------------------------------------------------------------------------
# Part A. attention_bwd
# ------------------------------------------------------------------------------------------------------------------------
def _passage_mask(B, Lk, neg, seed, holes=0.0, dead_passages=None):
    """FiD's padded 384-key passages with bench's lengths (148..276 live keys), random holes in the live keys, and
    optionally a run of wholly masked passages in batch row B - 1 (whole key chunks dead)."""
    g = torch.Generator().manual_seed(seed)
    j = torch.arange(Lk)
    n_pass = (Lk + 383) // 384
    rows = []
    for b in range(B):
        lens = torch.randint(148, 277, (n_pass,), generator=g)
        live = j % 384 < lens[j // 384]
        if holes:
            live &= torch.rand(Lk, generator=g) >= holes
        if dead_passages is not None and b == B - 1:
            live &= ~((j // 384 >= dead_passages[0]) & (j // 384 < dead_passages[1]))
        live[0] = True
        rows.append(torch.where(live, 0.0, neg))
    return torch.stack(rows)


def _length_mask(B, L, seed):
    """Encoder self-attention mask (-10000 past each passage's length), lengths in bench's 148..276 of 384 scaled to L;
    row 0 full length."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = max(1, L * 148 // 384), max(2, L * 276 // 384)
    lens = torch.randint(lo, hi + 1, (B,), generator=g)
    lens[0] = L
    return (torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0


def _run_bwd(dev, dtype, B, H, Lq, Lk, mask, bias, scale, causal, split, drop, seed, qmul, what):
    """Backward from NaN-guarded strided buffers, with block_live off and on, checked against the fp64 oracle."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(seed)
    HD = H * 64
    q16 = (torch.randn(B * Lq, HD, generator=g) * qmul).to(dtype)
    k16 = torch.randn(B * Lk, HD, generator=g).to(dtype)
    v16 = torch.randn(B * Lk, HD, generator=g).to(dtype)
    do16 = torch.randn(B * Lq, HD, generator=g).to(dtype)
    maskd = mask.to(dev) if mask is not None else None
    biasd = bias.to(dev) if bias is not None else None
    Q = q16.double().view(B, Lq, H, 64).to(dev)
    K = k16.double().view(B, Lk, H, 64).to(dev)
    V = v16.double().view(B, Lk, H, 64).to(dev)
    DO = do16.double().view(B, Lq, H, 64).to(dev)
    keep, inv, dkey = None, 1.0, None
    if drop:
        dkey = (P_DROP, 1234 + seed, 4 * seed)
        keep = ops.attention_dropout_mask(B, H, Lq, Lk, P_DROP, dkey[1], dkey[2], dev)
        inv = _inv_keep(P_DROP)
    O64, lse64 = abo.forward(Q, K, V, maskd, biasd, scale, causal, keep, inv)
    o16 = O64.reshape(B * Lq, HD).to(dtype)
    ref = abo.attention_bwd(Q, K, V, o16.double().view(B, Lq, H, 64), DO, maskd, biasd, scale, causal, keep, inv,
                            dtype=dtype)

    # inputs: q at column 8, V before K in one kv buffer, O and dO as strided views; every other column NaN
    qbuf = _nan_filled((B * Lq, HD + 72), dtype, dev)
    qbuf[:, 8:8 + HD] = q16.to(dev)
    kvbuf = _nan_filled((B * Lk, 2 * HD + 40), dtype, dev)
    v_col0, k_col0 = 8, HD + 24
    kvbuf[:, v_col0:v_col0 + HD] = v16.to(dev)
    kvbuf[:, k_col0:k_col0 + HD] = k16.to(dev)
    obuf = _nan_filled((B * Lq, HD + 64), dtype, dev)
    obuf[:, 32:32 + HD] = o16.to(dev)
    dobuf = _nan_filled((B * Lq, HD + 48), dtype, dev)
    dobuf[:, 16:16 + HD] = do16.to(dev)
    lse = lse64.float().contiguous()

    live = ops.key_block_live(maskd)
    results = {}
    for bl in ((None, live) if live is not None else (None,)):
        if split:
            dqbuf = _nan_filled((B * Lq, HD), dtype, dev)
            dq_col0 = 0
        else:
            dqbuf = _nan_filled((B * Lq, HD + 128), dtype, dev)
            dq_col0 = 64
        dkvbuf = _nan_filled((B * Lk, 2 * HD + 64), dtype, dev)
        dk_col0, dv_col0 = 8, HD + 24
        dbias = ops.attention_bwd(qbuf, 8, kvbuf, k_col0, kvbuf, v_col0, obuf[:, 32:32 + HD], dobuf[:, 16:16 + HD],
                                  dqbuf, dq_col0, dkvbuf, dk_col0, dkvbuf, dv_col0, B, H, Lq, Lk, add_mask=maskd,
                                  bias_delta=biasd, need_dbias=bias is not None, scale=scale, causal_value=causal,
                                  lse=lse, split_keys=split, dropout=dkey, block_live=bl)
        tag = f"{what} block_live={bl is not None}"
        # sentinels: the columns around the written heads keep their NaN bits, the written ones are finite
        for buf, cols in ((dqbuf, [(dq_col0, dq_col0 + HD)]), (dkvbuf, [(dk_col0, dk_col0 + HD), (dv_col0, dv_col0 + HD)])):
            outside = torch.ones(buf.shape[1], dtype=torch.bool, device=dev)
            for c0, c1 in cols:
                outside[c0:c1] = False
                assert bool(torch.isfinite(buf[:, c0:c1]).all()), f"{tag}: non-finite output"
            assert bool((buf.view(torch.int16)[:, outside] == NAN_BITS[dtype]).all()), f"{tag}: write outside the heads"
        dq = dqbuf[:, dq_col0:dq_col0 + HD]
        dk = dkvbuf[:, dk_col0:dk_col0 + HD]
        dv = dkvbuf[:, dv_col0:dv_col0 + HD]
        _assert_within(dq, ref["dq"].reshape(B * Lq, HD), ref["dq_bound"].reshape(B * Lq, HD), f"{tag} dQ")
        _assert_within(dk, ref["dk"].reshape(B * Lk, HD), ref["dk_bound"].reshape(B * Lk, HD), f"{tag} dK")
        _assert_within(dv, ref["dv"].reshape(B * Lk, HD), ref["dv_bound"].reshape(B * Lk, HD), f"{tag} dV")
        if bias is not None:
            _assert_within(dbias, ref["dbias"], ref["dbias_bound"], f"{tag} dbias")
        if maskd is not None:
            dead = (maskd <= -1e4).reshape(B * Lk)
            assert bool((dk[dead] == 0).all()) and bool((dv[dead] == 0).all()), f"{tag}: masked keys got dK / dV"
        results[bl is not None] = (dq.clone(), dk.clone(), dv.clone())
    if len(results) == 2:
        (dq0, dk0, dv0), (dq1, dk1, dv1) = results[False], results[True]
        assert torch.equal(dk0.view(torch.int16), dk1.view(torch.int16)), f"{what}: dK differs with block_live"
        assert torch.equal(dv0.view(torch.int16), dv1.view(torch.int16)), f"{what}: dV differs with block_live"
        if not split:
            assert torch.equal(dq0.view(torch.int16), dq1.view(torch.int16)), f"{what}: dQ differs with block_live"
    return ref


# (S, L): T5 encoder self-attention with relative-position bias and dbias, passage-length masks
ENC_CASES = [(3, 100), (8, 200), (3, 384), (8, 384), (3, 512)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S,L", ENC_CASES, ids=[f"S{s}-L{l}" for s, l in ENC_CASES])
def test_encoder_self_attention_bwd(dev, dtype, S, L):
    H = 12
    g = torch.Generator().manual_seed(L + S)
    bias = 0.5 * torch.randn(H, 2 * L - 1, generator=g)
    _run_bwd(dev, dtype, S, H, L, L, _length_mask(S, L, seed=L), bias, 1.0, 0.0, False, False, seed=S * L, qmul=0.35,
             what=f"enc S{S} L{L}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [173, 512])
def test_bert_self_attention_bwd(dev, dtype, L):
    _run_bwd(dev, dtype, 4, 12, L, L, _length_mask(4, L, seed=L + 1), None, 0.125, 0.0, False, False, seed=L, qmul=1.0,
             what=f"bert L{L}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("T", [1, 7, 32, 65, 130])
def test_decoder_causal_self_attention_bwd(dev, dtype, T):
    """Causal -10000 with T5's decoder bias; T = 65 and 130 put the causal edge across the 64-query / 64-key tiles."""
    H = 12
    g = torch.Generator().manual_seed(T)
    bias = 0.5 * torch.randn(H, 2 * T - 1, generator=g)
    _run_bwd(dev, dtype, 2, H, T, T, None, bias, 1.0, -10000.0, False, False, seed=T + 7, qmul=0.35, what=f"dec T{T}")


# (B, H, T, Lk, split_keys, scale, dead passages of the last row): FiD cross-attention over padded 384-key passages
CROSS_CASES = [
    (1, 12, 1, 192, False, 1.0, None),
    (2, 12, 8, 300, False, 1.0, None),
    (2, 12, 8, 192, True, 1.0, None),            # forced split, one chunk
    (2, 32, 64, 300, True, 1.0, None),           # forced split, two chunks of 3 + 2 blocks
    (1, 32, 32, 1088, True, 1.0, None),          # 5 chunks of 4 blocks, the last of 1
    (2, 12, 65, 1088, False, 1.0, None),         # forced un-split, two query blocks
    (2, 12, 32, 8000, True, 0.125, (6, 12)),     # scale != 1 through the dq_accum atomics
    (2, 12, 32, 15360, True, 1.0, (10, 21)),     # FiD-base training: 11 chunks of 22 blocks, dead chunks
    (1, 32, 64, 15360, True, 1.0, (9, 16)),      # Atlas-xl heads
    (2, 32, 65, 15360, True, 1.0, None),
    (1, 12, 32, 15360, False, 1.0, (10, 21)),    # forced un-split at full length
]
CROSS_IDS = [f"B{c[0]}-H{c[1]}-T{c[2]}-Lk{c[3]}-{'split' if c[4] else 'whole'}" for c in CROSS_CASES]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,T,Lk,split,scale,dead", CROSS_CASES, ids=CROSS_IDS)
def test_cross_attention_bwd(dev, dtype, B, H, T, Lk, split, scale, dead):
    mask = _passage_mask(B, Lk, NEG[dtype], seed=Lk + T, holes=0.1, dead_passages=dead)
    _run_bwd(dev, dtype, B, H, T, Lk, mask, None, scale, 0.0, split, False, seed=Lk + 3 * T + H, qmul=0.4 / scale,
             what=f"cross B{B} H{H} T{T} Lk{Lk} split={split}")


def test_split_key_cases_cover_the_chunk_layouts(dev):
    """The split-key cases above include one chunk, several chunks with a short last one, and a chunk of dead blocks
    only (counted with the launch formula and this device's SM count)."""
    from atlas_b200 import ops

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    one = short_last = dead_chunk = False
    for B, H, T, Lk, split, _, dead in CROSS_CASES + [(b, h, t, lk, True, 1.0, d) for b, h, t, lk, d in DROP_CROSS]:
        if not split:
            continue
        kc = _key_chunks(B, H, T, Lk, sms)
        nkb = (Lk + 63) // 64
        per = (nkb + kc - 1) // kc
        one |= kc == 1
        short_last |= kc > 1 and nkb % per != 0
        live = ops.key_block_live(_passage_mask(B, Lk, -1e9, seed=Lk + T, holes=0.1, dead_passages=dead).to(dev))
        for b in range(B):
            for c in range(kc):
                blocks = live[b, c * per:min(nkb, (c + 1) * per)]
                dead_chunk |= blocks.numel() > 0 and not bool(blocks.any())
    assert one and short_last and dead_chunk, (one, short_last, dead_chunk)


# dropout p = 0.1 with the kernel-exported keep mask in the reference
DROP_CROSS = [(2, 12, 32, 15360, (10, 21))]


@pytest.mark.parametrize("dtype", DTYPES)
def test_dropout_attention_bwd(dev, dtype):
    """An encoder case, and a cross case with dropout + block_live + split_keys (default-dropout FiD training)."""
    g = torch.Generator().manual_seed(3)
    L, H = 384, 12
    bias = 0.5 * torch.randn(H, 2 * L - 1, generator=g)
    _run_bwd(dev, dtype, 3, H, L, L, _length_mask(3, L, seed=5), bias, 1.0, 0.0, False, True, seed=11, qmul=0.35,
             what="dropout enc")
    for B, H, T, Lk, dead in DROP_CROSS:
        mask = _passage_mask(B, Lk, NEG[dtype], seed=Lk + T, holes=0.1, dead_passages=dead)
        _run_bwd(dev, dtype, B, H, T, Lk, mask, None, 1.0, 0.0, True, True, seed=13, qmul=0.4,
                 what=f"dropout cross Lk{Lk}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_grad_ops_wiring_at_fid_size(dev, dtype):
    """grad_ops.cross_attention / self_attention with the mask's `_atlas_block_live` attached as fid.py does: the
    gradients of q, kv (split keys, dead blocks) and qkv, bias (dbias) against the oracle fed the kernels' own O."""
    from atlas_b200 import grad_ops, ops

    B, H, T, Lk = 2, 12, 32, 15360
    g = torch.Generator().manual_seed(77)
    q = (torch.randn(B * T, H * 64, generator=g) * 0.4).to(dtype).to(dev).requires_grad_()
    kv = torch.randn(B * Lk, 2 * H * 64, generator=g).to(dtype).to(dev).requires_grad_()
    mask = _passage_mask(B, Lk, NEG[dtype], seed=5, holes=0.1, dead_passages=(10, 21)).to(dev)
    mask._atlas_block_live = ops.key_block_live(mask)
    dout = torch.randn(B * T, H * 64, generator=g).to(dtype).to(dev)
    out = grad_ops.cross_attention(q, kv, B, H, T, Lk, add_mask=mask)
    out.backward(dout)
    Q = q.detach().double().view(B, T, H, 64)
    K, V = (t.reshape(B, Lk, H, 64) for t in kv.detach().double().split(H * 64, dim=1))
    ref = abo.attention_bwd(Q, K, V, out.detach().double().view(B, T, H, 64), dout.double().view(B, T, H, 64), mask,
                            dtype=dtype)
    _assert_within(q.grad, ref["dq"].reshape(B * T, -1), ref["dq_bound"].reshape(B * T, -1), "grad_ops cross dq")
    gk, gv = kv.grad.split(H * 64, dim=1)
    _assert_within(gk, ref["dk"].reshape(B * Lk, -1), ref["dk_bound"].reshape(B * Lk, -1), "grad_ops cross dk")
    _assert_within(gv, ref["dv"].reshape(B * Lk, -1), ref["dv_bound"].reshape(B * Lk, -1), "grad_ops cross dv")

    S, L = 4, 384
    qkv = (torch.randn(S * L, 3 * H * 64, generator=g) * 0.35).to(dtype).to(dev).requires_grad_()
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev).requires_grad_()
    amask = _length_mask(S, L, seed=9).to(dev)
    amask._atlas_block_live = ops.key_block_live(amask)
    dout = torch.randn(S * L, H * 64, generator=g).to(dtype).to(dev)
    out = grad_ops.self_attention(qkv, S, H, L, add_mask=amask, bias_delta=bias)
    out.backward(dout)
    Qs, Ks, Vs = (t.reshape(S, L, H, 64) for t in qkv.detach().double().split(H * 64, dim=1))
    ref = abo.attention_bwd(Qs, Ks, Vs, out.detach().double().view(S, L, H, 64), dout.double().view(S, L, H, 64), amask,
                            bias.detach(), dtype=dtype)
    gq, gk, gv = qkv.grad.split(H * 64, dim=1)
    for name, got in (("dq", gq), ("dk", gk), ("dv", gv)):
        _assert_within(got, ref[name].reshape(S * L, -1), ref[name + "_bound"].reshape(S * L, -1), f"grad_ops self {name}")
    _assert_within(bias.grad, ref["dbias"], ref["dbias_bound"], "grad_ops self dbias")


def _lse_bound(mag, p, lse):
    """fp32 log-sum-exp: 1e-5 for the exponentials and the sum, plus the P-weighted fp32 error of the scores (2^-21 of
    the magnitude of their terms) and the rounding of lse itself."""
    return 1e-5 + 2.0 ** -21 * (p * mag).sum(-1) + 2.0 ** -22 * lse.abs()


@pytest.mark.parametrize("dtype", DTYPES)
def test_forward_lse_matches_fp64(dev, dtype):
    """The log-sum-exp the backward consumes, from each forward that produces it: ops.attention(return_lse=True), the
    split kernel + combine, and the stream kernel + combine."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(21)
    # encoder self-attention with bias and mask; decoder causal self-attention
    for B, H, L, causal in ((3, 12, 384, 0.0), (2, 12, 65, -10000.0)):
        qkv = (torch.randn(B * L, 3 * H * 64, generator=g) * 0.5).to(dtype).to(dev)
        bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev)
        mask = _length_mask(B, L, seed=L).to(dev) if not causal else None
        _, lse = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, B, H, L, L, add_mask=mask, bias_delta=bias,
                               causal_value=causal, return_lse=True)
        q, k, _ = (t.reshape(B, L, H, 64) for t in qkv.double().split(H * 64, dim=1))
        for b in range(B):
            s, mag = abo._scores(q, k, mask, bias, 1.0, causal, b)
            l64 = torch.logsumexp(s, -1)
            _assert_within(lse[b], l64, _lse_bound(mag, torch.exp(s - l64[..., None]), l64), f"attention lse L{L}")
    # cross-attention: split kernel (T > 64, or Lk < 1024) and stream kernel (T <= 64, Lk >= 1024)
    for B, H, T, Lk, split in ((2, 12, 65, 1536, 384), (2, 12, 8, 768, 384), (2, 12, 32, 15360, 384), (1, 32, 1, 3072, 384)):
        q = (torch.randn(B * T, H * 64, generator=g) * 0.4).to(dtype).to(dev)
        kv = torch.randn(B * Lk, 2 * H * 64, generator=g).to(dtype).to(dev)
        mask = _passage_mask(B, Lk, NEG[dtype], seed=T, holes=0.1).to(dev)
        _, lse = ops.cross_attention_split(q, 0, kv, 0, H * 64, B, H, T, Lk, add_mask=mask, split=split, return_lse=True)
        Q = q.double().view(B, T, H, 64)
        K = kv[:, :H * 64].double().view(B, Lk, H, 64)
        for b in range(B):
            s, mag = abo._scores(Q, K, mask, None, 1.0, 0.0, b)
            l64 = torch.logsumexp(s, -1)
            _assert_within(lse[b], l64, _lse_bound(mag, torch.exp(s - l64[..., None]), l64), f"cross lse T{T} Lk{Lk}")


# ------------------------------------------------------------------------------------------------------------------------
# Part B. csrc/backward.cu
# ------------------------------------------------------------------------------------------------------------------------
def _sum_depth(rows, sms):
    """Longest chain of fp32 additions in the norm kernel's dw / db: rows per warp, then the shared and global atomics."""
    grid = min((rows + 7) // 8, 4 * sms)
    return (rows + grid * 8 - 1) // (grid * 8) * 8 + grid + 8


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("H", [520, 768, 776, 1024, 1032, 2048])
def test_layernorm_bwd_matches_fp64(dev, dtype, kind, H):
    """dx = rs (dxn - m1) - rs^2 x m2 (+ dres), dw = sum dy r16(xn), db = sum dy, from strided row views.  H hits 3, 4
    and 8 vectors per lane, ragged lanes, register and shared-atomic accumulation; 4301 and 30720 rows take more than one
    grid-stride sweep."""
    from atlas_b200 import ops

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    u, sub = UNIT[dtype], SUB[dtype]
    eps = 1e-12 if kind == 0 else 1e-6
    g = torch.Generator().manual_seed(H + kind)
    w16 = (1.0 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(dev)
    for n, rows in enumerate((1, 333, 4224 + 77, 30720)):
        xbuf = torch.zeros((rows, H + 24), dtype=dtype, device=dev)
        xbuf[:, 8:8 + H] = (torch.randn(rows, H, generator=g) * 1.5 + 0.3).to(dtype).to(dev)
        dybuf = torch.zeros((rows, H + 16), dtype=dtype, device=dev)
        dybuf[:, :H] = torch.randn(rows, H, generator=g).to(dtype).to(dev)
        x, dy = xbuf[:, 8:8 + H], dybuf[:, :H]
        dres = torch.randn(rows, H, generator=g).to(dtype).to(dev) if n % 2 else None
        dx, dw, db = ops.layernorm_bwd(x, dy, w16, eps, kind, dres=dres)

        xd, dyd, wd = x.double(), dy.double(), w16.double()
        mean = xd.mean(-1, keepdim=True) if kind == 0 else torch.zeros_like(xd[:, :1])
        rs = torch.rsqrt((xd * xd).mean(-1, keepdim=True) + eps)
        xn = (xd - mean) * rs
        dxn = dyd * wd
        m1 = dxn.mean(-1, keepdim=True) if kind == 0 else torch.zeros_like(mean)
        m2 = (dxn * xn).mean(-1, keepdim=True)
        ref = rs * (dxn - m1) - rs * rs * xd * m2
        if dres is not None:
            ref = ref + dres.double()
        # fp32 headroom on every product / sum that makes up dx (including the cancellation of its two terms)
        xn_mag = rs * (xd.abs() + mean.abs())
        acc = abo.C32 * (rs * (dxn.abs() + dxn.abs().mean(-1, keepdim=True))
                         + rs * rs * xd.abs() * ((dxn.abs() * xn_mag).mean(-1, keepdim=True) + m2.abs()))
        _assert_within(dx, ref, acc + (u + F32) * (ref.abs() + acc) + sub, f"dx kind{kind} H{H} rows{rows}")
        depth = _sum_depth(rows, sms) * 2.0 ** -24
        # dw sums dy r16(xn): one 16-bit rounding of each xn (taken at the fp64 xn, plus its fp32 error)
        dw_ref = (dyd * xn).sum(0)
        dw_bound = (dyd.abs() * ((u + abo.C32) * xn.abs() + abo.C32 * xn_mag + sub)).sum(0) \
            + depth * (dyd * xn).abs().sum(0)
        _assert_within(dw, dw_ref, dw_bound, f"dw kind{kind} H{H} rows{rows}")
        if kind == 0:
            _assert_within(db, dyd.sum(0), depth * dyd.abs().sum(0) + 1e-30, f"db H{H} rows{rows}")
        else:
            assert db is None


def _ce_case(V, rows, dtype, g):
    x = torch.randn(rows, V, generator=g) * 3.0
    labels = torch.randint(0, V, (rows,), generator=g)
    labels[0] = 0
    if rows > 1:
        labels[1] = V - 1
    if rows > 3:
        labels[2::7] = -100
        x[3, labels[3] if labels[3] >= 0 else 0] += 70.0           # peaked: spread above 60
        x[3] -= 30.0
    if rows > 5:
        big = 6.0e4 if dtype == torch.float16 else 1.0e38     # the loss (up to 2 big) stays finite in fp32
        x[5, :] = -big * torch.rand(V, generator=g)                 # near the top of the range, both signs
        x[5, V // 2] = big
    if rows > 6:
        x[6, :] = 0.0                                               # uniform row
    return x.to(dtype), labels


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("V", [2, 512, 32128])
@pytest.mark.parametrize("rows", [1, 19, 256])
def test_cross_entropy_matches_fp64(dev, dtype, V, rows):
    """lse within an fp32 bound of the fp64 logsumexp; loss = lse - x[label] (0 at -100); dlogits = (softmax -
    onehot) gscale within one 16-bit rounding plus P |lse_kernel - lse64|.  Labels 0 and V - 1, ignored rows, peaked
    rows, near-overflow logits."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(V + rows)
    x16, labels = _ce_case(V, rows, dtype, g)
    xbuf = torch.zeros((rows, V + 8), dtype=dtype, device=dev)
    xbuf[:, :V] = x16.to(dev)
    logits = xbuf[:, :V]
    lab = labels.to(dev)
    lse, loss = ops.cross_entropy_fwd(logits, lab)
    xd = x16.double().to(dev)
    l64 = torch.logsumexp(xd, -1)
    P = torch.exp(xd - l64[:, None])
    mx = xd.amax(-1, keepdim=True)
    depth = (V + 255) // 256 + 16
    lse_bound = 2.0 ** -24 * depth + 2.0 ** -23 * (P * (xd - mx).abs()).sum(-1) + 2.0 ** -23 * l64.abs()
    _assert_within(lse, l64, lse_bound, f"ce lse V{V} rows{rows}")
    valid = lab >= 0
    xy = xd.gather(1, lab.clamp_min(0)[:, None])[:, 0]
    loss_ref = torch.where(valid, l64 - xy, torch.zeros_like(l64))
    _assert_within(loss, loss_ref, torch.where(valid, lse_bound + 2.0 ** -23 * loss_ref.abs(), torch.zeros_like(l64)) + 1e-300,
                   f"ce loss V{V} rows{rows}")
    assert bool((loss[~valid] == 0).all())
    if V % 2:
        return
    gs = torch.tensor([1.7 / max(1, int(valid.sum()))], dtype=torch.float32, device=dev)
    dl = ops.cross_entropy_bwd(logits, lab, lse, gs)
    onehot = torch.zeros_like(xd)
    onehot[valid] = torch.nn.functional.one_hot(lab[valid], V).double()
    gsd = float(gs)
    ref = (P - onehot) * gsd * valid[:, None]
    dlse = (lse.double() - l64).abs()[:, None]
    acc = gsd * (P * (dlse + 2.0 ** -22 * ((xd - l64[:, None]).abs() + 1.0)) + 2.0 ** -23 * (P + onehot))
    bound = (acc + (UNIT[dtype] + F32) * (ref.abs() + acc) + SUB[dtype]) * valid[:, None] + 1e-300
    _assert_within(dl, ref, bound, f"ce dlogits V{V} rows{rows}")
    assert bool((dl[~valid] == 0).all())


@pytest.mark.parametrize("dtype", DTYPES)
def test_scatter_add_rows_and_colsum_exact(dev, dtype):
    """Exact-grid inputs (multiples of 1/8 in [-2, 2]) keep every fp32 partial sum exact in any atomic order, so the
    results must match the fp64 sums bit for bit: one table row hit 4000 times, skip_index, out-of-range ids, the
    modulo mode; colsum over up to 30720 rows."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(3)
    rows, H, table = 6000, 768, 300
    src = (torch.randint(-16, 17, (rows, H), generator=g).float() / 8).to(dtype)
    sbuf = torch.zeros((rows, H + 16), dtype=dtype, device=dev)
    sbuf[:, 8:8 + H] = src.to(dev)
    s = sbuf[:, 8:8 + H]
    idx = torch.randint(0, table, (rows,), generator=g)
    idx[:4000] = 7
    idx[4000:4100] = 0                      # the skipped (padding) id
    idx[4100:4150] = -3                     # out of range below
    idx[4150:4200] = table + 5              # out of range above
    idx = idx[torch.randperm(rows, generator=g)]
    got = ops.scatter_add_rows(s, table, index=idx.to(dev), skip_index=0)
    keep = (idx != 0) & (idx >= 0) & (idx < table)
    want = torch.zeros((table, H), dtype=torch.float64).index_add_(0, idx[keep], src.double()[keep])
    assert torch.equal(got.cpu(), want.float())
    assert float(got[7].abs().sum()) > 0 and float(got[0].abs().sum()) == 0.0
    L = 37
    got = ops.scatter_add_rows(s, L, modulo=L)
    want = torch.zeros((L, H), dtype=torch.float64).index_add_(0, torch.arange(rows) % L, src.double())
    assert torch.equal(got.cpu(), want.float())
    for M in (1, 255, 257, 30720):
        x = (torch.randint(-16, 17, (M, 2 * H), generator=g).float() / 8).to(dtype)
        xb = torch.zeros((M, 2 * H + 8), dtype=dtype, device=dev)
        xb[:, :2 * H] = x.to(dev)
        assert torch.equal(ops.colsum(xb[:, :2 * H]).cpu(), x.double().sum(0).float()), M


@pytest.mark.parametrize("dtype", DTYPES)
def test_masked_mean_pool_bwd_within_one_rounding(dev, dtype):
    """dx[b, l] = demb[b] / count[b] on live tokens, 0 elsewhere: rows with one, some and all tokens live."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(4)
    B, L, H = 6, 512, 768
    counts = torch.tensor([1, L, 7, 300, 1, 511])
    mask = torch.zeros(B, L, dtype=torch.int64)
    for b, c in enumerate(counts.tolist()):
        mask[b, torch.randperm(L, generator=g)[:c]] = 1
    mask[4] = 0
    mask[4, L - 1] = 1                                  # the only live token is the last one
    dbuf = torch.zeros((B, H + 32), dtype=dtype, device=dev)
    dbuf[:, 16:16 + H] = (torch.randn(B, H, generator=g) * 3).to(dtype).to(dev)
    demb = dbuf[:, 16:16 + H]
    dx = ops.masked_mean_pool_bwd(demb, mask.to(dev), L, H)
    live = mask.to(dev).bool()[..., None]
    ref = torch.where(live, (demb.double() / counts.to(dev)[:, None].double())[:, None, :], torch.zeros((), device=dev,
                                                                                                    dtype=torch.float64))
    bound = (UNIT[dtype] + 2.0 ** -22) * ref.abs() + SUB[dtype]
    _assert_within(dx, ref, torch.where(live, bound, torch.full_like(bound, 1e-300)), "pool bwd")
    assert bool((dx[~live.expand_as(dx)] == 0).all())


def _gelu_new(x):
    c, a = math.sqrt(2.0 / math.pi), 0.044715
    u = c * (x + a * x ** 3)
    t = torch.tanh(u)
    y = 0.5 * x * (1.0 + t)
    dy = 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * c * (1.0 + 3.0 * a * x * x)
    # fp32 error: tanhf and the rounding of u (|du| ~ 2^-22 |u|) move t by up to 2^-22 (1 + |u| (1 - t^2)) + 2^-23
    et = 2.0 ** -22 * (1.0 + u.abs() * (1.0 - t * t)) + 2.0 ** -23
    ey = 0.5 * x.abs() * et + 2.0 ** -22 * y.abs()
    edy = 0.5 * et + x.abs() * t.abs() * et * c * (1.0 + 3.0 * a * x * x) + 2.0 ** -21 * (
        0.5 * (1.0 + t).abs() + 0.5 * x.abs() * (1.0 - t * t) * c * (1.0 + 3.0 * a * x * x))
    return y, dy, ey, edy


def _gelu_erf(z):
    w = z / math.sqrt(2.0)
    p = 0.5 * (1.0 + torch.erf(w))
    phi = torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)
    # erff (+ the rounding of z / sqrt 2) and __expf (relative 2^-21 + 2^-22 |argument|)
    ep = 2.0 ** -22 * (1.0 + w.abs() * torch.exp(-w * w) * 1.13) + 2.0 ** -23
    ey = z.abs() * ep + 2.0 ** -22 * (z * p).abs()
    edy = ep + z.abs() * phi * (2.0 ** -21 + 2.0 ** -22 * 0.5 * z * z) + 2.0 ** -22 * (p + (z * phi).abs())
    return z * p, p + z * phi, ey, edy


@pytest.mark.parametrize("dtype", DTYPES)
def test_gated_gelu_and_gelu_erf_match_fp64(dev, dtype):
    """|x| up to 10, where tanh and erf saturate: each output within one 16-bit rounding plus the fp32 transcendental
    error (the gated forward keeps its second rounding: g = r16(r16(gelu_new(u0)) u1))."""
    from atlas_b200 import ops

    u_, sub = UNIT[dtype], SUB[dtype]
    g = torch.Generator().manual_seed(8)
    M, F = 300, 512
    xs = torch.linspace(-10.0, 10.0, M * F)[torch.randperm(M * F, generator=g)].view(M, F)
    u16 = torch.stack([xs, torch.randn(M, F, generator=g) * 2], -1).reshape(M, 2 * F).to(dtype).to(dev)
    dg16 = torch.randn(M, F, generator=g).to(dtype).to(dev)
    u0, u1, dgd = u16[:, 0::2].double(), u16[:, 1::2].double(), dg16.double()
    y, dy, ey, edy = _gelu_new(u0)
    out = ops.gated_gelu(u16)
    ref = y * u1
    inner = (ey + u_ * (y.abs() + ey) + sub) * u1.abs()
    _assert_within(out, ref, inner + (u_ + F32) * (ref.abs() + inner) + sub + 1e-300, "gated fwd")
    du = ops.gated_gelu(u16, dg16)
    for what, got, r, acc in (("gated bwd du0", du[:, 0::2], dgd * u1 * dy, (dgd * u1).abs() * edy + 2.0 ** -22 * (dgd * u1 * dy).abs()),
                              ("gated bwd du1", du[:, 1::2], dgd * y, dgd.abs() * ey + 2.0 ** -23 * (dgd * y).abs())):
        _assert_within(got, r, acc + (u_ + F32) * (r.abs() + acc) + sub + 1e-300, what)

    z16 = xs.to(dtype).to(dev)
    dz16 = torch.randn(M, F, generator=g).to(dtype).to(dev)
    zd, dzd = z16.double(), dz16.double()
    y, dy, ey, edy = _gelu_erf(zd)
    _assert_within(ops.gelu_erf(z16), y, ey + (u_ + F32) * (y.abs() + ey) + sub + 1e-300, "gelu_erf fwd")
    r = dzd * dy
    acc = dzd.abs() * edy + 2.0 ** -23 * r.abs()
    _assert_within(ops.gelu_erf(z16, dz16), r, acc + (u_ + F32) * (r.abs() + acc) + sub + 1e-300, "gelu_erf bwd")
