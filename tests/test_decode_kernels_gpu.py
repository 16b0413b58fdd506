"""The single-token decode kernels of `FiD.generate` (csrc/decode.cu) and the cross-attention statistics kernel of retriever
distillation (csrc/xattn_stats.cu), each against a float64 reference computed in this file from the same 16-bit inputs the
kernel reads, at the shapes, strides and masks where such kernels go wrong.  Then the decode-step logits of a whole
generation against the fp32 CPU restatement of the reference model (oracle/fid_cpu.py).

Accuracy of the 16-bit outputs: the kernels accumulate in fp32 and round once to 16 bits, so every element is held to one
ulp of the output type at |ref| plus an absolute floor of 1e-5 * max|V| (far below the 2e-3 * max of the layer tests)."""
import math

import pytest
import torch

import fid_cpu
import model_synth

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
NAN_BITS = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0}
# invert_attention_mask (transformers 4.18), as FiD.generate builds the cross-attention mask
NEG = {torch.float16: -1e4, torch.bfloat16: -1e9}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _ulp(ref, dtype):
    """One unit in the last place of `dtype` at |ref| (subnormal spacing below the normal range)."""
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    return torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin))) - mant)


def _assert_within(got, ref, bound, what):
    worst = float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())
    assert worst <= 1.0, f"{what}: max |got - ref| / bound = {worst:.3g}"


def _assert_one_rounding(got, ref, v_absmax, dtype, what):
    _assert_within(got, ref, _ulp(ref, dtype) + 1e-5 * v_absmax, what)


def _nan_filled(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


# ------------------------------------------------------------------------------------------------------------------------
# 1. decode_cross_attention
# ------------------------------------------------------------------------------------------------------------------------
# Per batch row, one kind of additive mask; q is scaled per kind so that some rows are peaked (logit spread above 30).
Q_MULT = {"soft": 2.5, "hard": 3.0, "tiles": 1.0, "last": 1.0, "full": 0.25}


def _cross_mask_row(kind, Lk, neg, g):
    j = torch.arange(Lk)
    if kind == "soft":                  # finite: a missing log2(e) on the mask term changes the weights
        return -4.0 * torch.rand(Lk, generator=g, dtype=torch.float64).float()
    if kind == "hard":                  # random dead keys
        return torch.where(torch.rand(Lk, generator=g) < 0.5, neg, 0.0)
    if kind == "tiles":                 # live keys in some 64-key tiles only: whole 64-, 256- and 1024-key ranges are dead
        region = ((j // 1024) % 2 == 0) & ((j // 256) % 2 == 0) & ((j // 64) % 3 != 1)
        live = region & (torch.rand(Lk, generator=g) < 0.5)
        live[int(region.nonzero()[-1])] = True
        return torch.where(live, 0.0, neg)
    if kind == "last":                  # the only live key is the last one (of a ragged last chunk)
        m = torch.full((Lk,), neg)
        m[-1] = 0.0
        return m
    assert kind == "full"               # every key masked: fp32 scores collapse to the mask, the softmax is uniform
    return torch.full((Lk,), -1e9)


# (Lk, B, H, scale, mask kind of each batch row): Lk ragged against the 16-key groups, the chunks and the 64-key tiles
CROSS_CASES = [
    (1, 2, 12, 1.0, ("soft", "full")),
    (17, 5, 1, 1.0, ("soft", "hard", "tiles", "last", "full")),
    (100, 5, 32, 0.125, ("soft", "hard", "tiles", "last", "full")),
    (2047, 2, 12, 1.0, ("tiles", "last")),
    (2048, 1, 32, 1.0, ("tiles",)),
    (3072 + 40, 5, 12, 1.0, ("soft", "hard", "tiles", "last", "full")),
    (15360, 2, 12, 1.0, ("hard", "tiles")),
]
CHUNKS = (16, 64, 80, 256, 1024)        # 64 and 256 are what FiD._decode_state picks; 1024 > Lk for most cases


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Lk,B,H,scale,kinds", CROSS_CASES, ids=[f"Lk{c[0]}-B{c[1]}-H{c[2]}" for c in CROSS_CASES])
def test_decode_cross_attention_matches_fp64(dev, dtype, Lk, B, H, scale, kinds):
    """softmax(q K^T scale + mask) V for one query per (batch, head), every chunk size, with and without the live-tile
    skip, from strided q / kv / out views whose extra columns hold NaN.  With the skip the result is bit-identical."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(1000 + Lk + 7 * B + H)
    HD = H * 64
    mult = torch.tensor([Q_MULT[k] for k in kinds]) / scale
    q16 = (torch.randn(B, HD, generator=g) * mult[:, None]).to(dtype)
    kv16 = torch.randn(B * Lk, 2 * HD, generator=g).to(dtype)
    qbuf = _nan_filled((B, HD + 72), dtype, dev)          # ldq > H*64, q starts at column 8
    qbuf[:, 8:8 + HD] = q16.to(dev)
    q = qbuf[:, 8:8 + HD]
    kvbuf = _nan_filled((B * Lk, 2 * HD + 64), dtype, dev)  # ldkv > 2*H*64, K | V start at column 64
    kvbuf[:, 64:64 + 2 * HD] = kv16.to(dev)
    kv = kvbuf[:, 64:64 + 2 * HD]
    outbuf = _nan_filled((B, HD + 64), dtype, dev)
    out = outbuf[:, 32:32 + HD]
    mask = torch.stack([_cross_mask_row(k, Lk, NEG[dtype], g) for k in kinds]).to(dev)

    K = kv16[:, :HD].double().view(B, Lk, H, 64).to(dev)
    V = kv16[:, HD:].double().view(B, Lk, H, 64).to(dev)
    s = torch.einsum("bhd,bjhd->bhj", q16.double().view(B, H, 64).to(dev), K) * scale
    v_absmax = float(V.abs().max())

    def ref_of(m):
        logits = s if m is None else s + m.double()[:, None, :]
        o = torch.einsum("bhj,bjhd->bhd", torch.softmax(logits, -1), V)
        if m is not None:
            for b, kind in enumerate(kinds):
                if kind == "full":      # -1e9 swallows every fp32 logit (|s log2 e| < 64 here): uniform, as the reference
                    o[b] = V[b].mean(0)
        return o.reshape(B, HD)

    if Lk > 1:
        assert float((s.amax(-1) - s.amin(-1)).max()) > 30.0     # peaked rows: the online-softmax rescale matters
    for m in (None, mask):
        ref = ref_of(m)
        live = ops.key_block_live(m)
        assert (live is None) == (m is None)
        for chunk in CHUNKS:
            got = {}
            for tl in (None, live) if m is not None else (None,):
                res = ops.decode_cross_attention(q, kv, B, H, Lk, add_mask=m, scale=scale, chunk=chunk, out=out, tile_live=tl)
                assert res.data_ptr() == out.data_ptr()
                got[tl is None] = out.clone()
                _assert_one_rounding(got[tl is None], ref, v_absmax, dtype,
                                     f"mask={m is not None} chunk={chunk} tile_live={tl is not None}")
            if len(got) == 2:
                assert torch.equal(got[True].view(torch.int16), got[False].view(torch.int16)), f"chunk={chunk}"
    assert bool(outbuf[:, :32].isnan().all()) and bool(outbuf[:, 32 + HD:].isnan().all())


# ------------------------------------------------------------------------------------------------------------------------
# 2. decode_self_attention
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Tmax,bias,scale", [(1, 9, True, 1.0), (12, 1, True, 1.0), (12, 64, True, 1.0),
                                               (32, 130, True, 1.0), (12, 9, False, 0.5)])
def test_decode_self_attention_steps_match_fp64(dev, dtype, H, Tmax, bias, scale):
    """Step t = 0 .. Tmax-1 as `generate` runs it (t in device memory): the new K | V lands in cache row t bit for bit,
    the other rows keep their bits (unwritten rows a NaN pattern that would poison any read past t), and the output is
    causal attention over rows 0..t with T5's unidirectional relative-position bias.  A captured CUDA graph of one step
    plus a device-side t += 1, replayed Tmax times, reproduces the eager outputs bit for bit."""
    from atlas_b200 import ops
    from atlas_b200.fid import bias_by_delta

    B, HD = 3, H * 64
    g = torch.Generator().manual_seed(17 * H + Tmax)
    w = torch.randn(32, H, generator=g) * 2.0                         # relative_attention_bias.weight [buckets, H]
    bias_delta = bias_by_delta(w.to(dev), Tmax, Tmax, False, 32) if bias else None
    pos_bias = fid_cpu.position_bias(w, Tmax, Tmax, False, 32)[0].double().to(dev)     # [H, Tmax, Tmax], built apart
    rows16 = torch.randn(Tmax, B, 3 * HD, generator=g)
    rows16[:, :, :HD] *= 3.0                                          # peaked rows
    rows16 = rows16.to(dtype).to(dev)
    cache = torch.empty((B, Tmax, 2 * HD), dtype=dtype, device=dev)
    qkvbuf = _nan_filled((B, 3 * HD + 64), dtype, dev)
    qkv = qkvbuf[:, 64:]
    outbuf = _nan_filled((B, HD + 64), dtype, dev)
    out = outbuf[:, 32:32 + HD]
    t_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    cache.view(torch.int16).fill_(NAN_BITS[dtype])

    eager = []
    for t in range(Tmax):
        qkv.copy_(rows16[t])
        t_dev.fill_(t)
        before = cache.clone()
        ops.decode_self_attention(qkv, cache, t_dev, H, bias_delta=bias_delta, scale=scale, out=out)
        eager.append(out.clone())
        c16 = cache.view(torch.int16)
        assert torch.equal(c16[:, t], rows16[t, :, HD:].contiguous().view(torch.int16)), t
        assert torch.equal(c16[:, :t], before.view(torch.int16)[:, :t]), t
        assert bool((c16[:, t + 1:] == NAN_BITS[dtype]).all()), t
        qd = rows16[t, :, :HD].double().view(B, H, 64)
        K = rows16[:t + 1, :, HD:2 * HD].double().view(t + 1, B, H, 64)
        V = rows16[:t + 1, :, 2 * HD:].double().view(t + 1, B, H, 64)
        logits = torch.einsum("bhd,jbhd->bhj", qd, K) * scale
        if bias:
            logits = logits + pos_bias[None, :, t, :t + 1]
        ref = torch.einsum("bhj,jbhd->bhd", torch.softmax(logits, -1), V).reshape(B, HD)
        _assert_one_rounding(eager[-1], ref, float(V.abs().max()), dtype, f"t={t}")
    assert bool(outbuf[:, :32].isnan().all()) and bool(outbuf[:, 32 + HD:].isnan().all())

    cache.view(torch.int16).fill_(NAN_BITS[dtype])
    t_dev.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decode_self_attention(qkv, cache, t_dev, H, bias_delta=bias_delta, scale=scale, out=out)
        t_dev.add_(1)
    for t in range(Tmax):
        qkv.copy_(rows16[t])
        graph.replay()
        assert torch.equal(out.view(torch.int16), eager[t].view(torch.int16)), t
    assert int(t_dev) == Tmax


# ------------------------------------------------------------------------------------------------------------------------
# 3. decode_argmax
# ------------------------------------------------------------------------------------------------------------------------
EOS, PAD = 1, 0


def _greedy_ref(logits, t, min_length, done):
    """transformers 4.18 greedy_search on one step: EOS banned while t + 1 < min_length, torch.argmax (first NaN, else the
    lowest index of the maximum), finished rows emit pad."""
    x = logits.double().cpu().clone()
    if t + 1 < min_length and x.shape[1] > EOS:
        x[:, EOS] = -math.inf
    nxt = x.argmax(-1)
    return torch.where(done.cpu().bool(), torch.full_like(nxt, PAD), nxt)


def _argmax_state(B, T, dev):
    seq = torch.full((B, T), -7, dtype=torch.int64, device=dev)
    tok_in = torch.full((B,), -7, dtype=torch.int64, device=dev)
    done = torch.zeros(B, dtype=torch.uint8, device=dev)
    t_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    return seq, tok_in, done, t_dev


def _step_logits(B, V, t, dtype, g):
    """Random finite logits with the maximum planted at several indices owned by different threads, EOS-heavy rows (the
    ban must hold them off until min_length), and a row whose only finite entry is the banned EOS (picks 0)."""
    x = torch.randn(B, V, generator=g)
    ties = [[3, 259, 31000], [255, 256], [100, 7], [V - 1, V // 2], [24, 31000, 4000]]
    for b in range(B):
        idx = [i for i in ties[(b + t) % len(ties)] if i < V]
        x[b, idx] = 8.0
    for b in range(2, B, 5):
        x[b, EOS % V] = 9.0
    if B > 4:
        x[4] = -math.inf
        x[4, EOS % V] = 9.0
    return x.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("V", [1, 7, 255, 256, 257, 32128])
def test_decode_argmax_matches_torch_argmax(dev, dtype, V):
    """Greedy pick from a strided logits view (columns past V hold a larger value that must never win), eager and under
    graph replay with 65 blocks: lowest index among ties, EOS ban, pad after done; only seq[:, t+1] changes, tok_in is the
    new token, t advances by one per call."""
    from atlas_b200 import ops

    B, T, min_length = 65, 7, 4
    g = torch.Generator().manual_seed(V)
    for graphed in (False, True):
        seq, tok_in, done, t_dev = _argmax_state(B, T, dev)
        done[5::7] = 1                                                # rows already finished
        buf = torch.full((B, V + 5), 6e4, dtype=dtype, device=dev)
        logits = buf[:, :V]
        if graphed:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                ops.decode_argmax(logits, seq, tok_in, done, t_dev, EOS, PAD, min_length)
        want_seq = seq.cpu().clone()
        want_done = done.cpu().clone()
        for t in range(T - 1):
            step = _step_logits(B, V, t, dtype, g)
            logits.copy_(step)
            if graphed:
                graph.replay()
            else:
                ops.decode_argmax(logits, seq, tok_in, done, t_dev, EOS, PAD, min_length)
            nxt = _greedy_ref(step, t, min_length, want_done)
            want_seq[:, t + 1] = nxt
            want_done |= (nxt == EOS).to(torch.uint8)
            assert torch.equal(seq.cpu(), want_seq), (graphed, t)
            assert torch.equal(tok_in.cpu(), nxt), (graphed, t)
            assert torch.equal(done.cpu(), want_done), (graphed, t)
            assert int(t_dev) == t + 1, (graphed, t)
        if V > EOS:
            assert bool(want_done[2::5].all())                        # EOS won once the ban lifted (t + 1 == min_length)
        if V > 3:
            assert int(want_seq[4, min_length - 1]) == 0               # all -inf after the EOS ban: index 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_decode_argmax_nan_rows_pick_the_first_nan(dev, dtype):
    """torch.argmax semantics on NaN: the first NaN wins over any number, an all-NaN row picks 0 (never an out-of-vocabulary
    sentinel); a NaN at a banned EOS is ignored.  Only the returned ids are read."""
    from atlas_b200 import ops

    nan, inf = float("nan"), math.inf
    small = torch.tensor([[1, nan, 5, nan], [nan] * 4, [-inf] * 4, [2, 7, 7, 1], [3, 2, 1, nan]])
    g = torch.Generator().manual_seed(5)
    big = torch.randn(6, 32128, generator=g)
    big[0, [300, 20000]] = nan
    big[0, 5] = 50.0
    big[1] = nan
    big[2, 31999] = nan
    big[3, [EOS, 17]] = nan                                           # EOS banned below: 17 wins
    big[4, EOS] = nan                                                 # EOS banned below: the maximum wins
    big[5, 256:] = nan
    for x, min_length in ((small, 0), (big, 3)):
        x = x.to(dtype)
        B = x.shape[0]
        seq, tok_in, done, t_dev = _argmax_state(B, 3, dev)
        ld_buf = torch.zeros((B, x.shape[1] + 3), dtype=dtype, device=dev)
        ld_buf[:, :x.shape[1]] = x.to(dev)
        ops.decode_argmax(ld_buf[:, :x.shape[1]], seq, tok_in, done, t_dev, EOS, PAD, min_length)
        want = _greedy_ref(x, 0, min_length, torch.zeros(B, dtype=torch.bool))
        assert tok_in.cpu().tolist() == want.tolist() and seq[:, 1].cpu().tolist() == want.tolist()
    assert _greedy_ref(small.to(dtype), 0, 0, torch.zeros(5, dtype=torch.bool)).tolist() == [1, 0, 0, 1, 3]


# ------------------------------------------------------------------------------------------------------------------------
# 4. cross_attention_stats
# ------------------------------------------------------------------------------------------------------------------------
# (T, Lk, H, B, scale): the second to fourth 32-query blocks, a ragged last 32-key block
STATS_CASES = [
    (1, 31, 1, 3, 1.0),
    (8, 1920, 12, 3, 1.0),
    (32, 100, 32, 3, 0.125),
    (33, 32, 12, 1, 1.0),
    (100, 15360, 12, 1, 1.0),
    (128, 1920, 32, 3, 1.0),
]


def _split_of(Lk):
    """Key segments of FiD's split-KV cross-attention (fid.py: the largest divisor of Lk up to 384, else up to 512)."""
    return next((s for s in range(min(384, Lk), 63, -1) if Lk % s == 0), None) or \
        next(s for s in range(min(512, Lk), 0, -1) if Lk % s == 0)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("T,Lk,H,B,scale", STATS_CASES, ids=[f"T{c[0]}-Lk{c[1]}-H{c[2]}-B{c[3]}" for c in STATS_CASES])
def test_cross_attention_stats_matches_fp64(dev, dtype, T, Lk, H, B, scale):
    """The head means of S = q K^T scale + mask, P = exp(S - lse) and ||V|| P (src/fid.py:333-343) in fp64, with V before K
    and extra columns in the kv rows, q at a column offset, soft / hard / fully masked rows, and lse from fp64 and from
    the production attention (fid.py passes the cross-attention's own lse).  fp32 outputs without a 16-bit rounding:
    the bound is the fp32 arithmetic's, about 1e-5 relative, plus the rounding of the mask-sized terms."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(31 * T + Lk + H)
    HD = H * 64
    q_col0, v_col0 = 16, 8
    k_col0 = v_col0 + HD + 16
    qbuf = _nan_filled((B * T, q_col0 + HD + 8), dtype, dev)
    q16 = (torch.randn(B * T, HD, generator=g) * 2.0).to(dtype)
    qbuf[:, q_col0:q_col0 + HD] = q16.to(dev)
    kvbuf = _nan_filled((B * Lk, k_col0 + HD + 24), dtype, dev)
    k16 = torch.randn(B * Lk, HD, generator=g).to(dtype)
    v16 = torch.randn(B * Lk, HD, generator=g).to(dtype)
    kvbuf[:, k_col0:k_col0 + HD] = k16.to(dev)
    kvbuf[:, v_col0:v_col0 + HD] = v16.to(dev)
    # row 0 soft, row 1 hard with dead keys, row 2 fully masked at -1e4 (at -1e9 the fp32 logits and lse cannot resolve
    # the row at all, see the precision note in csrc/xattn_stats.cu)
    kinds = ("soft", "hard", "full")[:B] if B > 1 else ("hard",)
    rows = []
    for kind in kinds:
        if kind == "soft":
            rows.append(-4.0 * torch.rand(Lk, generator=g))
        elif kind == "hard":
            r = torch.where(torch.rand(Lk, generator=g) < 0.4, -1e9, 0.0)
            r[0] = 0.0
            rows.append(r)
        else:
            rows.append(torch.full((Lk,), -1e4))
    mask = torch.stack(rows).to(dev)

    Q = q16.double().view(B, T, H, 64).to(dev)
    K = k16.double().view(B, Lk, H, 64).to(dev)
    Vd = v16.double().view(B, Lk, H, 64).to(dev)
    S = torch.einsum("bthd,bjhd->bhtj", Q, K) * scale + mask.double()[:, None, None, :]
    D = torch.einsum("bthd,bjhd->bhtj", Q.abs(), K.abs()) * scale         # magnitude of the dot products' terms
    lse64 = torch.logsumexp(S, -1)
    vn = Vd.norm(dim=-1).permute(0, 2, 1)[:, :, None, :]                  # ||V[b, j, h, :]|| as [B, H, 1, Lk]

    _, lse_prod = ops.cross_attention_split(qbuf, q_col0, kvbuf, k_col0, v_col0, B, H, T, Lk, add_mask=mask, scale=scale,
                                            split=_split_of(Lk), return_lse=True)
    hard_dead = (mask <= -1e8)[:, None, :].expand(B, T, Lk)
    has_live = (mask > -5000).any(-1)
    for name, lse in (("fp64 lse", lse64), ("attention lse", lse_prod.double())):
        got_s, got_p, got_n = ops.cross_attention_stats(qbuf, q_col0, kvbuf, k_col0, v_col0, B, H, T, Lk, lse.float(),
                                                        add_mask=mask, scale=scale)
        P = torch.exp(S - lse[..., None])
        # per-element relative error of P from fp32: the dot products, the rounding of the mask-sized S and lse, __expf
        rel = 1e-5 + 2.0 ** -21 * D + 2.0 ** -22 * (S.abs() + lse.abs()[..., None])
        for what, got, ref, tol in (
                ("scores", got_s, S.mean(1), 1e-5 * (D + mask.double().abs()[:, None, None, :]).mean(1)),
                ("probs", got_p, P.mean(1), (P * rel).mean(1)),
                ("norms", got_n, (vn * P).mean(1), (vn * P * rel).mean(1))):
            _assert_within(got, ref, tol, f"{name} {what}")
        sums = got_p.double().sum(-1)[has_live]
        assert float((sums - 1.0).abs().max()) <= 1e-4, name
        for got in (got_p, got_n):
            assert float(torch.where(hard_dead, got.abs(), 0.0).max()) <= 1e-6, name


def test_cross_attention_stats_rejects_more_than_128_queries(dev):
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    B, H, T, Lk = 1, 2, 129, 64
    q = torch.zeros((B * T, H * 64), dtype=torch.bfloat16, device=dev)
    kv = torch.zeros((B * Lk, 2 * H * 64), dtype=torch.bfloat16, device=dev)
    lse = torch.zeros((B, H, T), dtype=torch.float32, device=dev)
    with pytest.raises(AtlasB200Error, match="T <= 128"):
        ops.cross_attention_stats(q, 0, kv, 0, H * 64, B, H, T, Lk, lse)


# ------------------------------------------------------------------------------------------------------------------------
# 5. decode-step logits of a whole generation against the fp32 CPU oracle
# ------------------------------------------------------------------------------------------------------------------------
def _passages(B, n_ctx, L, lens, vocab, seed):
    """Token rows closed by EOS like the reader's tokenizer; a length-1 passage holds only EOS."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, vocab, (B, n_ctx, L), generator=g)
    lens = torch.tensor(lens).view(B, n_ctx)
    mask = torch.arange(L)[None, None, :] < lens[..., None]
    ids = ids * mask
    ids.scatter_(2, (lens - 1)[..., None], EOS)
    return ids.view(B, n_ctx * L), mask.view(B, n_ctx * L)


# (n_ctx, L, passage lengths): Lk = 384 decodes with chunk 64, Lk = 3072 with chunk 256; short passages leave dead
# 64-key tiles and dead chunks, and one passage per row holds only EOS
GEN_CASES = [
    (3, 128, [5, 128, 1, 40, 2, 1]),
    (8, 384, [12, 1, 60, 7, 33, 2, 64, 20, 1, 3, 45, 9, 30, 18, 5, 61]),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n_ctx,L,lens", GEN_CASES, ids=["Lk384", "Lk3072"])
def test_generate_step_logits_match_cpu_oracle(dev, dtype, n_ctx, L, lens):
    """Every generated token is torch.argmax of that step's logits under the EOS ban and pad rules (no near-tie exemption),
    and the step logits are as close to the fp32 oracle's teacher-forced logits as the GPU's own teacher-forced forward
    is (within 2x)."""
    from atlas_b200.fid import FiD, T5ConfigLite

    cfg = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    model = FiD(T5ConfigLite(**cfg))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    model = model.to(dtype).to(dev).eval()
    model.cuda_graphs = False
    B, min_length = 2, 4
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    ids, mask = _passages(B, n_ctx, L, lens, cfg["vocab_size"], seed=n_ctx)
    steps = []
    decode_step = model._decode_step_logits

    def recording(st):
        logits = decode_step(st)
        steps.append(logits.clone())
        return logits

    model._decode_step_logits = recording
    with torch.no_grad():
        seq = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), max_length=12, min_length=min_length)
    n = min(len(steps), seq.shape[1] - 1)
    assert n >= min_length
    done = torch.zeros(B, dtype=torch.bool)
    for t in range(n):
        nxt = _greedy_ref(steps[t], t, min_length, done)
        assert seq[:, t + 1].cpu().tolist() == nxt.tolist(), t
        done |= nxt == EOS

    dec_in = seq[:, :n]
    with torch.no_grad():
        tf = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), decoder_input_ids=dec_in, use_cache=False)
    _, ref, _ = fid_cpu.fid_forward({k: v.float() for k, v in sd.items()}, model_synth.T5_CFG, ids, mask, dec_in.cpu(),
                                    n_context=n_ctx)
    got = torch.stack(steps[:n], 1).float().cpu()
    err_step = float((got - ref).abs().max())
    err_tf = float((tf.logits.float().cpu() - ref).abs().max())
    print(f"max |logits - fp32 oracle|: decode steps {err_step:.3g}, teacher-forced {err_tf:.3g}, "
          f"ratio {err_step / err_tf:.3f}")
    assert err_step <= 2.0 * err_tf, f"decode steps {err_step:.3g} vs teacher-forced {err_tf:.3g}"
