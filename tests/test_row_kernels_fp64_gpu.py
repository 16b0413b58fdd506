"""GPU: the row kernels of csrc/elementwise.cu (layernorm kinds 0 / 1, bert_embed_ln, masked_mean_pool), bert_embed_sum, the
fp16 overflow clamp with a device row count and the live-tile tables, against the float64 references of
oracle/rowops_oracle.py.  The layernorm check is an interval of allowed 16-bit outputs (one or two values where the fp32
error is below half an ulp), not a tolerance.  Strided views are surrounded by NaN sentinel columns that must survive.
Every case prints `RATIO <what>: <worst>` (distance from the interval's centre over its half width, <= 1 passes) and, for
the layernorm, the fraction of outputs whose interval is a single value and how many outputs took the second value of a
two-value interval."""
import math

import pytest
import torch

import rowops_oracle as ro

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTYPES = [F16, BF16]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _nan_view(rows, H, dtype, dev, pad=8):
    """[rows, H] view at column `pad` (16-byte aligned) of a NaN-filled [rows, H + 2 pad] buffer, and the buffer."""
    buf = torch.full((rows, H + 2 * pad), float("nan"), dtype=dtype, device=dev)
    return buf[:, pad:pad + H], buf


def _sentinels_intact(buf, H, pad=8):
    return bool(torch.isnan(buf[:, :pad].float()).all()) and bool(torch.isnan(buf[:, pad + H:].float()).all())


def _check_norm(y, x, w, b, eps, kind, dtype, what):
    lo, hi, single = ro.layernorm_interval(x, w, b, eps, kind, dtype)
    ok, ratio = ro.interval_check(y, lo, hi)
    nearest = ro.layernorm_ref_value(x, w, b, eps, kind, dtype)
    second = int(((y.double() != nearest) & ok & ~single).sum())
    worst = float(ratio[ok].max()) if bool(ok.any()) else math.inf
    print(f"RATIO {what}: {worst:.4f} single={float(single.double().mean()):.4f} second={second}")
    assert bool(ok.all()), (what, int((~ok).sum()), torch.nonzero(~ok)[:4].tolist())
    return single


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("H", [8, 64, 248, 512, 520, 768, 776, 1024, 2048])
def test_layernorm_fp64(dev, dtype, kind, H):
    """1 to 8 vectors per lane and ragged lanes; normal, constant, zero, 40-sigma offset, outlier, tiny and eps-sized rows;
    zero and negative weights; both eps; strided x and y between NaN sentinels."""
    from atlas_b200 import ops

    rows = 301
    x = ro.norm_rows(rows, H, dtype, seed=H * 2 + kind, device=dev)
    w, b = (t.to(dev) for t in ro.norm_weights(H, dtype, seed=H))
    for eps in (1e-12, 1e-6):
        xv, _ = _nan_view(rows, H, dtype, dev)
        xv.copy_(x)
        yv, ybuf = _nan_view(rows, H, dtype, dev)
        ops.layernorm(xv, w, b if kind == 0 else None, eps=eps, kind=kind, out=yv)
        _check_norm(yv, x, w, b, eps, kind, dtype, f"layernorm k{kind} {dtype} H{H} eps{eps:g}")
        assert _sentinels_intact(ybuf, H)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", [1, 7, 9, 4301, 30720, 122880])
def test_layernorm_row_counts(dev, dtype, rows):
    """Row counts up to the T5-base encoder (320 passages x 384 tokens) at H = 768, contiguous."""
    from atlas_b200 import ops

    H = 768
    x = ro.norm_rows(rows, H, dtype, seed=rows, device=dev)
    w, b = (t.to(dev) for t in ro.norm_weights(H, dtype, seed=7))
    for kind, eps in ((0, 1e-12), (1, 1e-6)):
        y = ops.layernorm(x, w, b if kind == 0 else None, eps=eps, kind=kind)
        _check_norm(y, x, w, b, eps, kind, dtype, f"layernorm k{kind} {dtype} rows{rows}")


def test_layernorm_bf16_square_sum_overflow(dev):
    """A bf16 row whose sum of squares overflows fp32: the reference's fp32 arithmetic gives rstd = 0, so y = b (kind 0), 0
    (kind 1).  The other rows of the launch are unaffected."""
    from atlas_b200 import ops

    H = 768
    x = ro.norm_rows(8, H, BF16, seed=3, device=dev)
    x[5] = torch.linspace(1e20, 3e20, H, device=dev).to(BF16)
    w, b = (t.to(dev) for t in ro.norm_weights(H, BF16, seed=4))
    y0 = ops.layernorm(x, w, b, eps=1e-12, kind=0)
    y1 = ops.layernorm(x, w, None, eps=1e-6, kind=1)
    assert torch.equal(y0[5], b) and bool((y1[5] == 0).all())
    _check_norm(y0, x, w, b, 1e-12, 0, BF16, "layernorm overflow k0")
    _check_norm(y1, x, w, b, 1e-6, 1, BF16, "layernorm overflow k1")


def _launches():
    from atlas_b200._lib import lib

    return int(lib().atlas_b200_launch_count())


def test_row_kernels_refuse_bad_shapes_and_misaligned_pointers(dev):
    """EINVAL before any launch: H = 2056 (> 2048), H % 8 != 0, and every pointer the 16-byte (4-byte for bert_embed_sum)
    vector accesses would read or write misaligned."""
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    w = torch.ones(2056, dtype=BF16, device=dev)
    b = torch.zeros(2056, dtype=BF16, device=dev)
    buf = torch.zeros(16, 2064, dtype=BF16, device=dev)
    cases = [
        lambda: ops.layernorm(buf[:, :2056], w, b, kind=0),                            # H too large
        lambda: ops.layernorm(buf[:, :12], w[:12], b[:12], kind=0),                     # H % 8
        lambda: ops.layernorm(buf[:, 4:4 + 768], w, b, kind=0),                         # x 8-byte aligned
        lambda: ops.layernorm(buf[:, 8:8 + 768], w[1:], b, kind=0),                     # weight
        lambda: ops.layernorm(buf[:, 8:8 + 768], w, b[4:], kind=0),                     # bias
        lambda: ops.layernorm(buf[:, :768], w, None, kind=1, out=buf[:, 2:2 + 768]),    # y
    ]
    ids = torch.zeros(2, 5, dtype=torch.int64, device=dev)
    table = torch.zeros(64 * 770, dtype=BF16, device=dev)
    t = table[1:1 + 10 * 768].view(10, 768)                                           # 2-byte aligned table
    t4 = table[2:2 + 10 * 768].view(10, 768)                                          # 4-byte aligned
    good = table[:10 * 768].view(10, 768)
    cases += [
        lambda: ops.bert_embed_ln(ids, None, t4, good, good, w[:768], b[:768], 1e-12),
        lambda: ops.bert_embed_ln(ids, None, good, t4, good, w[:768], b[:768], 1e-12),
        lambda: ops.bert_embed_ln(ids, None, good, good, t4, w[:768], b[:768], 1e-12),
        lambda: ops.bert_embed_ln(ids, None, good, good, good, w[1:769], b[:768], 1e-12),
        lambda: ops.bert_embed_sum(ids, None, t, good, good),
        lambda: ops.bert_embed_sum(ids, None, good, good, t),
    ]
    S, nb = 2, 1
    live = torch.ones(S, nb, dtype=torch.uint8, device=dev)
    keep, off, src, count = ops.segment_tile_scan(live)
    big = torch.zeros(S * 64 + 1, 768, dtype=BF16, device=dev)
    before = _launches()
    cases += [
        lambda: ops.embed_packed_tiles(torch.zeros(S * 64, dtype=torch.int64, device=dev), t4, src),
        lambda: ops.expand_packed_tiles(big.view(-1)[4:4 + S * 64 * 768].view(S * 64, 768), off),
        lambda: ops.compact_live_tiles(big.view(-1)[4:4 + S * 64 * 768].view(S * 64, 768), live.view(-1)),
        lambda: ops.clamp_inf_(torch.zeros(64 * 769, dtype=F16, device=dev)[4:4 + 64 * 768].view(64, 768)),
    ]
    for i, c in enumerate(cases):
        with pytest.raises(AtlasB200Error):
            c()
        assert _launches() == before, f"case {i} launched a kernel"
    torch.cuda.synchronize()


def _embed_tables(V, H, dtype, seed, dev):
    g = torch.Generator().manual_seed(seed)
    word = (torch.randn(V, H, generator=g) * 0.5).to(dtype).to(dev)
    type_ = (torch.randn(2, H, generator=g) * 0.5).to(dtype).to(dev)
    pos = (torch.randn(512, H, generator=g) * 0.5).to(dtype).to(dev)
    return word, type_, pos, g


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [1, 37, 512])
@pytest.mark.parametrize("with_tt", [False, True])
def test_bert_embed_fp64(dev, dtype, L, with_tt):
    """bert_embed_sum bit-exact against r16(r16(word + type) + pos); bert_embed_ln inside the layernorm interval of that sum
    and bit-identical to layernorm(bert_embed_sum(ids)) (the training and inference paths agree).  Ids 0 and V - 1."""
    from atlas_b200 import ops

    V, H, B = 1000, 768, 3
    word, type_, pos, g = _embed_tables(V, H, dtype, L * 2 + with_tt, dev)
    w, b = (t.to(dev) for t in ro.norm_weights(H, dtype, seed=L))
    ids = torch.randint(0, V, (B, L), generator=g)
    ids[0, 0] = 0
    ids[-1, -1] = V - 1
    tts = torch.randint(0, 2, (B, L), generator=g) if with_tt else None
    ids_d, tts_d = ids.to(dev), (tts.to(dev) if with_tt else None)
    s = ops.bert_embed_sum(ids_d, tts_d, word, type_, pos)
    want = ro.embed_sum64(ids, tts, word.cpu(), type_.cpu(), pos.cpu(), L, dtype)
    assert torch.equal(s.reshape(-1, H).cpu().double(), want)
    y = ops.bert_embed_ln(ids_d, tts_d, word, type_, pos, w, b, 1e-12)
    _check_norm(y.reshape(-1, H), want.to(dev), w, b, 1e-12, 0, dtype, f"bert_embed_ln {dtype} L{L} tt{int(with_tt)}")
    assert torch.equal(y, ops.layernorm(s, w, b, eps=1e-12, kind=0))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H", [8, 100, 768])
@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.int64])
def test_masked_mean_pool_fp64(dev, dtype, H, mask_dtype):
    """Inside the interval of r16(f32(r16(fp32 sum)) / f32(count)); an empty-mask row gives NaN; fp16 sums that overflow give
    +-inf; written into strided bank rows whose neighbours keep their NaN sentinels."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(H)
    B, L = 7, 512
    x = (torch.randn(B, L, H, generator=g) * 3).to(dtype)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[1] = L
    mask = torch.arange(L)[None] < lens[:, None]
    mask[2, 10:200] = False                                            # a hole
    mask[0] = False                                                    # empty
    if dtype == F16:
        x[1, :, : min(H, 4)] = 3000.0                                  # 512 x 3000 overflows the fp16 sum
        x[1, :, 4:6] = -200.0                                          # 102400: the sum overflows, the mean (-200) would not
    bank, buf = _nan_view(2 * B + 3, H, dtype, dev)
    out = bank[3:3 + 2 * B:2]                                          # every other bank row
    ops.masked_mean_pool(x.to(dev), mask.to(mask_dtype).to(dev), out=out)
    lo, hi = ro.pool_interval(x, mask, dtype)
    ok, ratio = ro.interval_check(out.cpu(), lo, hi)
    print(f"RATIO masked_mean_pool {dtype} H{H} {mask_dtype}: {float(ratio[ok].max()):.4f}")
    assert bool(ok.all()), torch.nonzero(~ok)[:4].tolist()
    assert bool(torch.isnan(out[0].float()).all())
    if dtype == F16:
        assert bool(torch.isinf(out[1, : min(H, 6)].float()).all())
    others = torch.ones(2 * B + 3, dtype=torch.bool)
    others[3:3 + 2 * B:2] = False
    assert bool(torch.isnan(bank[others.to(dev)].float()).all()) and _sentinels_intact(buf, H)


# ---------------------------------------------------------------------------------------------------------------------
# fp16 overflow clamp with a device row count
def _clamp_case(dev):
    M, N, count = 1000, 768, 640
    g = torch.Generator().manual_seed(8)
    x = (torch.randn(M, N, generator=g) * 20000).clamp(-65000, 65000).half()
    x[:count, 5] = 65000.0                                             # live rows: values above the clamp bound, no inf
    x[count:, 7] = float("inf")                                        # never-computed rows: inf and 65000 sentinels
    x[count:, 9] = 65000.0
    return x.to(dev), count


def _clamp_want(x, n):
    cv = torch.finfo(torch.float16).max - 1000
    want = x.clone()
    want[:n] = torch.clamp(x[:n].float(), min=-cv, max=cv).half()
    return want


def test_clamp_inf_reads_only_the_counted_rows(dev):
    from atlas_b200 import ops

    x0, count = _clamp_case(dev)
    M = x0.shape[0]
    ss0 = torch.full((M,), -1.0, device=dev)
    cnt = torch.tensor([count], dtype=torch.int32, device=dev)
    x, ss = x0.clone(), ss0.clone()
    ops.clamp_inf_(x, row_ss=ss, rows=cnt)
    assert torch.equal(x, x0) and torch.equal(ss, ss0)                 # no inf in the counted rows: nothing changes
    x0[3, 100] = float("inf")                                          # an inf in a live row
    for n in (count, 0, -5, M + 7):
        x, ss = x0.clone(), ss0.clone()
        cnt.fill_(n)
        ops.clamp_inf_(x, row_ss=ss, rows=cnt)
        k = min(max(n, 0), M)
        if k <= 3:                                                     # the inf row is not counted: untouched
            assert torch.equal(x, x0) and torch.equal(ss, ss0), n
            continue
        want = _clamp_want(x0, k)
        assert torch.equal(x, want), n
        ref_ss = want[:k].double().pow(2).sum(-1)
        fin = torch.isfinite(ref_ss)
        rel = ((ss[:k].double() - ref_ss).abs() / ref_ss.clamp_min(1e-30))[fin]
        print(f"RATIO clamp row_ss n{n}: {float(rel.max()) / (768 * 2 ** -24):.4f}")
        assert float(rel.max()) <= 768 * 2 ** -24
        assert torch.equal(ss[k:], ss0[k:])


def test_clamp_inf_row_count_follows_graph_replays(dev):
    from atlas_b200 import ops

    x0, count = _clamp_case(dev)
    x0[3, 100] = float("inf")
    x0[700, 1] = float("-inf")                                         # inside only when the count grows past 700
    x = x0.clone()
    cnt = torch.tensor([count], dtype=torch.int32, device=dev)
    ss = torch.zeros(x.shape[0], device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.clamp_inf_(x, row_ss=ss, rows=cnt)                         # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.clamp_inf_(x, row_ss=ss, rows=cnt)
    for n in (count, 2, 1000, 701):
        x.copy_(x0)
        cnt.fill_(n)
        graph.replay()
        torch.cuda.synchronize()
        want = _clamp_want(x0, n) if n > 3 else x0
        assert torch.equal(x, want), n


def test_fp16_packed_encoder_never_sees_junk_rows(dev):
    """The padding-compacted fp16 encoder computes only its first *count rows; the rest of each buffer is allocator memory.
    With the caching allocator's free blocks filled with inf beforehand, no clamp may fire at any sub-layer: the inputs
    are small, so only a junk row could hold an inf."""
    import model_synth
    from atlas_b200 import ops
    from atlas_b200.fid import FiD, T5ConfigLite

    cfg = {k: v for k, v in dict(model_synth.T5_CFG, num_layers=2, num_decoder_layers=1).items()
           if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    model = FiD(T5ConfigLite(**cfg))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 404)
    model.load_state_dict(sd)
    model = model.half().to(dev).eval()
    B, n_ctx, L = 2, 4, 384
    ids, mask, _ = model_synth.fid_inputs(seed=6, B=B, n_ctx=n_ctx, L=L, T=4, vocab=cfg["vocab_size"])
    mask = mask.view(B, n_ctx, L).clone()
    mask[:, :, 40:] = False                                            # one 64-row tile per passage: 5/6 of every buffer is junk
    ids = (ids.view(B, n_ctx, L) * mask).view(B, -1)
    mask = mask.view(B, -1)
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    d = cfg["d_model"]
    fired = []
    real = ops.clamp_inf_

    def spy(x, row_ss=None, rows=None):
        out = real(x, row_ss=row_ss, rows=rows)
        fired.append(int(ops._inf_flags[x.device].item()))
        return out

    saved = ops._ENC_PACKED
    ops._ENC_PACKED = True
    ops.clamp_inf_ = spy
    try:
        for fuse in (True, False):
            model.fuse_norm = fuse
            sizes = [B * n_ctx * L * n for n in (d, 3 * d, 2 * cfg["d_ff"], cfg["d_ff"])]
            junk = [torch.full((n,), float("inf"), dtype=torch.float16, device=dev) for n in sizes for _ in range(3)]
            del junk                                                   # the allocator keeps the inf-filled blocks cached
            with torch.no_grad():
                r = model._encode_rows(ids.to(dev), mask.to(dev), packed=True)
            assert isinstance(r, tuple)
            n = int(r[3])
            assert bool(torch.isfinite(r[0][:n]).all())
    finally:
        ops.clamp_inf_ = real
        ops._ENC_PACKED = saved
    assert len(fired) > 0 and sum(fired) == 0, fired


# ---------------------------------------------------------------------------------------------------------------------
# live-tile tables
@pytest.mark.parametrize("n_tiles", [1, 1023, 1024, 1025, 1920, 5000])
@pytest.mark.parametrize("pattern", ["random", "dead", "live"])
def test_compact_live_tiles_tables(dev, n_tiles, pattern):
    """tile_off = exclusive cumsum of the live flags (-1 for dead tiles), count = 64 x live: the scan's carry across its
    1024-tile passes; the copied rows are the live tiles' rows."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(n_tiles)
    flags = {"random": torch.rand(n_tiles, generator=g) < 0.4, "dead": torch.zeros(n_tiles, dtype=torch.bool),
             "live": torch.ones(n_tiles, dtype=torch.bool)}[pattern]
    d = 8
    x = torch.arange(n_tiles * 64 * d, dtype=torch.float32).remainder(2039).to(BF16).view(n_tiles * 64, d).to(dev)
    x_live, off, count = ops.compact_live_tiles(x, flags.to(torch.uint8).to(dev))
    want = torch.where(flags, torch.cumsum(flags.int(), 0) - 1, torch.full((n_tiles,), -1, dtype=torch.int64))
    assert torch.equal(off.cpu(), want.int()) and int(count) == 64 * int(flags.sum())
    n = int(count)
    assert torch.equal(x_live[:n], x.view(-1, 64, d)[flags.to(dev)].reshape(n, d))
