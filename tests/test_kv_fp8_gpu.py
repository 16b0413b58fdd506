"""The opt-in FP8 (e4m3) cross K|V cache of KV-cached generation (csrc/kv_fp8.cu, the e4m3 kernels of csrc/decode.cu and
csrc/attention_stream.cu, FiD.generate(cross_kv_dtype="fp8")).

  - the quantizer's codes and scales are bit-identical to the CPU oracle (oracle/kv_fp8_oracle.py);
  - both attention kernels against a float64 reference built from the DEQUANTIZED K / V, held to the bound of
    tests/test_decode_kernels_gpu.py (one ulp of the output type + 1e-5 max|V|) plus, for the stream kernel, the 16-bit
    rounding of p * vscale before the P.V MMA;
  - CUDA-graph replay equals eager launches bit for bit;
  - the fp8 decode-step logits against a CPU decoder over the same dequantized cross K / V (isolating the kernels from the
    quantization loss), within 2x the 16-bit path's teacher-forced error against the fp32 oracle; token agreement with the
    16-bit path and the logit change quantization causes are printed, not asserted;
  - the state's cross K|V bytes, and one Atlas.generate with 4 beams."""
import pytest
import torch

import fid_cpu
import kv_fp8_oracle as ko
import model_synth

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
NEG = {torch.float16: -1e4, torch.bfloat16: -1e9}
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}       # unit roundoff of the 16-bit types
EOS = 1
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _ulp(ref, dtype):
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    return torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin))) - mant)


def _ratio(got, ref, bound):
    return float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())


def _report(name, r):
    WORST[name] = max(WORST.get(name, 0.0), r)
    print(f"worst error / bound so far, {name}: {WORST[name]:.3g}")


# ------------------------------------------------------------------------------------------------------------------------
# 1. quantizer
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,H", [(1, 12), (8 * 15360, 12), (2 * 15360 + 7, 32), (333, 32)])
def test_quantizer_bit_identical_to_oracle(dev, dtype, rows, H):
    """Codes and scales equal the oracle's bits, from a strided input view (extra NaN columns that must not leak in) into
    strided outputs; per-row magnitudes from 1e-3 to 1e3, zero blocks and non-finite blocks included."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(rows + H)
    C = 2 * H
    x = torch.randn(rows, C * 64, generator=g) * torch.exp(torch.empty(rows, 1).uniform_(-7, 7, generator=g))
    x[0, :64] = 0.0
    if rows > 3:
        x[1, 64 + 3] = float("nan")
        x[2, 5 * 64] = float("inf")
        x[3, 64:128] = 2.0 ** -10 * torch.randint(-8, 9, (64,), generator=g)       # subnormal codes
    x = x.to(dtype)
    xbuf = torch.full((rows, C * 64 + 72), float("nan"), dtype=dtype, device=dev)
    xbuf[:, 8:8 + C * 64] = x.to(dev)
    obuf = torch.full((rows, C * 64 + 16), 0xA5, dtype=torch.uint8, device=dev)
    sbuf = torch.full((rows, C + 3), -7.0, dtype=torch.float32, device=dev)
    codes, scales = ops.quantize_kv_e4m3(xbuf[:, 8:8 + C * 64], out=obuf[:, :C * 64], scale_out=sbuf[:, :C])
    want_c, want_s = ko.quantize_e4m3(x)
    assert torch.equal(codes.cpu(), want_c)
    assert torch.equal(scales.cpu().view(torch.int32), want_s.view(torch.int32))
    assert bool((obuf[:, C * 64:] == 0xA5).all()) and bool((sbuf[:, C:] == -7.0).all())


def test_quantizer_rejects_bad_layouts(dev):
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    x = torch.zeros((4, 128), dtype=torch.bfloat16, device=dev)
    with pytest.raises(AtlasB200Error):
        ops.quantize_kv_e4m3(x.float())
    with pytest.raises(AtlasB200Error):
        ops.quantize_kv_e4m3(x[:, :100])
    with pytest.raises(AtlasB200Error):
        ops.quantize_kv_e4m3(x.t())
    with pytest.raises(AtlasB200Error):
        ops.quantize_kv_e4m3(x, out=torch.zeros((4, 128), dtype=torch.int8, device=dev))


# ------------------------------------------------------------------------------------------------------------------------
# 2. attention kernels over the e4m3 cache
# ------------------------------------------------------------------------------------------------------------------------
Q_MULT = {"soft": 2.5, "hard": 3.0, "tiles": 1.0, "last": 1.0, "full": 0.25}


def _cross_mask_row(kind, Lk, neg, g):
    j = torch.arange(Lk)
    if kind == "soft":
        return -4.0 * torch.rand(Lk, generator=g, dtype=torch.float64).float()
    if kind == "hard":
        return torch.where(torch.rand(Lk, generator=g) < 0.5, neg, 0.0)
    if kind == "tiles":
        region = ((j // 1024) % 2 == 0) & ((j // 256) % 2 == 0) & ((j // 64) % 3 != 1)
        live = region & (torch.rand(Lk, generator=g) < 0.5)
        live[int(region.nonzero()[-1])] = True
        return torch.where(live, 0.0, neg)
    if kind == "last":
        m = torch.full((Lk,), neg)
        m[-1] = 0.0
        return m
    assert kind == "full"
    return torch.full((Lk,), -1e9)


# the case matrix of tests/test_decode_kernels_gpu.py: (Lk, B, H, scale, mask kind of each batch row)
CROSS_CASES = [
    (1, 2, 12, 1.0, ("soft", "full")),
    (17, 5, 1, 1.0, ("soft", "hard", "tiles", "last", "full")),
    (100, 5, 32, 0.125, ("soft", "hard", "tiles", "last", "full")),
    (2047, 2, 12, 1.0, ("tiles", "last")),
    (2048, 1, 32, 1.0, ("tiles",)),
    (3072 + 40, 5, 12, 1.0, ("soft", "hard", "tiles", "last", "full")),
    (15360, 2, 12, 1.0, ("hard", "tiles")),
]
CHUNKS = (16, 64, 80, 256, 1024)


def _e4m3_inputs(B, Lk, H, kinds, scale, dtype, dev, g):
    """Quantized K|V in strided views (codes at column 16 of wider rows, scales at column 2), their fp64 dequantization, q,
    and the per-row masks.  V rows of very different magnitude so the per-key vscale matters."""
    from atlas_b200 import ops

    HD = H * 64
    mult = torch.tensor([Q_MULT[k] for k in kinds]) / scale
    kv16 = torch.randn(B * Lk, 2 * HD, generator=g) * torch.exp(torch.empty(B * Lk, 1).uniform_(-1.5, 1.5, generator=g))
    kv16 = kv16.to(dtype)
    # q halved: K rows here are up to e^1.5 larger than the 16-bit test's
    q16 = (torch.randn(B, HD, generator=g) * mult[:, None] * 0.5).to(dtype)
    codes, sc = ko.quantize_e4m3(kv16)
    cbuf = torch.full((B * Lk, 2 * HD + 32), 0x7F, dtype=torch.uint8, device=dev)      # 0x7F = e4m3 NaN around the view
    cbuf[:, 16:16 + 2 * HD] = codes.to(dev)
    sbuf = torch.full((B * Lk, 2 * H + 5), float("nan"), dtype=torch.float32, device=dev)
    sbuf[:, 2:2 + 2 * H] = sc.to(dev)
    deq = ko.dequantize_e4m3(codes, sc)
    K = deq[:, :HD].view(B, Lk, H, 64).to(dev)
    V = deq[:, HD:].view(B, Lk, H, 64).to(dev)
    vsc = sc[:, H:].double().view(B, Lk, H).to(dev)
    v8 = codes[:, HD:].contiguous().view(torch.float8_e4m3fn).double().view(B, Lk, H, 64).to(dev)
    mask = torch.stack([_cross_mask_row(k, Lk, NEG[dtype], g) for k in kinds]).to(dev)
    assert torch.equal(ops.quantize_kv_e4m3(kv16.to(dev))[0].cpu(), codes)
    return q16, cbuf[:, 16:16 + 2 * HD], sbuf[:, 2:2 + 2 * H], K, V, vsc, v8, mask


def _softmax_ref(s, m, kinds, V):
    logits = s if m is None else s + m.double()[:, None, :]
    p = torch.softmax(logits, -1)                                           # [B, H, Lk]
    if m is not None:
        for b, kind in enumerate(kinds):
            if kind == "full":      # -1e9 swallows every fp32 logit: uniform, as in the 16-bit test
                p[b] = 1.0 / p.shape[-1]
    return p


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Lk,B,H,scale,kinds", CROSS_CASES, ids=[f"Lk{c[0]}-B{c[1]}-H{c[2]}" for c in CROSS_CASES])
def test_decode_cross_attention_e4m3_matches_fp64(dev, dtype, Lk, B, H, scale, kinds):
    """The greedy decode kernel over the codes: every chunk size, with and without the live-tile skip (bit-identical), from
    strided q / codes / scales / out views."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(2000 + Lk + 7 * B + H)
    HD = H * 64
    q16, kv8, ksc, K, V, _, _, mask = _e4m3_inputs(B, Lk, H, kinds, scale, dtype, dev, g)
    qbuf = torch.full((B, HD + 72), float("nan"), dtype=dtype, device=dev)
    qbuf[:, 8:8 + HD] = q16.to(dev)
    q = qbuf[:, 8:8 + HD]
    outbuf = torch.full((B, HD + 64), float("nan"), dtype=dtype, device=dev)
    out = outbuf[:, 32:32 + HD]
    s = torch.einsum("bhd,bjhd->bhj", q16.double().view(B, H, 64).to(dev), K) * scale
    v_absmax = float(V.abs().max())
    for m in (None, mask):
        ref = torch.einsum("bhj,bjhd->bhd", _softmax_ref(s, m, kinds, V), V).reshape(B, HD)
        bound = _ulp(ref, dtype) + 1e-5 * v_absmax
        live = ops.key_block_live(m)
        for chunk in CHUNKS:
            got = {}
            for tl in (None, live) if m is not None else (None,):
                res = ops.decode_cross_attention_e4m3(q, kv8, ksc, B, H, Lk, add_mask=m, scale=scale, chunk=chunk, out=out,
                                                      tile_live=tl)
                assert res.data_ptr() == out.data_ptr()
                got[tl is None] = out.clone()
                r = _ratio(got[tl is None], ref, bound)
                _report("decode_cross_attention_e4m3", r)
                assert r <= 1.0, f"mask={m is not None} chunk={chunk} tile_live={tl is not None}: {r:.3g}"
            if len(got) == 2:
                assert torch.equal(got[True].view(torch.int16), got[False].view(torch.int16)), chunk
    assert bool(outbuf[:, :32].isnan().all()) and bool(outbuf[:, 32 + HD:].isnan().all())


BEAM_CASES = [
    (1, 2, 12, 1, ("soft", "full")),
    (100, 3, 32, 4, ("soft", "hard", "last")),
    (2047, 2, 12, 16, ("tiles", "last")),
    (3072 + 40, 5, 12, 4, ("soft", "hard", "tiles", "last", "full")),
    (15360, 2, 12, 8, ("hard", "tiles")),
    (15360, 1, 12, 16, ("tiles",)),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Lk,B,H,nb,kinds", BEAM_CASES, ids=[f"Lk{c[0]}-B{c[1]}-H{c[2]}-nb{c[3]}" for c in BEAM_CASES])
def test_stream_cross_attention_e4m3_matches_fp64(dev, dtype, Lk, B, H, nb, kinds):
    """The stream kernel over the codes (nb beams of a batch element against its one cache), chunks of 64 / 256 / 1024
    keys, with and without the live-tile skip (bit-identical).  Bound: the decode bound plus sum_j u16 * p_j * vscale_j *
    |v8_j| for the rounding of p * vscale to 16 bits (fp16: plus its subnormal floor at the kernel's 256x boost)."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(3000 + Lk + 7 * B + H + nb)
    HD = H * 64
    q1, kv8, ksc, K, V, vsc, v8, mask = _e4m3_inputs(B, Lk, H, kinds, 1.0, dtype, dev, g)
    q16 = (q1.repeat_interleave(nb, 0).float() * torch.linspace(0.5, 1.5, nb).repeat(B)[:, None]).to(dtype)
    q = q16.to(dev)
    s = torch.einsum("bnhd,bjhd->bnhj", q16.double().view(B, nb, H, 64).to(dev), K)
    v_absmax = float(V.abs().max())
    floor = 2.0 ** -25 / 256 if dtype == torch.float16 else 0.0
    for m in (None, mask):
        p = _softmax_ref(s.reshape(B, nb * H, Lk), m, kinds, V).view(B, nb, H, Lk)
        ref = torch.einsum("bnhj,bjhd->bnhd", p, V).reshape(B * nb, HD)
        pv = (U16[dtype] * p * vsc.permute(0, 2, 1)[:, None] + floor)                     # [B, nb, H, Lk]
        round_pv = torch.einsum("bnhj,bjhd->bnhd", pv, v8.abs()).reshape(B * nb, HD)
        bound = _ulp(ref, dtype) + 1e-5 * v_absmax + round_pv
        live = ops.key_block_live(m)
        for chunk in (64, 256, 1024):
            got = {}
            for tl in (None, live) if m is not None else (None,):
                out = ops.decode_cross_attention_beams_e4m3(q, kv8, ksc, B, nb, H, Lk, m, chunk, tile_live=tl)
                got[tl is None] = out
                r = _ratio(out, ref, bound)
                _report("cross_attention_stream_e4m3", r)
                assert r <= 1.0, f"mask={m is not None} chunk={chunk} tile_live={tl is not None}: {r:.3g}"
            if len(got) == 2:
                assert torch.equal(got[True].view(torch.int16), got[False].view(torch.int16)), chunk


def test_e4m3_kernels_reject_bad_layouts(dev):
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    B, H, Lk = 2, 2, 64
    q = torch.zeros((B, H * 64), dtype=torch.bfloat16, device=dev)
    kv8 = torch.zeros((B * Lk, 2 * H * 64), dtype=torch.uint8, device=dev)
    sc = torch.zeros((B * Lk, 2 * H), dtype=torch.float32, device=dev)
    for args in ((q.float(), kv8, sc), (q, kv8.view(torch.int8), sc), (q, kv8, sc.half()), (q, kv8[:, :-64], sc),
                 (q, kv8, sc[:, :-1]), (q[:1], kv8, sc)):
        with pytest.raises(AtlasB200Error):
            ops.decode_cross_attention_e4m3(*args, B, H, Lk)
    with pytest.raises(AtlasB200Error):
        ops.decode_cross_attention_e4m3(q, kv8, sc, B, H, Lk, chunk=24)
    with pytest.raises(AtlasB200Error):
        ops.decode_cross_attention_beams_e4m3(q, kv8, sc, B, 1, H, Lk, None, 80)


def test_e4m3_entry_points_reject_misaligned_views(dev):
    """Views whose strides pass but whose first element is not 16-byte aligned raise instead of faulting, through the ops
    wrappers and through the C entry points directly (the wrappers' own check bypassed)."""
    import ctypes

    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error, lib

    B, H, Lk = 2, 2, 64
    HD = H * 64
    q = torch.zeros((B, HD + 8), dtype=torch.bfloat16, device=dev)
    kvb = torch.zeros((B * Lk, 2 * HD + 32), dtype=torch.uint8, device=dev)
    kv8, kv8_off = kvb[:, :2 * HD], kvb[:, 8:8 + 2 * HD]          # row stride 288: a multiple of 16 bytes
    sc = torch.zeros((B * Lk, 2 * H), dtype=torch.float32, device=dev)
    x = torch.zeros((4, 2 * 64 + 8), dtype=torch.float16, device=dev)
    with pytest.raises(AtlasB200Error, match="aligned"):
        ops.quantize_kv_e4m3(x[:, 1:1 + 128])
    with pytest.raises(AtlasB200Error, match="aligned"):
        ops.quantize_kv_e4m3(x[:, :128], out=torch.zeros((4, 136), dtype=torch.uint8, device=dev)[:, 4:132])
    with pytest.raises(AtlasB200Error, match="aligned"):
        ops.decode_cross_attention_e4m3(q[:, :HD], kv8_off, sc, B, H, Lk)
    with pytest.raises(AtlasB200Error, match="aligned"):
        ops.decode_cross_attention_beams_e4m3(q[:, :HD], kv8_off, sc, B, 1, H, Lk, None, 64)
    ops.decode_cross_attention_e4m3(q[:, :HD], kv8, sc, B, H, Lk)                 # aligned: runs
    L = lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    part = torch.zeros((B * 4, HD), dtype=torch.float32, device=dev)
    ml = torch.zeros((B * 4, H, 2), dtype=torch.float32, device=dev)
    qm = q[:, 1:1 + HD]                                            # 2-byte offset
    assert L.atlas_b200_quantize_kv_e4m3(p(x).value + 2, x.stride(0), 4, 2, p(kvb), kvb.stride(0), p(sc), sc.stride(0), 0,
                                         None) == 1
    assert b"aligned" in L.atlas_b200_last_error()
    assert L.atlas_b200_decode_cross_attention_e4m3(p(qm), q.stride(0), p(kv8_off), kvb.stride(0), p(sc), sc.stride(0), 0, HD,
                                                    None, None, B, H, Lk, 16, 1.0, p(part), p(ml), 1, None) == 1
    assert b"aligned" in L.atlas_b200_last_error()
    assert L.atlas_b200_cross_attention_stream_e4m3(p(q), q.stride(0), 0, p(kv8_off), kvb.stride(0), p(sc), sc.stride(0), 0,
                                                    HD, None, None, B, H, 1, Lk, 64, 1.0, p(part), p(ml), 1, None) == 1
    assert b"aligned" in L.atlas_b200_last_error()
    dev_other = torch.device("cpu")
    with pytest.raises(AtlasB200Error):
        ops.decode_cross_attention_e4m3(q[:, :HD], kv8, sc, B, H, Lk, add_mask=torch.zeros((B, Lk), device=dev_other))


@pytest.mark.parametrize("dtype", DTYPES)
def test_e4m3_kernels_graph_replay_is_bit_identical(dev, dtype):
    """One captured graph holding the quantizer and both attention kernels, replayed on new inputs, equals eager calls."""
    from atlas_b200 import ops

    B, H, Lk, nb = 2, 12, 3072, 4
    g = torch.Generator().manual_seed(9)
    kv16 = torch.empty((B * Lk, 2 * H * 64), dtype=dtype, device=dev)
    q = torch.empty((B, H * 64), dtype=dtype, device=dev)
    qb = torch.empty((B * nb, H * 64), dtype=dtype, device=dev)
    mask = torch.where(torch.rand(B, Lk, generator=g) < 0.3, NEG[dtype], 0.0).to(dev)
    live = ops.key_block_live(mask)
    kv8 = torch.empty((B * Lk, 2 * H * 64), dtype=torch.uint8, device=dev)
    sc = torch.empty((B * Lk, 2 * H), dtype=torch.float32, device=dev)

    def step():
        ops.quantize_kv_e4m3(kv16, out=kv8, scale_out=sc)
        a = ops.decode_cross_attention_e4m3(q, kv8, sc, B, H, Lk, add_mask=mask, chunk=256, tile_live=live)
        b = ops.decode_cross_attention_beams_e4m3(qb, kv8, sc, B, nb, H, Lk, mask, 256, tile_live=live)
        return a, b

    def fill(seed):
        gg = torch.Generator().manual_seed(seed)
        kv16.copy_(torch.randn(kv16.shape, generator=gg).to(dtype))
        q.copy_((torch.randn(q.shape, generator=gg) * 2).to(dtype))
        qb.copy_((torch.randn(qb.shape, generator=gg) * 2).to(dtype))

    fill(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ga, gb = step()
    for seed in (1, 2, 3):
        fill(seed)
        graph.replay()
        gak, gbk = ga.clone(), gb.clone()
        ea, eb = step()
        assert torch.equal(gak.view(torch.int16), ea.view(torch.int16)), seed
        assert torch.equal(gbk.view(torch.int16), eb.view(torch.int16)), seed


# ------------------------------------------------------------------------------------------------------------------------
# 3. end to end: FiD.generate(cross_kv_dtype="fp8")
# ------------------------------------------------------------------------------------------------------------------------
def _passages(B, n_ctx, L, lens, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, vocab, (B, n_ctx, L), generator=g)
    lens = torch.tensor(lens).view(B, n_ctx)
    m = torch.arange(L)[None, None, :] < lens[..., None]
    ids = ids * m
    ids.scatter_(2, (lens - 1)[..., None], EOS)
    return ids.view(B, n_ctx * L), m.view(B, n_ctx * L)


def _model(dtype, dev, over=None):
    from atlas_b200.fid import FiD, T5ConfigLite

    cfg = dict(model_synth.T5_CFG, **(over or {}))
    model = FiD(T5ConfigLite(**{k: v for k, v in cfg.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    return model.to(dtype).to(dev).eval(), sd, cfg


# (model size, n_ctx, L, passage lengths, B, beams): tiny synthetic FiD, and FiD-base dimensions (12 decoder layers, d 768,
# 12 heads, the full vocabulary; 2 encoder layers - the encoder runs once and is not under test) over 2 x 1024 / 3072 keys
E2E_CASES = [
    ("tiny", 3, 128, [5, 128, 1, 40, 2, 1], 2, 1),
    ("tiny", 8, 384, [12, 1, 60, 7, 33, 2, 64, 20, 1, 3, 45, 9, 30, 18, 5, 61], 2, 4),
    ("base", 4, 256, [256, 100, 17, 230, 3, 256, 64, 128], 2, 1),
    ("base", 4, 256, [256, 100, 17, 230, 3, 256, 64, 128], 2, 4),
]
BASE = dict(vocab_size=32128, d_model=768, d_kv=64, d_ff=2048, num_heads=12, num_layers=2, num_decoder_layers=12)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("size,n_ctx,L,lens,B,nb", E2E_CASES, ids=[f"{c[0]}-Lk{c[1] * c[2]}-nb{c[5]}" for c in E2E_CASES])
def test_generate_fp8_step_logits_match_dequantized_cpu_decoder(dev, dtype, size, n_ctx, L, lens, B, nb):
    """Every step's logits of the fp8 run (eager, recorded) against the CPU decoder over the dequantized cache the run
    built, within 2x the 16-bit path's teacher-forced error against the fp32 oracle.  Reported: token agreement of the
    CUDA-graph fp8 run with the eager one (the fused RMSNorm's fp32 atomics can move a bf16 logit by an ulp between runs, so
    near-ties may flip, as on the 16-bit path; graph replay itself is checked bit for bit at the kernel level above) and
    with the 16-bit run, and the logit change quantization causes."""
    model, sd, cfg = _model(dtype, dev, BASE if size == "base" else None)
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    ids, mask = _passages(B, n_ctx, L, lens, cfg["vocab_size"], seed=n_ctx + L)
    ids, mask = ids.to(dev), mask.to(dev)
    kw = dict(max_length=10, min_length=4, num_beams=nb)
    steps = []
    decode_step = model._decode_step_logits

    def recording(st):
        logits = decode_step(st)
        steps.append(logits.clone())
        return logits

    encoded = []
    encode = model.encode

    def recording_encode(*a):
        e = encode(*a)
        encoded.append(e.clone())
        return e

    model.cuda_graphs = False
    model._decode_step_logits = recording
    model.encode = recording_encode
    with torch.no_grad():
        seq8 = model.generate(input_ids=ids, attention_mask=mask, cross_kv_dtype="fp8", **kw)
    model._decode_step_logits = decode_step
    model.encode = encode
    Lk = n_ctx * L
    key = (B, Lk, 10, dtype, dev) + (() if nb == 1 else (nb,)) + ("fp8",)
    st = model.__dict__["_decode_states"][key]
    H = cfg["num_heads"]
    HD = H * 64
    # the cache holds each layer's own projection of the encoder output this generation used: dequantized, within half an
    # e4m3 step (relative 2^-4, absolute 2^-10 * scale on subnormal codes) plus the 16-bit rounding of the projection (2^-8
    # relative, with slack) of the fp32 product of the same 16-bit encoder output and weights (+ its fp32 accumulation order)
    assert len(encoded) == 1
    enc = encoded[0].reshape(B * Lk, -1).float().cpu()
    G = model._weights()[1]
    cross_k, cross_v = [], []
    for i in range(cfg["num_decoder_layers"]):
        sc_i = st.cross_scale[i].cpu()
        deq = ko.dequantize_e4m3(st.cross_kv[i].cpu(), sc_i)
        w = G[f"decoder.block.{i}.layer.1.EncDecAttention.kv"].float().cpu()
        proj = (enc @ w.T).double()
        bound = (2.0 ** -4 + 2.0 ** -7) * proj.abs() + 2.0 ** -9 * sc_i.double().repeat_interleave(64, 1) + \
            2.0 ** -20 * (enc.abs() @ w.abs().T).double() + 1e-6
        r = _ratio(deq, proj, bound)
        _report("cached K|V vs projection", r)
        assert r <= 1.0, f"layer {i}: cached K|V vs the layer's projection, error / bound {r:.3g}"
        deq = deq.view(B, Lk, 2 * HD)
        cross_k.append(deq[..., :HD])
        cross_v.append(deq[..., HD:])
    model.cuda_graphs = True
    with torch.no_grad():
        seq8g = model.generate(input_ids=ids, attention_mask=mask, cross_kv_dtype="fp8", **kw)
        seq16 = model.generate(input_ids=ids, attention_mask=mask, **kw)
    graph_agree = float((seq8g == seq8).float().mean()) if seq8g.shape == seq8.shape else float("nan")

    sd32 = {k: v.float() for k, v in sd.items()}
    n = min(len(steps), seq8.shape[1] - 1)
    # the rows each step decoded: greedy = the sequence itself; beams = the ancestry of every row at every step is not
    # kept, so compare beams on step 0 only (all nb rows of a batch element hold the start token)
    if nb == 1:
        dec_in = seq8[:, :n].cpu()
        got = torch.stack(steps[:n], 1).float().cpu()
    else:
        dec_in = seq8[:, :1].cpu()
        got = steps[0].float().cpu().view(B, nb, -1)[:, :1]
        n = 1
    ref8 = ko.decoder_logits(sd32, cfg, mask.cpu(), dec_in, cross_k, cross_v)
    with torch.no_grad():
        tf = model(input_ids=ids, attention_mask=mask, decoder_input_ids=dec_in.to(dev), use_cache=False)
    _, ref32, _ = fid_cpu.fid_forward(sd32, cfg, ids.cpu(), mask.cpu(), dec_in, n_context=n_ctx)
    err_step = float((got - ref8).abs().max())
    err_tf = float((tf.logits.float().cpu() - ref32).abs().max())
    quant = float((ref8 - ref32).abs().max())
    agree = float((seq8[:, : seq16.shape[1]] == seq16[:, : seq8.shape[1]]).float().mean()) if seq8.shape == seq16.shape \
        else float("nan")
    print(f"{size} nb={nb} {dtype}: fp8 steps vs dequantized CPU decoder {err_step:.3g}, 16-bit teacher-forced vs fp32 "
          f"{err_tf:.3g} (ratio {err_step / err_tf:.3f}); logit change from quantization (CPU, fp32) {quant:.3g}; token "
          f"agreement with the 16-bit run {agree:.3f} ({tuple(seq8.shape)} vs {tuple(seq16.shape)}), fp8 graph vs eager "
          f"{graph_agree:.3f}")
    assert err_step <= 2.0 * err_tf, f"fp8 decode steps {err_step:.3g} vs 16-bit teacher-forced {err_tf:.3g}"


@pytest.mark.parametrize("nb", [1, 4])
def test_fp8_state_bytes_and_options(dev, nb):
    """The fp8 state's cross K|V (codes + scales) is at most 0.54x the 16-bit state's; cross_kv_dtype other than None /
    "fp8" raises; use_cache=False with "fp8" raises."""
    from atlas_b200._lib import AtlasB200Error

    model, _, cfg = _model(torch.bfloat16, dev)
    n_ctx, L, B = 3, 128, 2
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    ids, mask = _passages(B, n_ctx, L, [5, 128, 1, 40, 2, 1], cfg["vocab_size"], seed=1)
    ids, mask = ids.to(dev), mask.to(dev)
    with torch.no_grad():
        model.generate(input_ids=ids, attention_mask=mask, max_length=6, num_beams=nb)
        model.generate(input_ids=ids, attention_mask=mask, max_length=6, num_beams=nb, cross_kv_dtype="fp8")
    states = model.__dict__["_decode_states"]
    base = (B, n_ctx * L, 6, torch.bfloat16, dev) + (() if nb == 1 else (nb,))

    def nbytes(st):
        ts = list(st.cross_kv) + list(st.cross_scale or [])
        return sum(t.numel() * t.element_size() for t in ts)

    b16, b8 = nbytes(states[base]), nbytes(states[base + ("fp8",)])
    print(f"nb={nb}: cross K|V state bytes 16-bit {b16}, fp8 {b8} ({b8 / b16:.4f}x)")
    assert b8 <= 0.54 * b16
    for bad in ("fp16", torch.float8_e4m3fn, "e4m3", 8):
        with pytest.raises(AtlasB200Error):
            model.generate(input_ids=ids, attention_mask=mask, max_length=6, num_beams=nb, cross_kv_dtype=bad)
    with pytest.raises(AtlasB200Error, match="use_cache"):
        model.generate(input_ids=ids, attention_mask=mask, max_length=6, use_cache=False, cross_kv_dtype="fp8")


def test_fp8_prefix_constrained_steps(dev):
    """The eager prefix_allowed_tokens_fn step reads the fp8 cache too: every generated token is an allowed one."""
    model, _, cfg = _model(torch.bfloat16, dev)
    n_ctx, L, B = 3, 128, 2
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    ids, mask = _passages(B, n_ctx, L, [5, 128, 1, 40, 2, 1], cfg["vocab_size"], seed=2)
    allowed = list(range(2, 40)) + [EOS]
    for nb in (1, 3):
        with torch.no_grad():
            out = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), max_length=8, min_length=3, num_beams=nb,
                                 prefix_allowed_tokens_fn=lambda b, s: allowed, cross_kv_dtype="fp8")
        toks = out[:, 1:].cpu()
        assert bool(((toks == model.config.pad_token_id) | torch.isin(toks, torch.tensor(allowed))).all()), nb


def test_atlas_generate_fp8_beams(dev):
    """Atlas.generate reads opt.generation_cross_kv_dtype: one 4-beam run on the fp8 cache completes."""
    import atlas_synth
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    opt = atlas_synth.make_opt()
    opt.generation_num_beams = 4
    opt.generation_cross_kv_dtype = "fp8"
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    reader = FiD(T5ConfigLite(**{k: v for k, v in model_synth.T5_CFG.items()
                                 if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}))
    reader.load_state_dict(model_synth.fill_state_dict(reader.state_dict(), seed=202)[0])
    contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    contriever.load_state_dict(model_synth.fill_state_dict(contriever.state_dict(), seed=101)[0])
    m = Atlas(opt, reader.to(dev).eval(), DualEncoderRetriever(opt, contriever.to(dev)).eval(), reader_tok,
              retriever_tok).eval()
    passages = atlas_synth.make_corpus()
    query, _ = atlas_synth.make_batch()
    ps = [passages[: atlas_synth.TOPK] for _ in query]
    with torch.no_grad():
        reader_tokens, _ = m.tokenize_passages(query, ps)
        out = m.generate(reader_tokens, query)
    assert out.shape[0] == len(query) and 1 < out.shape[1] <= opt.generation_max_length
    states = m.reader.__dict__["_decode_states"]
    assert any(k[-1] == "fp8" and k[-2] == 4 for k in states)
