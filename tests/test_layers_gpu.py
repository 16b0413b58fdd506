"""GPU numerics of the normalisation / embedding / pooling / attention kernels against plain PyTorch
fp32 references of the same ops (rounding points restated from the reference model code)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def test_fp16_inf_clamp(dev):
    """ops.clamp_inf_ = the reference's `if dtype == fp16 and isinf(h).any(): h = clamp(h, +-(65504 - 1000))`
    (src/modeling_t5.py:657-708) decided on the device: untouched without an inf, torch.clamp's values with one."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(3)
    x = (torch.randn(777, 768, generator=g) * 30000).half()            # plenty of values between 64512 and 65504, some inf
    finite = x.clone()
    finite[torch.isinf(finite)] = 65504.0
    assert not torch.isinf(finite).any() and (finite.abs() > 64512).any()
    y = ops.clamp_inf_(finite.clone().to(dev))
    assert torch.equal(y.cpu(), finite)                                 # no inf anywhere: nothing is clamped
    withinf = finite.clone()
    withinf[5, 7] = float("inf")
    withinf[700, 0] = float("-inf")
    withinf[3, 3] = float("nan")
    clamp_value = torch.finfo(torch.float16).max - 1000
    want = torch.clamp(withinf.float(), min=-clamp_value, max=clamp_value).half()
    ss = torch.zeros(777, dtype=torch.float32, device=dev)
    got = ops.clamp_inf_(withinf.clone().to(dev), row_ss=ss)
    assert torch.equal(torch.nan_to_num(got.cpu().float(), nan=-1.0), torch.nan_to_num(want.float(), nan=-1.0))
    ref_ss = want.float().pow(2).sum(-1)
    ok = ~torch.isnan(ref_ss)
    assert torch.allclose(ss.cpu()[ok], ref_ss[ok], rtol=1e-5)
    # other dtypes pass through (the reference tests `dtype == torch.float16`)
    b = torch.full((8, 768), float("inf"), dtype=torch.bfloat16, device=dev)
    assert torch.isinf(ops.clamp_inf_(b)).all()
    # strided view (a column slice of a wider buffer)
    wide = torch.zeros(64, 1536, dtype=torch.float16, device=dev)
    wide[:, 768:] = 65000.0
    wide[1, 800] = float("inf")
    ops.clamp_inf_(wide[:, 768:])
    assert float(wide[:, 768:].max()) == 64512.0 and float(wide[:, :768].abs().max()) == 0.0


def test_fid_fp16_overflow_is_clamped_like_the_reference(dev):
    """A FiD block whose feed-forward output overflows fp16: with the device-side clamp the forward stays finite and equals an
    fp16 torch restatement of the reference's block arithmetic (clamp included) on the same kernels' inputs."""
    import os, sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import model_synth
    from atlas_b200.fid import FiD, T5ConfigLite

    cfg = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    reader = FiD(T5ConfigLite(**cfg))
    sd, _ = model_synth.fill_state_dict(reader.state_dict(), 202)
    sd["encoder.block.0.layer.1.DenseReluDense.wo.weight"] = sd["encoder.block.0.layer.1.DenseReluDense.wo.weight"] * 3000.0
    reader.load_state_dict(sd)
    reader = reader.half().to(dev).eval()
    reader.encoder.config.n_context, reader.encoder.config.bsz = 3, 2
    ids, mask, labels = model_synth.fid_inputs()
    for fuse in (True, False):
        reader.fuse_norm = fuse
        reader.cuda_graphs = False
        with torch.no_grad():
            enc = reader.encode(ids.to(dev), mask.to(dev))
        assert torch.isfinite(enc).all(), f"fuse_norm={fuse}: the overflow reached the encoder output"
        assert float(enc.abs().max()) > 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B,H,T,Lk", [(2, 3, 32, 4000), (1, 12, 7, 15360), (3, 2, 64, 1088), (2, 1, 1, 2048)])
def test_cross_attention_stream_kernel(dev, dtype, B, H, T, Lk):
    """csrc/attention_stream.cu (few target tokens against the concatenated encoder keys, src/fid.py:298-349): skipping the
    fully masked 64-key tiles does not change a bit, with ragged key counts and a long fully masked tail.  The values are
    held against the fp64 oracle in tests/test_attention_fwd_gpu.py (test_stream_kernel, same shapes)."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(B * 1000 + T)
    q = (torch.randn(B * T, H * 64, generator=g) * 0.5).to(dtype).to(dev)
    kv = (torch.randn(B * Lk, 2 * H * 64, generator=g) * 0.5).to(dtype).to(dev)
    valid = torch.rand(B, Lk, generator=g) > 0.25
    valid[:, 0] = True
    valid[0, Lk // 2:] = False                       # a long fully-masked tail (whole chunks without a live key)
    neg = -1e4 if dtype == torch.float16 else -1e9
    mask = ((~valid).float() * neg).to(dev)
    assert ops._XATTN_STREAM
    out = ops.cross_attention_split(q, 0, kv, 0, H * 64, B, H, T, Lk, add_mask=mask, scale=1.0, split=Lk)
    assert torch.isfinite(out.float()).all()
    ops._SKIP_MASKED = False
    try:
        full = ops.cross_attention_split(q, 0, kv, 0, H * 64, B, H, T, Lk, add_mask=mask, scale=1.0, split=Lk)
    finally:
        ops._SKIP_MASKED = True
    assert torch.equal(full, out)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("S,H,L,use_bias", [(7, 3, 384, True), (5, 2, 200, True), (4, 12, 512, False), (3, 1, 512, True)])
def test_masked_key_blocks_are_skipped_without_changing_the_result(dev, dtype, S, H, L, use_bias):
    """ops.key_block_live: 64-key blocks made of masked keys only (padding to text_maxlength) are neither loaded nor computed
    by the attention kernel.  Their softmax weights are exactly 0 in fp32, so the output must be BIT-identical to
    the run that computes every block.  The values are held against the fp64 oracle in tests/test_attention_fwd_gpu.py
    (test_masked_segments_and_holes, same shapes)."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(S * 100 + L)
    qkv = (torch.randn(S * L, 3 * H * 64, generator=g) * 0.3).to(dtype).to(dev)
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev) if use_bias else None
    lens = torch.randint(1, L + 1, (S,), generator=g)
    lens[0], lens[1] = L, 3                                     # nothing to skip / almost everything
    mask = ((torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0).to(dev)
    if S > 3:
        mask[3, 70:140] = -10000.0                              # a hole of masked keys in the middle (one whole block)
    live = ops.key_block_live(mask)
    assert live is not None and live.shape == (S, (L + 63) // 64) and int(live[1].sum()) == 1 and bool(live[0].all())
    a = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=mask, bias_delta=bias, block_live=live)
    b = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=mask, bias_delta=bias)
    assert torch.equal(a, b), float((a.float() - b.float()).abs().max())
    assert torch.isfinite(a.float()).all()
    # a fully masked segment keeps every block (uniform-over-masked-keys softmax like the reference)
    allm = torch.full((2, L), -10000.0, device=dev)
    assert bool(ops.key_block_live(allm).all())



@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_compacted_cross_kv_rows_path_is_identical(dev, dtype):
    """Cross K | V projected only for the encoder positions inside live 64-key tiles (ops.compact_live_tiles + ops.linear with
    a device-side row count + the stream kernel reading the compacted rows) against the dense projection + the same kernel:
    bit-identical attention output; the compaction tables against a torch restatement."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(5)
    B, H, T, n, Lp, d = 3, 12, 32, 5, 384, 768
    Lk = n * Lp
    enc = (torch.randn(B * Lk, d, generator=g) * 0.5).to(dtype).to(dev)
    wkv = (torch.randn(2 * H * 64, d, generator=g) / 27.7).to(dtype).to(dev)
    q = (torch.randn(B * T, H * 64, generator=g) * 0.5).to(dtype).to(dev)
    lens = torch.randint(20, Lp + 1, (B, n), generator=g)
    lens[0, 0], lens[1, 2] = Lp, 1
    valid = torch.arange(Lp)[None, None, :] < lens[..., None]
    mask = ((~valid).reshape(B, Lk).float() * -1e9).to(dev)
    live = ops.key_block_live(mask)
    enc_live, tile_off, count = ops.compact_live_tiles(enc, live)
    flags = live.reshape(-1).bool().cpu()
    want_off = torch.where(flags, torch.cumsum(flags.int(), 0) - 1, torch.full_like(flags.int(), -1))
    assert torch.equal(tile_off.cpu(), want_off.int()) and int(count) == 64 * int(flags.sum())
    rows = enc.view(-1, 64, d)[flags.to(dev)].reshape(-1, d)
    assert torch.equal(enc_live[: rows.shape[0]], rows)
    kv_live = ops.linear(enc_live, wkv, rows=count)
    kv_dense = ops.linear(enc, wkv)
    assert torch.equal(kv_live[: rows.shape[0]].view(-1, 64, 2 * H * 64), kv_dense.view(-1, 64, 2 * H * 64)[flags.to(dev)])
    a = ops.cross_attention_stream_compact(q, kv_live, live, tile_off, B, H, T, Lk, mask, scale=1.0)
    b = ops.cross_attention_split(q, 0, kv_dense, 0, H * 64, B, H, T, Lk, add_mask=mask, scale=1.0, split=384, tile_live=live)
    assert torch.equal(a, b)
