"""The padding-compacted FiD encoder in the training step and at text_maxlength up to 576 (include/atlas_b200.h "Padding-compacted
FiD encoder"; fid.py FiD._encode_train / _encode_rows).

A padded position never reaches a live one, so on every live row the packed step computes what the padded step computes,
dropout masks included.  Checked: the packed attention forward (with lse and dropout) and backward against the padded kernels
on the kept rows; the row-mapped hidden-state dropout bit for bit; whole training steps packed against padded, with a
negative control that shows the bound catches mismatched dropout masks; the no-grad forward and greedy generation at 512
and 576 tokens."""
import pytest
import torch

import model_synth

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
T5_KW = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _segments(S, L, seed):
    """Additive key mask [S, L]: bench.py-like lengths (20 query + U[128, 256] passage tokens, capped at L), plus a segment with
    one live token, a full-length one and a fully masked one (which keeps every tile)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.clamp(20 + torch.randint(128, 257, (S,), generator=g), max=L)
    lens[0], lens[1] = 1, L
    mask = (torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0
    mask[2, :] = -10000.0
    return mask


def _packed_setup(dev, dtype, S, H, L, use_bias, seed):
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(S * L, 3 * H * 64, generator=g) * 0.35).to(dtype).to(dev)
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev) if use_bias else None
    mask = _segments(S, L, seed).to(dev)
    keep, off, src, count = ops.segment_tile_scan(ops.key_block_live(mask))
    rows = int(count)
    kept = keep.reshape(-1).bool()
    assert keep[0].sum() == 1 and keep[1].sum() == L // 64 and keep[2].sum() == L // 64
    packed = qkv.view(-1, 64, 3 * H * 64)[kept].reshape(rows, -1).contiguous()
    return qkv, packed, bias, mask, keep, off, src, rows, kept


def _close16(got, want, dtype, what):
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    scale = max(1.0, float(want.float().abs().max()))
    err = float((got.float() - want.float()).abs().max())
    assert err <= 2 * ulp * scale, (what, err)


SHAPES = [(L, H) for L in (64, 192, 384, 448, 512, 576) for H in (8, 12)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("use_bias", [True, False])
@pytest.mark.parametrize("L,H", SHAPES)
def test_packed_attention_forward(dev, dtype, p_drop, use_bias, L, H):
    """attention_packed(lse=True, dropout) on the kept rows against atlas_b200_attention_train on the padded layout."""
    from atlas_b200 import ops

    S = 7
    qkv, packed, bias, mask, keep, off, _, rows, kept = _packed_setup(dev, dtype, S, H, L, use_bias, L * 10 + H)
    drop = (p_drop, 4321, 96) if p_drop else None
    out_p, lse_p = ops.attention_packed(packed, keep, off, S, H, L, mask, bias, lse=True, dropout=drop)
    out_d, lse_d = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=mask, bias_delta=bias,
                                 return_lse=True, dropout=drop, block_live=keep)
    _close16(out_p, out_d.view(-1, 64, H * 64)[kept].reshape(rows, -1), dtype, "O")
    row_kept = kept.view(S, 1, L // 64, 1).expand(S, H, L // 64, 64).reshape(S, H, L)
    assert torch.allclose(lse_p[row_kept], lse_d[row_kept], rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("use_bias", [True, False])
@pytest.mark.parametrize("L,H", SHAPES)
def test_packed_attention_backward(dev, dtype, use_bias, L, H):
    """attention_packed_bwd against atlas_b200_attention_bwd_train on the padded layout, with dropout: dQ / dK / dV on the kept
    rows and dbias.  The padded rows' output gradient is 0, as in the model (the decoder's cross-attention masks them)."""
    from atlas_b200 import ops

    S = 7
    qkv, packed, bias, mask, keep, off, _, rows, kept = _packed_setup(dev, dtype, S, H, L, use_bias, L * 10 + H + 1)
    drop = (0.1, 99, 12)
    HD = H * 64
    out_p, lse_p = ops.attention_packed(packed, keep, off, S, H, L, mask, bias, lse=True, dropout=drop)
    out_d, lse_d = ops.attention(qkv, 0, qkv, HD, qkv, 2 * HD, S, H, L, L, add_mask=mask, bias_delta=bias, return_lse=True,
                                 dropout=drop, block_live=keep)
    g = torch.Generator().manual_seed(L + H)
    dout_d = torch.randn(S * L, HD, generator=g).to(dtype).to(dev)
    dout_d.view(-1, 64, HD)[~kept] = 0
    dout_p = dout_d.view(-1, 64, HD)[kept].reshape(rows, HD).contiguous()
    dqkv_p, dbias_p = ops.attention_packed_bwd(packed, out_p, dout_p, keep, off, S, H, L, mask, bias, lse_p,
                                               need_dbias=use_bias, dropout=drop)
    dqkv_d = torch.empty_like(qkv)
    dbias_d = ops.attention_bwd(qkv, 0, qkv, HD, qkv, 2 * HD, out_d, dout_d, dqkv_d, 0, dqkv_d, HD, dqkv_d, 2 * HD, S, H, L, L,
                                add_mask=mask, bias_delta=bias, need_dbias=use_bias, lse=lse_d, dropout=drop,
                                block_live=keep)
    want = dqkv_d.view(-1, 64, 3 * HD)[kept].reshape(rows, -1)
    for c, name in enumerate(("dQ", "dK", "dV")):
        _close16(dqkv_p[:, c * HD:(c + 1) * HD], want[:, c * HD:(c + 1) * HD], dtype, name)
    if use_bias:
        rel = float((dbias_p - dbias_d).norm() / dbias_d.norm())
        assert rel <= 1e-4, rel
    else:
        assert dbias_p is None


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("residual", [False, True])
def test_row_mapped_dropout(dev, dtype, residual):
    """ops.dropout with row_tiles equals the padded-layout dropout on the mapped rows, bit for bit."""
    from atlas_b200 import ops

    S, L, d = 9, 512, 768
    mask = _segments(S, L, 3).to(dev)
    keep, off, src, count = ops.segment_tile_scan(ops.key_block_live(mask))
    rows = int(count)
    kept = keep.reshape(-1).bool()
    g = torch.Generator().manual_seed(8)
    x = torch.randn(S * L, d, generator=g).to(dtype).to(dev)
    res = torch.randn(S * L, d, generator=g).to(dtype).to(dev) if residual else None
    pick = lambda t: t.view(-1, 64, d)[kept].reshape(rows, d).contiguous()   # noqa: E731
    want = pick(ops.dropout(x, 0.1, 77, 1234, residual=res))
    got = ops.dropout(pick(x), 0.1, 77, 1234, residual=pick(res) if residual else None, row_tiles=src[: rows // 64])
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def _reader(kind, dtype, dev, dropout):
    from atlas_b200.fid import FiD, T5ConfigLite

    kw = dict(T5_KW, dropout_rate=dropout)
    if kind == "relu":
        kw.update(d_model=512, num_heads=8, d_ff=2048, feed_forward_proj="relu", tie_word_embeddings=True)
    model = FiD(T5ConfigLite(**kw))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    if kind == "relu":
        sd["lm_head.weight"] = sd["shared.weight"].clone()
    model.load_state_dict(sd)
    return model.to(dtype).to(dev)


def _inputs(L, n_ctx, B, T, dev):
    ids, _, labels = model_synth.fid_inputs(seed=L, B=B, n_ctx=n_ctx, L=L, T=T)
    mask = _segments(B * n_ctx, L, L + 1).view(B, n_ctx * L) == 0
    return (ids * mask).to(dev), mask.to(dev), labels.to(dev)


def _step(reader, ids, mask, labels, seed, packed):
    from atlas_b200 import ops

    saved = ops._ENC_PACKED
    try:
        ops._ENC_PACKED = packed
        torch.manual_seed(seed)
        reader.zero_grad(set_to_none=True)
        out = reader(input_ids=ids, attention_mask=mask, labels=labels)
        out[0].backward()
    finally:
        ops._ENC_PACKED = saved
    return float(out[0].detach()), {n: p.grad.detach().float().clone() for n, p in reader.named_parameters() if p.grad is not None}


def _worst(g, ref):
    assert g.keys() == ref.keys()
    return max(float((g[n] - ref[n]).norm() / (ref[n].norm() + 1e-30)) for n in ref)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ckpt", [False, True])
@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("L", [384, 512])
@pytest.mark.parametrize("kind", ["tiny", "relu"])
def test_train_step_packed_equals_padded(dev, dtype, ckpt, p_drop, L, kind):
    """The whole training step with ATLAS_B200_ENC_PACKED on and off, same seed: loss within 1e-3 relative, every gradient
    within 1e-2 relative L2.  With dropout, the padded step under another seed misses that bound by at least 10x."""
    B, n_ctx, T = 2, 4, 8
    reader = _reader(kind, dtype, dev, p_drop)
    reader.encoder.config.n_context, reader.encoder.config.bsz = n_ctx, B
    reader.train()
    if ckpt:
        reader.gradient_checkpointing_enable()
    ids, mask, labels = _inputs(L, n_ctx, B, T, dev)
    l_pad, g_pad = _step(reader, ids, mask, labels, 5, packed=False)
    l_pk, g_pk = _step(reader, ids, mask, labels, 5, packed=True)
    assert abs(l_pk - l_pad) <= 1e-3 * abs(l_pad), (l_pk, l_pad)
    worst = _worst(g_pk, g_pad)
    assert worst <= 1e-2, worst
    if p_drop:
        _, g_other = _step(reader, ids, mask, labels, 6, packed=False)
        assert _worst(g_other, g_pad) >= 10 * 1e-2


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [512, 576])
def test_no_grad_forward_and_generation_packed_equals_padded(dev, dtype, L):
    """The no-grad forward at 384 < L <= 576 runs packed (the resident attention kernel on the packed rows): logits and loss
    against the padded forward, and greedy generation gives the same tokens."""
    from atlas_b200 import ops

    B, n_ctx, T = 2, 4, 8
    model = _reader("tiny", dtype, dev, 0.0).eval()
    model.fuse_norm = False           # no fp32 atomics in the norm statistics: the kept rows compute bit for bit the same
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    ids, mask, labels = _inputs(L, n_ctx, B, T, dev)
    assert ops.encoder_packs(ops.key_block_live((1.0 - mask.view(-1, L).float()) * -10000.0), L)
    outs, gens = {}, {}
    saved = ops._ENC_PACKED
    try:
        for packed in (True, False):
            ops._ENC_PACKED = packed
            model._graphs.clear()
            with torch.no_grad():
                outs[packed] = model(input_ids=ids, attention_mask=mask, labels=labels, use_cache=False)
                gens[packed] = model.generate(input_ids=ids, attention_mask=mask, max_length=12)
    finally:
        ops._ENC_PACKED = saved
        model._graphs.clear()
    a, b = outs[True], outs[False]
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    scale = max(1.0, float(b.logits.float().abs().max()))
    assert float((a.logits.float() - b.logits.float()).abs().max()) <= 8 * ulp * scale
    assert abs(float(a[0]) - float(b[0])) <= 1e-3 * max(1.0, abs(float(b[0])))
    assert torch.equal(gens[True], gens[False])
