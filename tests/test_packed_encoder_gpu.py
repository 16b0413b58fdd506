"""The padding-compacted FiD encoder (fid.py: FiD._encode_rows(packed=True); include/atlas_b200.h "Padding-compacted FiD encoder").

The reference encodes every passage padded to text_maxlength (src/atlas.py:261-270, src/fid.py:32-78).  Here the inference forward
keeps, per passage, the 64-row tiles up to its last live key and runs embedding, projections, attention and norms on those rows
only.  Checked: the segment tables against a torch restatement; the packed attention BIT-identical to the padded kernel on the
kept rows; embedding / expansion round trip; the whole FiD forward (logits, loss, encoder states of the kept rows, zeros at the
dropped ones) against the padded computation."""
import numpy as np
import pytest
import torch

import model_synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _keep_tables(live):
    """The CPU restatement of atlas_b200_segment_tile_scan (oracle/packing_oracle.py) as torch tensors."""
    import packing_oracle

    keep, off, src, rows = packing_oracle.segment_tables(live.cpu().numpy())
    return torch.from_numpy(keep), torch.from_numpy(off), torch.from_numpy(src), rows


@pytest.mark.parametrize("S,nb", [(1, 1), (7, 6), (320, 6), (2500, 3), (33, 9), (1023, 64), (1024, 64), (1025, 64)])
def test_segment_tile_scan(dev, S, nb):
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(S + nb)
    live = (torch.rand(S, nb, generator=g) < 0.5).to(torch.uint8)
    live[0] = 0                                                    # a segment without a live tile keeps all of them
    if S > 2:
        live[1] = 1
        live[2] = 0
        live[2, 0] = 1
    keep, off, src, count = ops.segment_tile_scan(live.to(dev))
    wk, wo, ws, wc = _keep_tables(live)
    assert torch.equal(keep.cpu(), wk) and torch.equal(off.cpu(), wo) and torch.equal(src.cpu(), ws) and int(count) == wc
    # and key_block_live against the oracle's rule on a token mask
    import packing_oracle

    tok = (torch.rand(S, nb * 64, generator=g) < 0.02).long()
    got = ops.key_block_live(((1 - tok).float() * -10000.0).to(dev))
    assert torch.equal(got.cpu(), torch.from_numpy(packing_oracle.live_tiles(tok.numpy())))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("S,H,L,use_bias", [(40, 12, 384, True), (7, 3, 384, True), (5, 2, 320, False), (9, 4, 256, True),
                                            (6, 12, 192, True), (11, 2, 128, True), (4, 3, 64, False)])
def test_attention_packed_equals_padded(dev, dtype, S, H, L, use_bias):
    """Segment s keeps its first n_s tiles; q / k / v / out rows of the kept tiles sit back to back.  Same kernel, same key order:
    the kept rows are bit-identical to the padded run for L > 128 and within a 16-bit rounding tolerance below."""
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(S * 1000 + L)
    nb = L // 64
    qkv = (torch.randn(S * L, 3 * H * 64, generator=g) * 0.3).to(dtype)
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev) if use_bias else None
    lens = torch.randint(1, L + 1, (S,), generator=g)
    lens[0], lens[1] = L, 3
    mask = (torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0
    if S > 3 and L >= 192:
        mask[3, 70:140] = -10000.0                                 # a hole: block 1 of segment 3 is dead but kept (prefix rule)
        lens[3] = max(int(lens[3]), 150)
        mask[3, 140:150] = 0.0
    if S > 4:
        mask[4, :] = -10000.0                                      # no live key at all: keeps every tile
    mask = mask.to(dev)
    live = ops.key_block_live(mask)
    keep, off, src, count = ops.segment_tile_scan(live)
    n_rows = int(count)
    kept = keep.reshape(-1).bool()
    packed = torch.zeros_like(qkv).to(dev)
    packed[:n_rows] = qkv.to(dev).view(-1, 64, 3 * H * 64)[kept].reshape(n_rows, -1)
    packed[n_rows:] = float("nan")                                 # rows past the count must never matter
    out_p = ops.attention_packed(packed, keep, off, S, H, L, mask, bias, scale=1.0,
                                 out=torch.full((S * L, H * 64), 7.0, dtype=dtype, device=dev))
    out_d = ops.attention(qkv.to(dev), 0, qkv.to(dev), H * 64, qkv.to(dev), 2 * H * 64, S, H, L, L, add_mask=mask,
                          bias_delta=bias, scale=1.0, block_live=keep)
    want = out_d.view(-1, 64, H * 64)[kept].reshape(n_rows, -1)
    if L > 128:
        assert torch.equal(out_p[:n_rows], want), float((out_p[:n_rows].float() - want.float()).abs().max())
    else:
        tol = 2e-2 if dtype == torch.bfloat16 else 3e-3
        assert float((out_p[:n_rows].float() - want.float()).abs().max()) <= tol
    assert bool((out_p[n_rows:] == 7.0).all())                     # nothing is written past the packed rows
    # and the padded run with `keep` equals the one with the plain live mask (dead tiles inside the prefix weigh 0)
    out_l = ops.attention(qkv.to(dev), 0, qkv.to(dev), H * 64, qkv.to(dev), 2 * H * 64, S, H, L, L, add_mask=mask,
                          bias_delta=bias, scale=1.0, block_live=live)
    assert torch.equal(out_l, out_d)


def test_embed_and_expand_packed_tiles(dev):
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(3)
    S, nb, d, vocab = 9, 6, 768, 1000
    table = torch.randn(vocab, d, generator=g).to(torch.bfloat16).to(dev)
    ids = torch.randint(0, vocab, (S * nb * 64,), generator=g).to(dev)
    live = (torch.rand(S, nb, generator=g) < 0.6).to(torch.uint8).to(dev)
    keep, off, src, count = ops.segment_tile_scan(live)
    n_rows = int(count)
    kept = keep.reshape(-1).bool()
    h = ops.embed_packed_tiles(ids, table, src)
    assert torch.equal(h[:n_rows], table[ids].view(-1, 64, d)[kept].reshape(n_rows, d)) and float(h[n_rows:].abs().max()) == 0
    assert torch.equal(ops.embed_packed_tiles(ids.to(torch.int32), table, src), h)      # int32 ids like torch's lookup
    back = ops.expand_packed_tiles(h, off).view(-1, 64, d)
    assert torch.equal(back[kept], table[ids].view(-1, 64, d)[kept]) and float(back[~kept].abs().max()) == 0


def test_linear_rows_computes_only_the_counted_rows(dev):
    from atlas_b200 import ops

    g = torch.Generator().manual_seed(4)
    M, K, N = 4096, 768, 2304
    x = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(dev)
    w = (torch.randn(N, K, generator=g) / 27.7).to(torch.bfloat16).to(dev)
    res = (torch.randn(M, N, generator=g) * 0.5).to(torch.bfloat16).to(dev)
    full = ops.linear(x, w, residual=res)
    for rows in (0, 64, 1984, 4096):
        cnt = torch.tensor([rows], dtype=torch.int32, device=dev)
        out = torch.full((M, N), 3.0, dtype=torch.bfloat16, device=dev)
        ss = torch.zeros(M, dtype=torch.float32, device=dev)
        ops.linear(x, w, residual=res, out=out, out_ss=ss, rows=cnt)
        assert torch.equal(out[:rows], full[:rows])
        done = -(-rows // 256) * 256                                # whole 256-row blocks are computed
        assert bool((out[done:] == 3.0).all()) and float(ss[done:].abs().max() if done < M else 0.0) == 0.0
        want_ss = full[:rows].float().pow(2).sum(-1)
        assert torch.allclose(ss[:rows], want_ss, rtol=2e-3, atol=1e-2)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("fuse_norm", [True, False])
def test_fid_forward_packed_equals_padded(dev, dtype, fuse_norm):
    """Whole forward, 2 x 5 passages x 384 positions (22 - 384 real tokens each, one passage fully padded): logits / loss of the
    packed encoder against the padded one (same kernels row for row; the fused-norm statistics accumulate with fp32 atomics, so
    the bar is a few 16-bit ulps, not bit equality), encoder states equal on the kept tiles and 0 on the dropped ones."""
    from atlas_b200 import ops
    from atlas_b200.fid import FiD, T5ConfigLite

    cfg = {k: v for k, v in dict(model_synth.T5_CFG, num_layers=3, num_decoder_layers=2).items()
           if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    model = FiD(T5ConfigLite(**cfg))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 909)
    model.load_state_dict(sd)
    model = model.to(dtype).to(dev).eval()
    model.fuse_norm = fuse_norm
    B, n_ctx, L, T = 2, 5, 384, 8
    ids, mask, labels = model_synth.fid_inputs(seed=5, B=B, n_ctx=n_ctx, L=L, T=T, vocab=cfg["vocab_size"])
    mask = mask.view(B, n_ctx, L).clone()
    mask[0, 1, 22:] = False                                        # one tile
    mask[1, 3, :] = False                                          # a passage of padding only
    mask[1, 0, :] = True                                           # a full one
    ids = (ids.view(B, n_ctx, L) * mask).view(B, -1)
    mask = mask.view(B, -1)
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
    outs = {}
    saved = ops._ENC_PACKED
    try:
        for packed in (True, False):
            ops._ENC_PACKED = packed
            model._graphs.clear()
            with torch.no_grad():
                outs[packed] = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev), use_cache=False)
    finally:
        ops._ENC_PACKED = saved
        model._graphs.clear()
    a, b = outs[True], outs[False]
    scale = max(1.0, float(b.logits.float().abs().max()))
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    assert float((a.logits.float() - b.logits.float()).abs().max()) <= 8 * ulp * scale
    assert abs(float(a[0]) - float(b[0])) <= 2e-2
    live = ops.key_block_live((1.0 - mask.view(B * n_ctx, L).float().to(dev)) * -10000.0)
    keep = ops.segment_tile_scan(live)[0].reshape(-1).bool()
    ea = a.encoder_last_hidden_state.reshape(-1, 64, cfg["d_model"]).float()
    eb = b.encoder_last_hidden_state.reshape(-1, 64, cfg["d_model"]).float()
    assert float(ea[~keep].abs().max()) == 0.0
    escale = max(1.0, float(eb[keep].abs().max()))
    assert float((ea[keep] - eb[keep]).abs().max()) <= 8 * ulp * escale
    assert int(keep.sum()) < keep.numel()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B,L", [(8, 384), (37, 192), (5, 128), (3, 64), (4, 200)])
def test_contriever_packed_equals_padded(dev, dtype, B, L):
    """`Contriever.encode` on the packed rows (queries padded to text_maxlength, index-refresh batches padded to the longest
    passage) against the padded encoder: the hidden states of the kept tiles (bit-identical for L > 128), zeros at the dropped
    tiles, and the pooled embeddings.  L = 200 is not a multiple of 64: padded."""
    from atlas_b200 import ops
    from atlas_b200.retrievers import BertConfigLite, Contriever

    model = Contriever(BertConfigLite(**dict(model_synth.CONTRIEVER_CFG, num_hidden_layers=3)))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 77)
    model.load_state_dict(sd)
    model = model.to(dtype).to(dev).eval()
    ids, mask = model_synth.contriever_inputs(seed=B + L, B=B, L=L, vocab=model_synth.CONTRIEVER_CFG["vocab_size"])
    mask = mask.clone()
    mask[0, 5:] = 0                                                # a 5-token query: one tile
    mask[1, :] = 1
    ids, mask = (ids * mask).to(dev), mask.to(dev)
    if not ops._BERT_PACKED:
        pytest.skip("ATLAS_B200_BERT_PACKED=0")
    saved = ops._ENC_PACKED
    try:
        ops._ENC_PACKED = True
        with torch.no_grad():
            hp = model.encode(ids, mask)
            ep = model(input_ids=ids, attention_mask=mask)
        ops._ENC_PACKED = False
        with torch.no_grad():
            hd = model.encode(ids, mask)
            ed = model(input_ids=ids, attention_mask=mask)
    finally:
        ops._ENC_PACKED = saved
    if L % 64 == 0:
        live = ops.key_block_live((1.0 - mask.float()) * -10000.0)
        keep = ops.segment_tile_scan(live)[0].bool().repeat_interleave(64, dim=1)      # [B, L]
        assert float(hp[~keep].abs().max() if bool((~keep).any()) else 0.0) == 0.0
    else:
        keep = torch.ones_like(mask, dtype=torch.bool)
    tol = (2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10) * max(1.0, float(hd.abs().max()))
    if L > 128:
        assert torch.equal(hp[keep], hd[keep])
        assert torch.equal(ep, ed)
    else:
        assert float((hp[keep].float() - hd[keep].float()).abs().max()) <= 4 * tol
        assert float((ep.float() - ed.float()).abs().max()) <= 4 * tol
