"""GPU: the FiD decoder cross-attention on key ranges without a usable split-KV segment (`fid._cross_split` pads them with
masked zero rows), and the cross-attention statistics of targets longer than 128 tokens.

  * the padded split-KV forward against the fp64 oracle (oracle/attention_fwd_oracle.py), on padded ranges and on ranges
    with a regular split padded on purpose;
  * dropout forward and backward on a padded range against torch fed the keep mask of the UNPADDED range: a key's mask
    depends on its index only, so padding leaves the real keys' masks alone;
  * a tiny FiD (oracle/model_synth.py) trained at n_context = 3, text_maxlength = 200 with dropout, and the same model
    without dropout padded on purpose against its regular split;
  * the recording forward at 512 target tokens, `Atlas.forward` with eval / std gold scores at 3 x 200, and greedy
    generation over 1031 keys."""
import math
import os

import numpy as np
import pytest
import torch

import attention_fwd_oracle as afo
import atlas_synth
import model_synth
from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
REL = {torch.bfloat16: 4e-2, torch.float16: 6e-3}      # tests/test_dropout_gpu.py
T5_KW = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


@pytest.fixture
def force_pad(monkeypatch):
    """Make every FiD forward take the padded plan, also where the key range has a regular split."""
    from atlas_b200 import fid

    real = fid._cross_split

    def enable():
        monkeypatch.setattr(fid, "_cross_split", lambda Lk, dropout=False: real(Lk, dropout, force_pad=True))

    return enable


def close(got, ref, rel, what=""):
    got, ref = got.detach().float(), ref.detach().float()
    scale = float(ref.abs().max())
    err = float((got - ref).abs().max())
    l2 = float((got - ref).norm() / (ref.norm() + 1e-30))
    assert err <= rel * scale + 1e-6, f"{what}: max err {err:.3e} vs {rel:.1e} x {scale:.3e}"
    assert l2 <= rel, f"{what}: relative L2 error {l2:.3e} > {rel:.1e}"


def _enc_mask(B, Lk, seed, passage=200):
    """FiD's padded passages: each passage of `passage` keys live up to a random length, random holes; bool [B, Lk]."""
    g = torch.Generator().manual_seed(seed)
    j = torch.arange(Lk)
    n_pass = (Lk + passage - 1) // passage
    rows = []
    for _ in range(B):
        lens = torch.randint(passage // 3, passage + 1, (n_pass,), generator=g)
        live = (j % passage < lens[j // passage]) & (torch.rand(Lk, generator=g) >= 0.1)
        live[0] = True
        rows.append(live)
    return torch.stack(rows)


def _padded_inputs(B, H, T, Lk, dtype, dev, seed, dropout=False, force=False, all_masked_row=False):
    from atlas_b200 import fid

    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B * T, H * 64, generator=g) * 0.4).to(dtype).to(dev)
    kv = (torch.randn(B * Lk, 2 * H * 64, generator=g) * 0.4).to(dtype).to(dev)
    enc_mask = _enc_mask(B, Lk, seed)
    if all_masked_row:
        enc_mask[-1] = False
    enc_mask = enc_mask.to(dev)
    split, Lk_pad = fid._cross_split(Lk, dropout=dropout, force_pad=force)
    assert Lk_pad > Lk
    return q, kv, enc_mask, split, Lk_pad


# (B, H, T, Lk): 600 = 3 x 200 and 6000 = 30 x 200 have regular splits (padded on purpose), 1031 has none;
# T > 64 keeps the split-KV kernel (the stream kernel takes few target tokens over long ranges unpadded)
FWD_CASES = [(3, 4, 80, 600), (2, 3, 96, 1031), (1, 12, 72, 6000)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,T,Lk", FWD_CASES, ids=[f"Lk{c[3]}" for c in FWD_CASES])
def test_padded_cross_attention_matches_fp64(dev, dtype, B, H, T, Lk):
    """out and lse of the split-KV kernel + combine on the padded range, element by element within the oracle's bound of
    the unpadded attention.  fp16 adds a batch row whose real keys are all masked: the pad keys, masked twice as hard,
    still weigh 0."""
    from atlas_b200 import fid, ops

    q, kv, enc_mask, split, Lk_pad = _padded_inputs(B, H, T, Lk, dtype, dev, seed=Lk + T, force=True,
                                                    all_masked_row=dtype == torch.float16 and B > 1)
    mask = fid._cross_mask(enc_mask, B, Lk, dtype)
    mask_pad = fid._cross_mask(enc_mask, B, Lk, dtype, Lk_pad)
    assert torch.equal(mask_pad[:, :Lk], mask)
    kv_pad = fid._pad_keys(kv, B, Lk, Lk_pad)
    HD = H * 64
    out, lse = ops.cross_attention_split(q, 0, kv_pad, 0, HD, B, H, T, Lk_pad, add_mask=mask_pad, split=split,
                                         return_lse=True, tile_live=ops.key_block_live(mask_pad))
    Q = q.double().view(B, T, H, 64)
    K = kv[:, :HD].double().view(B, Lk, H, 64)
    V = kv[:, HD:].double().view(B, Lk, H, 64)
    O64, lse64, bo, bl = afo.forward_bound(Q, K, V, mask.double(), None, 1.0, 0.0, dtype=dtype)
    for what, got, ref, bound in (("out", out, O64.reshape(B * T, HD), bo.reshape(B * T, HD)), ("lse", lse, lse64, bl)):
        assert bool(torch.isfinite(got).all()), what
        worst = float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())
        assert worst <= 1.0, f"{what}: max |got - ref| / bound = {worst:.3g}"
    regular, Lk_reg = fid._cross_split(Lk)
    if Lk_reg == Lk:        # the regular split is held to the same bound
        out_r = ops.cross_attention_split(q, 0, kv, 0, HD, B, H, T, Lk, add_mask=mask, split=regular)
        worst = float(((out_r.double() - O64.reshape(B * T, HD)).abs() / bo.reshape(B * T, HD)).max())
        assert worst <= 1.0


def _ref_attention_dropout(q, k, v, add_mask, keep, inv):
    """fp32 T5 cross-attention with dropout on the probabilities, fed the keep mask (tests/test_dropout_gpu.py)."""
    B, Lq, H, _ = q.shape
    s = torch.einsum("bihd,bjhd->bhij", q, k) + add_mask[:, None, None, :]
    p = torch.softmax(s, dim=-1) * keep.float() * inv
    return torch.einsum("bhij,bjhd->bihd", p, v).reshape(B, Lq, H * 64)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,T,Lk", [(2, 4, 16, 3 * 200), (1, 12, 32, 30 * 200)], ids=["3x200", "30x200"])
def test_padded_cross_attention_dropout_fwd_bwd(dev, dtype, B, H, T, Lk):
    """The training cross-attention (grad_ops.cross_attention) on the padded range with dropout 0.1, forward and backward
    through the pad, against torch autograd of the unpadded attention fed `attention_dropout_mask` of the UNPADDED range."""
    from atlas_b200 import fid, grad_ops, ops

    p = 0.1
    torch.manual_seed(7 + Lk)
    q, kv, enc_mask, split, Lk_pad = _padded_inputs(B, H, T, Lk, dtype, dev, seed=3 + Lk, dropout=True)
    q, kv = q.requires_grad_(), kv.requires_grad_()
    mask = fid._cross_mask(enc_mask, B, Lk, dtype)
    mask_pad = fid._cross_mask(enc_mask, B, Lk, dtype, Lk_pad)
    mask_pad._atlas_block_live = ops.key_block_live(mask_pad)
    dout = torch.randn(B * T, H * 64, generator=torch.Generator().manual_seed(Lk)).to(dtype).to(dev)
    gen = torch.cuda.default_generators[dev.index or 0]
    seed, off = gen.initial_seed() & 0xFFFFFFFFFFFFFFFF, gen.get_offset()
    out = grad_ops.cross_attention(q, fid._pad_keys(kv, B, Lk, Lk_pad), B, H, T, Lk_pad, add_mask=mask_pad, scale=1.0,
                                   split=split, dropout_p=p)
    out.backward(dout)
    keep = ops.attention_dropout_mask(B, H, T, Lk, p, seed, off, dev).bool()
    p_eff = int(p * 65536 + 0.5) / 65536.0
    assert abs(float(keep.float().mean()) - (1 - p_eff)) < 5 * math.sqrt(p_eff * (1 - p_eff) / keep.numel())

    qr, kvr = q.detach().float().requires_grad_(), kv.detach().float().requires_grad_()
    k, v = (t.reshape(B, Lk, H, 64) for t in kvr.split(H * 64, dim=1))
    ref = _ref_attention_dropout(qr.reshape(B, T, H, 64), k, v, mask, keep, 1.0 / (1.0 - p_eff)).reshape(B * T, H * 64)
    ref.backward(dout.float())
    rel = REL[dtype]
    close(out, ref, rel / 2, "cross fwd (dropout, padded)")
    close(q.grad, qr.grad, rel, "dq")
    gk, gv = kv.grad.float().split(H * 64, dim=1)
    rk, rv = kvr.grad.split(H * 64, dim=1)
    close(gv, rv, rel, "dV")
    close(gk, rk, rel, "dK")


def _tiny_fid(dev, dropout, L=200, n_ctx=3, B=2, T=8, dtype=torch.bfloat16):
    from atlas_b200.fid import FiD, T5ConfigLite

    reader = FiD(T5ConfigLite(dropout_rate=dropout, **T5_KW))
    sd, _ = model_synth.fill_state_dict(reader.state_dict(), 202)
    reader.load_state_dict(sd)
    reader = reader.to(dtype).to(dev)
    reader.encoder.config.n_context, reader.encoder.config.bsz = n_ctx, B
    ids, mask, labels = model_synth.fid_inputs(B=B, n_ctx=n_ctx, L=L, T=T)
    return reader, ids.to(dev), mask.to(dev), labels.to(dev)


def _step(reader, ids, mask, labels, seed):
    torch.manual_seed(seed)
    reader.zero_grad(set_to_none=True)
    out = reader(input_ids=ids, attention_mask=mask, labels=labels)
    out[0].backward()
    grads = {n: p.grad.detach().float().clone() for n, p in reader.named_parameters() if p.grad is not None}
    return float(out[0]), out[1].detach().float(), grads


def test_fid_train_step_3x200_with_dropout(dev):
    """`--n_context 3 --text_maxlength 200 --dropout 0.1` (600 keys: padded to 640 under dropout): a full step has a finite
    loss and finite gradients on every parameter, and gradient checkpointing re-derives the same masks."""
    from atlas_b200 import fid

    assert fid._cross_split(600, dropout=True) == (320, 640)
    reader, ids, mask, labels = _tiny_fid(dev, 0.1)
    reader.train()
    l1, _, g1 = _step(reader, ids, mask, labels, 5)
    assert math.isfinite(l1) and len(g1) > 40
    assert all(bool(torch.isfinite(v).all()) for v in g1.values())
    reader.gradient_checkpointing_enable()
    l1c, _, g1c = _step(reader, ids, mask, labels, 5)
    assert l1c == l1
    for n in g1:        # fp32 atomics in a few weight gradients: equal up to summation order
        assert float((g1[n] - g1c[n]).abs().max()) <= 1e-3 * float(g1[n].abs().max()) + 1e-7, n


def test_fid_train_step_padded_equals_regular_split(dev, force_pad):
    """Without dropout 3 x 200 has a regular split (300); padded on purpose, logits, loss and every gradient stay within
    the tolerances the golden training tests hold bf16 to (tests/test_train_gpu.py: 8 % relative L2 per gradient)."""
    reader, ids, mask, labels = _tiny_fid(dev, 0.0)
    reader.train()
    l0, z0, g0 = _step(reader, ids, mask, labels, 5)
    force_pad()
    l1, z1, g1 = _step(reader, ids, mask, labels, 5)
    assert abs(l1 - l0) <= 2e-2 * max(1.0, abs(l0))
    close(z1, z0, 4e-2, "logits")
    assert g0.keys() == g1.keys()
    for n in g0:
        rel = float((g1[n] - g0[n]).norm() / (g0[n].norm() + 1e-30))
        assert rel <= 8e-2, (n, rel)


def _record(reader, ids, mask, dec):
    reader.overwrite_forward_crossattention()
    reader.create_crossattention_storage()
    with torch.no_grad():
        reader(input_ids=ids, attention_mask=mask, decoder_input_ids=dec, use_cache=False)
    return [tuple(t.clone() for t in r) for r in reader._xattn]


def test_recording_forward_512_target_tokens(dev, force_pad, monkeypatch):
    """The recording forward at T = 512 (four 128-token slices of the statistics kernel) over 3 x 200 keys: every row's
    probabilities sum to 1 over the live keys, the first 128 rows are those of a T = 128 forward of the same prefix (the
    decoder is causal), the padded range records what the regular split records, its slices of rows 256..383 and 384..511
    are the statistics kernel's output on those rows of q and lse, and the aggregates are finite."""
    from atlas_b200 import ops
    from atlas_b200.fid import FiD

    reader, ids, mask, _ = _tiny_fid(dev, 0.0)
    reader.eval()
    B, T = 2, 512
    labels = torch.randint(2, 512, (B, T), generator=torch.Generator().manual_seed(9)).to(dev)
    labels[1, 300:] = -100
    dec = reader._shift_right(labels)
    rec = _record(reader, ids, mask, dec)
    assert len(rec) == 2
    live = mask.view(B, 1, -1).expand(B, T, -1)
    for scores, probs, norms in rec:
        assert scores.shape == probs.shape == norms.shape == (B, T, 600)
        sums = probs.double().sum(-1)
        assert float((sums - 1.0).abs().max()) <= 1e-3
        assert float(probs.masked_fill(live, 0).abs().max()) <= 1e-6
    short = _record(reader, ids, mask, dec[:, :128])
    for r, s in zip(rec, short):
        for idx in range(3):        # on the live keys: the masked ones hold the mask value in the scores
            close(r[idx][:, :128][live[:, :128]], s[idx][live[:, :128]], 4e-2, f"record {idx}, rows 0..127")
    force_pad()
    seen = {}
    real_record = FiD._record_xattn

    def spy(self, q, kv, B_, H, T_, Lk, lse, m, layer=None, keys=None):
        seen[layer] = (q.detach().clone(), kv.detach().clone(), H, Lk, lse.clone(), m.clone(), keys)
        return real_record(self, q, kv, B_, H, T_, Lk, lse, m, layer=layer, keys=keys)

    monkeypatch.setattr(FiD, "_record_xattn", spy)
    padded = _record(reader, ids, mask, dec)
    for r, s in zip(rec, padded):
        for idx in range(3):
            close(s[idx][live], r[idx][live], 4e-2, f"padded record {idx}")
    assert sorted(seen) == [0, 1]
    for layer, (q, kv, H, Lk, lse, m, keys) in seen.items():
        assert (Lk, keys) == (640, 600)
        for t0 in (256, 384):
            qs = q.view(B, T, -1)[:, t0:t0 + 128].reshape(B * 128, -1)
            want = ops.cross_attention_stats(qs, 0, kv, 0, H * 64, B, H, 128, Lk, lse[:, :, t0:t0 + 128], add_mask=m,
                                             scale=1.0)
            for idx in range(3):
                assert torch.equal(padded[layer][idx][:, t0:t0 + 128], want[idx][..., :keys]), (layer, t0, idx)
    agg = reader.get_crossattention_scores(3, mask, labels=labels, ids=ids, mode="all")
    assert len(agg) >= 21 and all(bool(torch.isfinite(v).all()) for v in agg.values())
    reader.reset_score_storage()


@pytest.mark.parametrize("mode", ["evalnormsum", "stdnormsum"])
def test_atlas_step_gold_scores_3x200(dev, mode):
    """`Atlas.forward` in training mode with `--text_maxlength 200 --n_context 3 --dropout 0.1` and targets of 160 tokens:
    the eval* gold scores come from a no-grad recording forward, std* from the training forward (padded under dropout);
    both losses are finite and back-propagate."""
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    ret_ids = np.load(os.path.join(GOLDEN_DIR, "atlas_tiny.npz"))["ret_ids"]
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    corpus = atlas_synth.make_corpus()
    passages = [[corpus[int(i)] for i in row[:3]] for row in ret_ids]
    query, target = atlas_synth.make_batch()
    opt = atlas_synth.make_opt(gold_score_mode=mode, temperature_gold=0.1, temperature_score=0.1, text_maxlength=200,
                               target_maxlength=160, n_context=3, retriever_n_context=3,
                               compute_crossattention_stats=(mode == "stdnormsum"))
    reader = FiD(T5ConfigLite(dropout_rate=0.1, **T5_KW))
    sd, _ = model_synth.fill_state_dict(reader.state_dict(), seed=202)
    reader.load_state_dict(sd)
    reader.overwrite_forward_crossattention()
    reader.create_crossattention_storage()
    contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    sd, _ = model_synth.fill_state_dict(contriever.state_dict(), seed=101)
    contriever.load_state_dict(sd)
    model = Atlas(opt, reader.to(dev), DualEncoderRetriever(opt, contriever.to(dev)), reader_tok, retriever_tok).train()
    model.retrieve = lambda *a, **k: (passages, None)
    torch.manual_seed(0)
    stats = {}
    reader_loss, retriever_loss = model(None, query, target, train_retriever=True, iter_stats=stats)
    assert torch.isfinite(reader_loss) and torch.isfinite(retriever_loss) and retriever_loss.requires_grad
    (reader_loss + retriever_loss).backward()
    assert contriever.encoder.layer[0].attention.self.query.weight.grad is not None
    assert all(bool(torch.isfinite(p.grad).all()) for p in reader.parameters() if p.grad is not None)


@pytest.mark.parametrize("dtype", DTYPES)
def test_generate_1031_keys_uncached_matches_cached(dev, dtype):
    """One passage of 1031 tokens (a prime: no split-KV segment divides it): greedy generation re-running the decoder
    prefix (use_cache=False) gives the KV-cached decode's tokens wherever the teacher-forced top-2 gap exceeds the 16-bit
    noise (the rule of tests/test_round2_gpu.py: the encoder is not bit-reproducible run to run).  The teacher-forced
    forward at 80 target tokens runs the split-KV kernel on the padded range."""
    reader, _, _, _ = _tiny_fid(dev, 0.0, n_ctx=1, dtype=dtype)
    reader.eval()
    B, L = 2, 1031
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(2, 512, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.bool)
    mask[1, 700:] = False
    ids = (ids * mask).to(dev)
    mask = mask.to(dev)
    reader.encoder.config.n_context, reader.encoder.config.bsz = 1, B
    with torch.no_grad():
        a = reader.generate(input_ids=ids, attention_mask=mask, max_length=12, min_length=None)
        b = reader.generate(input_ids=ids, attention_mask=mask, max_length=12, min_length=None, use_cache=False)
        tf = reader(input_ids=ids, attention_mask=mask, decoder_input_ids=b[:, :-1], use_cache=False).logits.float()
        # the same prefix padded to 80 tokens: the split-KV kernel over the padded keys, causal rows unchanged
        dec80 = torch.cat([b[:, :-1], b.new_zeros(B, 81 - b.shape[1])], dim=1)
        tf80 = reader(input_ids=ids, attention_mask=mask, decoder_input_ids=dec80, use_cache=False).logits.float()
    close(tf80[:, : tf.shape[1]], tf, 4e-2, "teacher-forced logits, split-KV vs stream kernel")
    top2 = tf.topk(2, dim=-1)[0]
    gap_ok = (top2[..., 0] - top2[..., 1]) > (0.02 if dtype == torch.bfloat16 else 0.005)
    n = min(a.shape[1], b.shape[1])
    compared = 0
    for bi in range(B):
        for t in range(1, n):
            if not bool(gap_ok[bi, t - 1]):
                break                              # a near-tie may legitimately fork the greedy chains from here on
            assert int(a[bi, t]) == int(b[bi, t]), (bi, t, a[bi].tolist(), b[bi].tolist())
            compared += 1
    assert compared >= 2
