"""Beam search of `FiD.generate(num_beams > 1)`: the selection kernels (csrc/beam.cu) against the numpy restatement of
transformers 4.18 beam search (oracle/beam_oracle.py), the ancestry-gathered self-attention against the existing decode
kernel on an explicitly gathered cache, whole generations against the oracle driven by the GPU's own step logits, and the
`Atlas.generate` surface."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import atlas_synth
import beam_oracle as bo
import fid_cpu
import model_synth

pytestmark = pytest.mark.gpu

EOS, PAD = 1, 0
MODE = {torch.float16: "fp16", torch.bfloat16: "bf16"}
NAN_BITS = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _tiny_fid(dev, dtype, **over):
    from atlas_b200.fid import FiD, T5ConfigLite

    cfg = {k: v for k, v in dict(model_synth.T5_CFG, **over).items()
           if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    model = FiD(T5ConfigLite(**cfg))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    return model.to(dtype).to(dev).eval(), sd


def _beam_state(B, nb, Tmax, dev):
    from atlas_b200.fid import FiD

    fake = SimpleNamespace(config=SimpleNamespace(num_heads=1, num_decoder_layers=0))
    st = FiD._BeamState(fake, B, nb, 64, Tmax, torch.float16, dev)
    st.reset(0, PAD)
    return st


def _finalize(st, max_length, length_penalty):
    from atlas_b200.fid import FiD

    fake = SimpleNamespace(config=SimpleNamespace(pad_token_id=PAD, eos_token_id=EOS))
    return FiD._finalize_beams(fake, st, max_length, length_penalty).cpu().numpy()


def _gpu_hyps(st, b):
    n = int(st.hyp_state[b, 0])
    ins = st.hyp_ins[b, :n].tolist()
    order = sorted(range(n), key=lambda j: ins[j])
    return [(float(st.hyp_score[b, j]), st.hyp_tok[b, j, : int(st.hyp_len[b, j])].tolist()) for j in order]


# ------------------------------------------------------------------------------------------------------------------------
# 1. the selection kernels on synthetic logits, step by step against the oracle
# ------------------------------------------------------------------------------------------------------------------------
# (B, nb, V, length_penalty)
SELECT_CASES = [(5, 2, 3, 1.0), (3, 3, 1000, 0.5), (2, 4, 32128, 2.0), (4, 8, 1000, 1.0), (2, 16, 32128, 1.0),
                (1, 16, 3, 0.0)]


def _synthetic_logits(R, V, dtype, g, spread=4.0):
    x = torch.randn(R, V, generator=g) * spread
    x = x.to(dtype).float()
    # planted ties inside rows: a block of tokens repeats the row's largest values
    top = x.topk(min(4, V), dim=1).indices
    if V >= 16:
        x[:, V - 4:] = x.gather(1, top)
    return x


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,nb,V,lp", SELECT_CASES, ids=[f"B{c[0]}nb{c[1]}V{c[2]}lp{c[3]}" for c in SELECT_CASES])
def test_selection_kernels_match_oracle(dev, dtype, B, nb, V, lp):
    """beam_topk + beam_select over a whole search: the processed log-probs (EOS ban, additive mask, 16-bit rounding)
    against the fp64 log-softmax within one 16-bit rounding; then, fed those log-probs, the oracle must produce the same
    tokens, parents, beam scores (bit for bit: the same fp32 sums), done flags, hypotheses and finalize output.  Planted:
    ties inside rows, exact ties across beams (two beams given equal scores and equal logits), EOS pushed to the top in
    some batch elements at different steps, and a 0 / -inf mask on some steps."""
    from atlas_b200 import ops

    R, max_length, min_length = B * nb, 7, 2
    g = torch.Generator().manual_seed(1000 * nb + V)
    st = _beam_state(B, nb, max_length, dev)
    orc = bo.BeamSearch(B, nb, V, max_length, min_length, lp, mode="fp32", eos=EOS, pad=PAD)
    lp_out = torch.empty((R, V), dtype=torch.float32, device=dev)
    step = 0
    while not orc.finished:
        x = _synthetic_logits(R, V, dtype, g)
        if step >= 1 and nb >= 2:                      # exact ties across beams 0 and 1 of batch element 0
            x[1] = x[0]
            st.beam_scores[1] = st.beam_scores[0]
            orc.beam_scores[1] = orc.beam_scores[0]
        for b in range(B):                              # batch element b: EOS far on top from step b + 1
            if step >= b + 1:
                x[b * nb:(b + 1) * nb, EOS] = x[b * nb:(b + 1) * nb].max(dim=1).values + 10.0 + 0.5 * (b % 2)
        mask = None
        if step % 2 == 1:
            mask = torch.where(torch.rand(R, V, generator=g) < 0.3, -float("inf"), 0.0)
            mask[:, :2] = 0.0
        logits = x.to(dtype).to(dev)
        t = int(st.t_dev)
        ops.beam_topk(logits, st.beam_scores, st.t_dev, 2 * nb, EOS, min_length, True,
                      add_mask=mask.to(dev) if mask is not None else None, cand_score=st.cand_score, cand_tok=st.cand_tok,
                      lp_out=lp_out)
        ops.beam_select(st.cand_score, st.cand_tok, nb, V, *st.select_buffers(), EOS, PAD, lp)
        # the processed log-probs: one 16-bit rounding of the fp64 log-softmax, the ban and the mask exactly
        ref = bo.round_to(bo.log_softmax(logits.double().cpu().numpy()), MODE[dtype])
        if t + 1 < min_length:
            ref[:, EOS] = -np.inf
        if mask is not None:
            ref = ref + mask.numpy()
        got = lp_out.cpu().numpy().astype(np.float64)
        fin = np.isfinite(ref)
        with np.errstate(invalid="ignore"):
            assert np.array_equal(np.isfinite(got), fin) and np.array_equal(np.isnan(got), np.isnan(ref))
        # one 16-bit rounding plus the fp32 error of log(sum): near 0 (a dominant token, sum = 1 + eps) the latter is ~1e-7
        # absolute, more than a 16-bit ulp there - the reference's fp32 log_softmax carries the same error
        bound = bo.ulp16(ref[fin], MODE[dtype]) + 4 * 2.0 ** -23 * (1 + np.abs(ref[fin]))
        assert (np.abs(got[fin] - ref[fin]) <= bound).all()
        rec = orc.step(logprobs=got)
        assert st.tok_in.cpu().tolist() == rec["tokens"].tolist(), step
        assert st.parent.cpu().tolist() == rec["parents"].tolist(), step
        assert np.array_equal(st.beam_scores.cpu().numpy(), rec["scores"].astype(np.float32)), step
        assert [bool(d) for d in st.done.cpu().tolist()] == orc.done, step
        assert st.sequences(t + 1).cpu().tolist() == orc.sequences(), step
        for b in range(B):
            assert _gpu_hyps(st, b) == orc.hyps[b].beams, (step, b)
        step += 1
    assert int(st.t_dev) == step
    assert np.array_equal(_finalize(st, max_length, lp), orc.finalize())
    if V >= 2 * nb:     # (with V < 2 nb most beams carry the -1e9 start scores, and no batch element can finish)
        assert any(orc.done), "no batch element finished: the case exercises nothing of the scorer"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_selection_all_minus_inf_and_nan_rows(dev, dtype):
    """Rows of -inf or NaN logits (log_softmax: NaN everywhere) and a row whose only finite logit is banned: NaN ranks above
    every number and ties go to the lower index, so every picked token is in [0, V) and the oracle agrees."""
    from atlas_b200 import ops

    B, nb, V, max_length = 3, 4, 1000, 3      # two steps: NaN beam scores reach the scorer, never a full hypothesis list
    R = B * nb
    g = torch.Generator().manual_seed(7)
    st = _beam_state(B, nb, max_length, dev)
    orc = bo.BeamSearch(B, nb, V, max_length, 10, 1.0, mode="fp32", eos=EOS, pad=PAD)   # EOS banned throughout
    lp_out = torch.empty((R, V), dtype=torch.float32, device=dev)
    while not orc.finished:
        x = _synthetic_logits(R, V, dtype, g)
        x[0] = -float("inf")
        x[nb + 1] = float("nan")
        x[2 * nb, :] = -float("inf")
        x[2 * nb, EOS] = 3.0
        ops.beam_topk(x.to(dtype).to(dev), st.beam_scores, st.t_dev, 2 * nb, EOS, 10, True, cand_score=st.cand_score,
                      cand_tok=st.cand_tok, lp_out=lp_out)
        ops.beam_select(st.cand_score, st.cand_tok, nb, V, *st.select_buffers(), EOS, PAD, 1.0)
        rec = orc.step(logprobs=lp_out.cpu().numpy().astype(np.float64))
        tok = st.tok_in.cpu()
        assert bool(((tok >= 0) & (tok < V)).all())
        assert tok.tolist() == rec["tokens"].tolist() and st.parent.cpu().tolist() == rec["parents"].tolist()
    assert np.array_equal(_finalize(st, max_length, 1.0), orc.finalize())


def test_beam_select_rejects_too_many_beams(dev):
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    nb = ops.MAX_BEAMS + 1                       # well-formed buffers: the kernel entry's own limit refuses the call
    st = _beam_state(1, nb, 4, dev)
    with pytest.raises(AtlasB200Error, match="nb <= 16"):
        ops.beam_select(st.cand_score, st.cand_tok, nb, 100, *st.select_buffers(), EOS, PAD, 1.0)


# ------------------------------------------------------------------------------------------------------------------------
# 2. the ancestry-gathered self-attention
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_beam_self_attention_equals_gathered_cache(dev, dtype):
    """Each step under a random ancestry: the output equals decode_self_attention on the cache gathered along the
    ancestry, bit for bit; the new K | V lands in slot (r, t) and no other slot changes; a captured graph of one step
    (the ancestry buffer chosen by t's parity on the device) replays the eager steps bit for bit."""
    from atlas_b200 import ops
    from atlas_b200.fid import bias_by_delta

    B, nb, H, Tmax = 2, 3, 4, 9
    R, HD = B * nb, H * 64
    g = torch.Generator().manual_seed(11)
    bias = bias_by_delta((torch.randn(32, H, generator=g) * 2.0).to(dev), Tmax, Tmax, False, 32)
    rows16 = (torch.randn(Tmax, R, 3 * HD, generator=g) * 2.0).to(dtype).to(dev)
    # ancestry per step: rows pick parents inside their batch element
    ancs = [torch.arange(R, dtype=torch.int32)[:, None].repeat(1, Tmax)]
    for t in range(Tmax - 1):
        par = torch.tensor([b * nb + int(torch.randint(nb, (1,), generator=g)) for b in range(B) for _ in range(nb)])
        nxt = ancs[-1].clone()
        nxt[:, : t + 1] = ancs[-1][par, : t + 1]
        nxt[:, t + 1] = torch.arange(R, dtype=torch.int32)
        ancs.append(nxt)
    anc = torch.zeros((2, R, Tmax), dtype=torch.int32, device=dev)
    cache = torch.empty((R, Tmax, 2 * HD), dtype=dtype, device=dev)
    cache.view(torch.int16).fill_(NAN_BITS[dtype])
    t_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    qkv = torch.empty((R, 3 * HD), dtype=dtype, device=dev)
    out = torch.empty((R, HD), dtype=dtype, device=dev)
    eager = []
    for t in range(Tmax):
        anc[t & 1].copy_(ancs[t])
        qkv.copy_(rows16[t])
        t_dev.fill_(t)
        before = cache.clone()
        ops.decode_self_attention_beam(qkv, cache, t_dev, anc, H, bias_delta=bias, out=out)
        eager.append(out.clone())
        c16, b16 = cache.view(torch.int16), before.view(torch.int16)
        assert torch.equal(c16[:, t], rows16[t, :, HD:].contiguous().view(torch.int16)), t
        assert torch.equal(c16[:, :t], b16[:, :t]) and torch.equal(c16[:, t + 1:], b16[:, t + 1:]), t
        a = ancs[t][:, : t + 1].long().to(dev)
        gathered = torch.empty_like(cache)
        gathered.view(torch.int16).fill_(NAN_BITS[dtype])
        gathered[:, : t + 1] = cache[a, torch.arange(t + 1, device=dev)[None, :]]
        ref = ops.decode_self_attention(qkv, gathered, t_dev, H, bias_delta=bias)
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), t

    cache.view(torch.int16).fill_(NAN_BITS[dtype])
    t_dev.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decode_self_attention_beam(qkv, cache, t_dev, anc, H, bias_delta=bias, out=out)
        t_dev.add_(1)
    for t in range(Tmax):
        anc[t & 1].copy_(ancs[t])
        qkv.copy_(rows16[t])
        graph.replay()
        assert torch.equal(out.view(torch.int16), eager[t].view(torch.int16)), t


# ------------------------------------------------------------------------------------------------------------------------
# 3. whole generations on the tiny FiD against the oracle driven by the GPU's step logits
# ------------------------------------------------------------------------------------------------------------------------
def _passages(B, n_ctx, L, lens, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, vocab, (B, n_ctx, L), generator=g)
    lens = torch.tensor(lens).view(B, n_ctx)
    mask = torch.arange(L)[None, None, :] < lens[..., None]
    ids = ids * mask
    ids.scatter_(2, (lens - 1)[..., None], EOS)
    return ids.view(B, n_ctx * L), mask.view(B, n_ctx * L)


# 3 passages of 128 tokens per batch element; short passages leave dead 64-key tiles, one holds only EOS
N_CTX, L_TOK, LENS = 3, 128, [5, 128, 1, 40, 2, 1]


def _recorded_generate(model, ids, mask, **kw):
    """generate() with every step's logits and the selection it led to recorded: steps[s] = (logits [R, V], tok_in and
    parent after step s)."""
    logits_of, sel = [], []
    decode_step = model._decode_step_logits

    def recording(st):
        if logits_of:
            sel.append((st.tok_in.cpu().clone(), st.parent.cpu().clone()))
        out = decode_step(st)
        logits_of.append(out.clone())
        recording.st = st
        return out

    model._decode_step_logits = recording
    try:
        seq = model.generate(input_ids=ids, attention_mask=mask, **kw)
    finally:
        model._decode_step_logits = decode_step
    st = recording.st
    sel.append((st.tok_in.cpu().clone(), st.parent.cpu().clone()))
    return seq, logits_of, sel, st


def _drive_oracle(orc, logits_of, sel, mode):
    """Step the oracle with the GPU's logits; compare every selection.  Returns the number of exempted decisions (a
    mismatch at a step whose oracle margin is under 2 ulps of the 16-bit log-prob: the beams diverge there, so the
    comparison stops)."""
    s = 0
    while not orc.finished:
        rec = orc.step(logits_of[s].double().cpu().numpy())
        tok, par = sel[s]
        same = tok.tolist() == rec["tokens"].tolist() and par.tolist() == rec["parents"].tolist()
        if not same:
            tight = rec["margin"] < 2 * float(bo.ulp16(rec["lp_scale"], mode))
            assert tight, (f"step {s}: GPU tokens {tok.tolist()} parents {par.tolist()} vs oracle "
                           f"{rec['tokens'].tolist()} {rec['parents'].tolist()}, margin {rec['margin']:.3g}")
            return 1
        s += 1
    return 0


def _ancestors(sel, T, R):
    """a[s][r]: the row that held final row r's prefix at step s (s = 0 .. T)."""
    a = [None] * (T + 1)
    a[T] = np.arange(R)
    for s in range(T - 1, -1, -1):
        a[s] = sel[s][1].numpy()[a[s + 1]]
    return a


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nb", [2, 4])
@pytest.mark.parametrize("lp", [0.5, 1.0, 2.0])
def test_generate_beams_match_oracle(dev, dtype, nb, lp):
    """Eager beam generation (min_length 3, max_length 10): every selection equals the oracle's on the same step logits
    (exempt only below a 2-ulp margin; the count is printed), the output equals the oracle's finalize, the beam rows' step
    logits match fid_cpu's fp32 teacher-forced logits of the same sequences within 2x of the GPU's own teacher-forced
    error (a wrong ancestry gather would not), and the graph-replayed generation and a repeat equal the eager one."""
    model, sd = _tiny_fid(dev, dtype)
    model.fuse_norm = False                       # bit-reproducible encoder (no fp32-atomic row statistics)
    B, max_length, min_length = 2, 10, 3
    model.encoder.config.n_context, model.encoder.config.bsz = N_CTX, B
    ids, mask = _passages(B, N_CTX, L_TOK, LENS, model_synth.T5_CFG["vocab_size"], seed=nb + 10)
    kw = dict(max_length=max_length, min_length=min_length, num_beams=nb, length_penalty=lp)
    model.cuda_graphs = False
    with torch.no_grad():
        seq, logits_of, sel, st = _recorded_generate(model, ids.to(dev), mask.to(dev), **kw)
    V = model.config.vocab_size
    orc = bo.BeamSearch(B, nb, V, max_length, min_length, lp, mode=MODE[dtype], eos=EOS, pad=PAD)
    exempt = _drive_oracle(orc, logits_of, sel, MODE[dtype])
    print(f"{dtype} nb={nb} lp={lp}: {orc.cur_len - 1} oracle steps, {len(logits_of)} GPU steps, {exempt} exemptions")
    if not exempt:
        assert seq.cpu().numpy().tolist() == orc.finalize().tolist()

    # step logits of the beam rows against the fp32 CPU oracle's teacher-forced logits of the same sequences
    T = len(logits_of)
    R = B * nb
    final = st.sequences(T).cpu()                                     # [R, T + 1]
    anc = _ancestors(sel, T, R)
    got = torch.stack([logits_of[s].float().cpu()[torch.from_numpy(anc[s])] for s in range(T)], 1)   # [R, T, V]
    ids_r, mask_r = ids.repeat_interleave(nb, 0), mask.repeat_interleave(nb, 0)
    model.encoder.config.bsz = R
    with torch.no_grad():
        tf = model(input_ids=ids_r.to(dev), attention_mask=mask_r.to(dev), decoder_input_ids=final[:, :T].to(dev),
                   use_cache=False).logits.float().cpu()
    _, ref, _ = fid_cpu.fid_forward({k: v.float() for k, v in sd.items()}, model_synth.T5_CFG, ids_r, mask_r, final[:, :T],
                                    n_context=N_CTX)
    err_step, err_tf = float((got - ref).abs().max()), float((tf - ref).abs().max())
    print(f"max |logits - fp32 oracle|: beam steps {err_step:.3g}, teacher-forced {err_tf:.3g}, ratio {err_step / err_tf:.3f}")
    assert err_step <= 2.0 * err_tf

    model.encoder.config.bsz = B
    model.cuda_graphs = True
    with torch.no_grad():
        g1 = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), **kw)
        g2 = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), **kw)
    assert torch.equal(g1, seq) and torch.equal(g2, seq)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_generate_beams_prefix_constraint(dev, dtype):
    """prefix_allowed_tokens_fn (the decoder prompt of src/atlas.py:621-636) through the eager beam path: the function sees
    every row's sequence rebuilt through the ancestry, and the result equals the oracle's with the same function."""
    model, _ = _tiny_fid(dev, dtype)
    model.fuse_norm = False
    B, nb, max_length = 2, 3, 8
    model.encoder.config.n_context, model.encoder.config.bsz = N_CTX, B
    ids, mask = _passages(B, N_CTX, L_TOK, LENS, model_synth.T5_CFG["vocab_size"], seed=5)
    forced = [[17, 23], [31, 5]]
    seen = []

    def allowed(b, sent):
        seen.append((b, [int(x) for x in sent]))
        pos = len(sent)
        return [forced[b][pos - 1]] if pos <= 2 else list(range(2, 300))

    with torch.no_grad():
        seq, logits_of, sel, _ = _recorded_generate(model, ids.to(dev), mask.to(dev), max_length=max_length, num_beams=nb,
                                                    min_length=None, prefix_allowed_tokens_fn=allowed)
    assert seq[:, 1:3].tolist() == forced
    assert all(s[0] == 0 for _, s in seen) and len(seen) >= B * nb * 3
    orc = bo.BeamSearch(B, nb, model.config.vocab_size, max_length, None, 1.0, mode=MODE[dtype], eos=EOS, pad=PAD,
                        prefix_fn=allowed)
    exempt = _drive_oracle(orc, logits_of, sel, MODE[dtype])
    print(f"prefix constraint {dtype}: {exempt} exemptions")
    if not exempt:
        assert seq.cpu().numpy().tolist() == orc.finalize().tolist()


def test_generate_beam_limits(dev):
    from atlas_b200._lib import AtlasB200Error

    model, _ = _tiny_fid(dev, torch.bfloat16)
    model.encoder.config.n_context, model.encoder.config.bsz = N_CTX, 2
    ids, mask = _passages(2, N_CTX, L_TOK, LENS, model_synth.T5_CFG["vocab_size"], seed=1)
    for kw in (dict(num_beams=17), dict(num_beams=4, num_return_sequences=2), dict(num_beams=4, early_stopping=True),
               dict(num_beams=4, do_sample=True), dict(num_beams=4, num_beam_groups=2)):
        with pytest.raises(AtlasB200Error):
            model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), max_length=5, **kw)


def test_greedy_min_length_none(dev):
    """min_length=None (the reference's --generation_min_length default) means no EOS ban, on the greedy path too."""
    model, _ = _tiny_fid(dev, torch.bfloat16)
    model.fuse_norm = False                       # bit-reproducible encoder (no fp32-atomic row statistics)
    model.encoder.config.n_context, model.encoder.config.bsz = N_CTX, 2
    ids, mask = _passages(2, N_CTX, L_TOK, LENS, model_synth.T5_CFG["vocab_size"], seed=1)
    with torch.no_grad():
        a = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), max_length=6, min_length=None)
        b = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), max_length=6, min_length=0)
    assert a.shape[0] == 2 and torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------------------
# 4. the Atlas surface and FiD-base size
# ------------------------------------------------------------------------------------------------------------------------
def test_atlas_generate_with_beams(dev):
    """Atlas.generate with --generation_num_beams 4 and --generation_min_length None (its default) returns sequences the
    evaluate loop decodes."""
    from atlas_b200.atlas import Atlas
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    opt = atlas_synth.make_opt(generation_num_beams=4, generation_min_length=None)
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    reader, _ = _tiny_fid(dev, torch.float32)
    retriever = DualEncoderRetriever(opt, Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG)).to(dev)).eval()
    m = Atlas(opt, reader, retriever, reader_tok, retriever_tok).eval()
    passages = atlas_synth.make_corpus()
    query, _ = atlas_synth.make_batch()
    chosen = [[passages[(5 * b + j) % len(passages)] for j in range(atlas_synth.TOPK)] for b in range(len(query))]
    with torch.no_grad():
        reader_tokens, _ = m.tokenize_passages(query, chosen)
        out = m.generate(reader_tokens, query)
    assert out.dtype == torch.int64 and out.shape[0] == len(query) and out.shape[1] <= opt.generation_max_length
    assert (out[:, 0] == 0).all() and bool(((out >= 0) & (out < atlas_synth.READER_VOCAB)).all())
    preds = [reader_tok.decode(g.tolist(), skip_special_tokens=True) for g in out]
    assert len(preds) == len(query) and all(isinstance(p, str) for p in preds)


def test_generate_beams_base_size(dev):
    """FiD-base decoder (12 layers, 32 128 tokens), B = 2, nb = 4, 40 x 384 keys, 16 steps under the graph: finishes, every
    token in [0, V)."""
    model, _ = _tiny_fid(dev, torch.bfloat16, vocab_size=32128, num_layers=2, num_decoder_layers=12)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(2, 32000, (2, 40 * 384), generator=g).to(dev)
    mask = torch.ones(2, 40 * 384, dtype=torch.bool, device=dev)
    model.encoder.config.n_context, model.encoder.config.bsz = 40, 2
    with torch.no_grad():
        seq = model.generate(input_ids=ids, attention_mask=mask, max_length=17, min_length=17, num_beams=4)
    assert seq.shape == (2, 17)
    assert bool(((seq >= 0) & (seq < 32128)).all())
