"""GPU parity of the TRAINING step: loss.backward() through atlas_b200.fid.FiD / atlas_b200.retrievers.Contriever
(forward kernels + hand-written backward kernels, atlas_b200/grad_ops.py) against
  (a) the gradients of the UNMODIFIED reference modules (tests/golden/grads_tiny.npz, oracle/make_golden_grads.py):
      L2 norm and a random projection of every parameter's gradient, full tensors of the small parameters;
  (b) element by element, the autograd of the CPU restatement (oracle/grad_oracle.py), itself pinned to (a) on CPU.
Accuracy budget: the golden also holds the reference's own bf16-parameter run; it sits up to 0.8 % (norm) / ~3 % of the
norm (projection) from its fp32 run.  The kernels compute in 16 bits with fp32 accumulation, so the bars are 3 % on the
norm, 15 % of the norm on the projection (a random projection of an error vector e is ~ N(0, |e|): over the ~50
parameters of a model the largest |z| is ~2.5, so this corresponds to |e| / |g| ~ 6 %) and 8 % relative L2 per tensor
(bf16; half of each for fp16, which has 3 more mantissa bits)."""
import os

import numpy as np
import pytest
import torch

import grad_oracle
import model_synth
from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu

T5_KW = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "grads_tiny.npz"))


def _check_against_golden(which, golden, grads, tol_norm, tol_proj):
    names = [n[len(which) + 11:] for n in golden.files if n.startswith(f"{which}_fp32/norm/")]
    assert set(names) <= set(grads), sorted(set(names) - set(grads))
    top = max(float(golden[f"{which}_fp32/norm/{n}"]) for n in names)
    for n in names:
        g = grads[n].float().cpu().numpy()
        assert np.isfinite(g).all(), n
        ref_norm = float(golden[f"{which}_fp32/norm/{n}"])
        if ref_norm < 1e-6 * top:                      # mathematically zero (BERT key bias)
            assert np.linalg.norm(g) <= 2e-3 * top, (n, np.linalg.norm(g))
            continue
        assert abs(np.linalg.norm(g) - ref_norm) <= tol_norm * ref_norm, (n, np.linalg.norm(g), ref_norm)
        proj = float((g * grad_oracle.direction(n, g.shape)).sum())
        assert abs(proj - float(golden[f"{which}_fp32/proj/{n}"])) <= tol_proj * ref_norm, (n, proj)
        key = f"{which}_fp32/full/{n}"
        if key in golden.files:
            ref = golden[key]
            assert np.linalg.norm(g - ref) <= 2 * tol_norm * np.linalg.norm(ref) + 1e-6, n


def _check_against_oracle(grads, ref, tol):
    top = max(float(v.norm()) for v in ref.values())
    for n, r in ref.items():
        g = grads[n].float().cpu()
        if float(r.norm()) < 1e-6 * top:
            continue
        rel = float((g - r).norm() / r.norm())
        assert rel <= tol, (n, rel)


def _fid(dev, dtype):
    from atlas_b200.fid import FiD, T5ConfigLite

    model = FiD(T5ConfigLite(**T5_KW))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    model = model.to(dtype).to(dev).train()
    model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
    return model, sd


def _fid_step(model, dev):
    ids, mask, labels = model_synth.fid_inputs()
    model.zero_grad(set_to_none=True)
    out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), decoder_input_ids=model._shift_right(labels.to(dev)),
                labels=labels.to(dev), use_cache=False)
    out[0].backward()
    return out, {n: p.grad for n, p in model.named_parameters()}


@pytest.mark.parametrize("dtype,tol", [(torch.bfloat16, 1.0), (torch.float16, 0.5), (torch.float32, 1.0)])
def test_fid_gradients_match_reference(dev, golden, dtype, tol):
    """fp32 parameters: bf16 compute, gradients delivered in fp32 (master weights, src/model_io.py:94-98 without
    --precision bf16); 16-bit parameters: gradients in the parameters' dtype like the reference's bf16 training."""
    model, sd = _fid(dev, dtype)
    out, grads = _fid_step(model, dev)
    assert all(g is not None and g.dtype == dtype for g in grads.values())
    assert abs(float(out[0]) - float(golden["fid_fp32/loss"])) <= 5e-2
    _check_against_golden("fid", golden, grads, 3e-2 * tol, 0.15 * tol)
    ids, mask, labels = model_synth.fid_inputs()
    _, ref = grad_oracle.fid_grads(sd, model_synth.T5_CFG, ids, mask, labels, 3, model._shift_right)
    _check_against_oracle(grads, ref, 8e-2 * tol)
    # the eval / no-grad path is untouched by the training path and gives the same loss
    model.eval()
    with torch.no_grad():
        ev = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))
    assert abs(float(ev[0]) - float(out[0])) <= 2e-2


def test_fid_gradient_checkpointing_and_encoder_outputs(dev):
    model, _ = _fid(dev, torch.bfloat16)
    out, grads = _fid_step(model, dev)
    model.gradient_checkpointing_enable()
    out2, grads2 = _fid_step(model, dev)
    assert abs(float(out[0]) - float(out2[0])) <= 1e-3
    for n in grads:     # recomputation runs the same deterministic forward kernels; fp32 atomics may reorder sums
        assert float((grads[n].float() - grads2[n].float()).norm()) <= 2e-2 * float(grads[n].float().norm()) + 1e-6, n
    model.gradient_checkpointing_disable()
    # decoder-only step on given encoder states (`encoder_outputs=`, src/atlas.py:364-370): gradients reach the decoder
    ids, mask, labels = model_synth.fid_inputs()
    model.zero_grad(set_to_none=True)
    enc = out.encoder_last_hidden_state.detach()
    o3 = model(attention_mask=mask.to(dev), encoder_outputs=[enc], labels=labels.to(dev))
    o3[0].backward()
    assert abs(float(o3[0]) - float(out[0])) <= 1e-2
    assert model.lm_head.weight.grad is not None and model.encoder.block[0].layer[0].SelfAttention.q.weight.grad is None


@pytest.mark.parametrize("dtype,tol", [(torch.bfloat16, 1.0), (torch.float16, 0.5), (torch.float32, 1.0)])
def test_contriever_gradients_match_reference(dev, golden, dtype, tol):
    from atlas_b200.retrievers import BertConfigLite, Contriever

    model = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 101)
    model.load_state_dict(sd)
    model = model.to(dtype).to(dev).train()
    ids, mask = model_synth.contriever_inputs()
    emb = model(input_ids=ids.to(dev), attention_mask=mask.to(dev))
    assert emb.requires_grad and emb.dtype == dtype
    w = torch.from_numpy(grad_oracle.direction("emb", tuple(emb.shape))).to(dev)
    loss = (emb.float() * w).sum() / emb.shape[0]
    loss.backward()
    assert abs(float(loss) - float(golden["contriever_fp32/loss"])) <= 0.15 * tol + 2e-2
    grads = {n: p.grad for n, p in model.named_parameters()}
    _check_against_golden("contriever", golden, grads, 3e-2 * tol, 0.15 * tol)
    _, ref = grad_oracle.contriever_grads(sd, model_synth.CONTRIEVER_CFG, ids, mask)
    _check_against_oracle(grads, ref, 8e-2 * tol)
    # frozen passage tower (query_side_retriever_training, src/retrievers.py:124-133): no graph, fast path
    with torch.no_grad():
        e2 = model(input_ids=ids.to(dev), attention_mask=mask.to(dev))
    assert not e2.requires_grad
    assert float((e2.float() - emb.detach().float()).abs().max()) <= 5e-2


def test_training_step_reduces_loss(dev):
    """A few SGD steps on one batch through the kernels' gradients drive the reader loss down (end-to-end sanity
    of sign and scale, fp32 master weights)."""
    model, _ = _fid(dev, torch.float32)
    ids, mask, labels = model_synth.fid_inputs()
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    losses = []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))
        out[0].backward()
        opt.step()
        losses.append(float(out[0]))
    assert losses[-1] < losses[0] - 0.3, losses


def test_atlas_training_step_matches_reference(dev):
    """One train.py step: `reader_loss, retriever_loss = model(...)`, `(reader_loss + retriever_loss).backward()`
    (src/atlas.py:399-550, train.py:90-101) on the reference's batch (oracle/make_golden_atlas_train.py): losses and the
    gradients of every reader and retriever parameter.  The retriever's gradient passes through the KL between the
    softmaxes of gold (reader perplexity) and retriever scores at temperature 0.1: the reference's own bf16-reader run
    moves those gradients by 2-3 % in norm and up to 0.3 norms in projection (stored in the golden), hence the wider bars
    for the retriever."""
    import atlas_synth
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    G = np.load(os.path.join(GOLDEN_DIR, "atlas_train_tiny.npz"))
    ret_ids = np.load(os.path.join(GOLDEN_DIR, "atlas_tiny.npz"))["ret_ids"]
    opt = atlas_synth.make_opt(temperature_gold=0.1, temperature_score=0.1)
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    reader = FiD(T5ConfigLite(**T5_KW))
    sd, _ = model_synth.fill_state_dict(reader.state_dict(), seed=202)
    reader.load_state_dict(sd)
    contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    sd, _ = model_synth.fill_state_dict(contriever.state_dict(), seed=101)
    contriever.load_state_dict(sd)
    retriever = DualEncoderRetriever(opt, contriever.to(dev))
    model = Atlas(opt, reader.to(dev), retriever, reader_tok, retriever_tok).eval()   # eval: no dropout, grads enabled
    corpus = atlas_synth.make_corpus()
    passages = [[corpus[int(i)] for i in row] for row in ret_ids]
    query, target = atlas_synth.make_batch()
    model.retrieve = lambda *a, **k: (passages, None)
    stats = {}
    reader_loss, retriever_loss = model(None, query, target, train_retriever=True, iter_stats=stats)
    assert reader_loss.requires_grad and retriever_loss.requires_grad
    (reader_loss + retriever_loss).backward()
    assert abs(float(reader_loss) - float(G["fp32/reader_loss"])) <= 6e-2
    assert abs(float(retriever_loss) - float(G["fp32/retriever_loss"])) <= 0.25 * float(G["fp32/retriever_loss"]) + 0.02
    names = [k[10:] for k in G.files if k.startswith("fp32/norm/")]
    mods = {"reader": reader, "retriever": retriever}
    top = {m: max(float(G[f"fp32/norm/{n}"]) for n in names if n.startswith(m)) for m in mods}
    checked = 0
    for n in names:
        m, pname = n.split(".", 1)
        p = dict(mods[m].named_parameters())[pname]
        assert p.grad is not None, n
        g = p.grad.float().cpu().numpy()
        assert np.isfinite(g).all(), n
        ref_norm = float(G[f"fp32/norm/{n}"])
        if ref_norm < 1e-5 * top[m]:
            continue
        tol_norm, tol_proj = (3e-2, 0.15) if m == "reader" else (0.15, 0.9)
        assert abs(np.linalg.norm(g) - ref_norm) <= tol_norm * ref_norm, (n, np.linalg.norm(g), ref_norm)
        proj = float((g * grad_oracle.direction(pname, g.shape)).sum())
        assert abs(proj - float(G[f"fp32/proj/{n}"])) <= tol_proj * ref_norm, (n, proj, float(G[f"fp32/proj/{n}"]))
        checked += 1
    assert checked >= 80


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_crossattention_score_capture_matches_reference(dev, dtype):
    """`overwrite_forward_crossattention` + `get_crossattention_scores` (src/fid.py:126-235,333-343): the recorded
    head-mean maps of every decoder layer (csrc/xattn_stats.cu) and all 24 aggregates against the reference's fp32 run
    (tests/golden/xattn_tiny.npz); budget = 3 x the reference's own bf16 drift of each aggregate, floor 2 %."""
    from atlas_b200.fid import FiD, T5ConfigLite

    G = np.load(os.path.join(GOLDEN_DIR, "xattn_tiny.npz"))
    model = FiD(T5ConfigLite(**T5_KW))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    model = model.to(dtype).to(dev).eval()
    model.overwrite_forward_crossattention()
    model.create_crossattention_storage()
    model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
    ids, mask, labels, mask_query = model_synth.fid_inputs_with_sep()
    with torch.no_grad():
        model(input_ids=ids.to(dev), attention_mask=mask.to(dev), decoder_input_ids=model._shift_right(labels.to(dev)),
              labels=labels.to(dev), use_cache=False)
        agg = model.get_crossattention_scores(3, mask.to(dev), labels=labels.to(dev), ids=ids.to(dev), mode="all",
                                              mask_query=mask_query.to(dev))
    assert len(model._xattn) == 2
    live = mask[:, None, :].expand(-1, labels.shape[1], -1).numpy()
    for li in range(2):
        for idx, name in ((0, "scores"), (1, "probs"), (2, "norms")):
            got = model._xattn[li][idx].float().cpu().numpy()
            ref = G[f"fp32/layer{li}/{name}"]
            scale = np.abs(ref[live]).max()
            assert np.abs(got - ref)[live].max() <= (6e-2 if dtype == torch.bfloat16 else 1e-2) * scale, (li, name)
            if name != "scores":     # masked keys carry no probability
                assert np.abs(got[~live]).max() <= 1e-6
    for k in [k[9:] for k in G.files if k.startswith("fp32/agg/")]:
        ref, ref16 = G[f"fp32/agg/{k}"], G[f"bf16/agg/{k}"]
        budget = max(3.0 * np.abs(ref16 - ref).max(), 2e-2 * np.abs(ref).max()) + 1e-6
        assert np.abs(agg[k].float().cpu().numpy() - ref).max() <= budget, k
    model.reset_score_storage()
    assert model._xattn == []


def test_atlas_step_with_crossattention_gold_scores(dev):
    """gold_score_mode `stdnormsum` (scores recorded during the training forward) and `evalnormsum` (a separate no-grad
    pass, `Atlas.eval_score` src/atlas.py:310-340) drive the retriever loss; compute_crossattention_stats fills corr/*."""
    import atlas_synth
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    ret_ids = np.load(os.path.join(GOLDEN_DIR, "atlas_tiny.npz"))["ret_ids"]
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    corpus = atlas_synth.make_corpus()
    passages = [[corpus[int(i)] for i in row] for row in ret_ids]
    query, target = atlas_synth.make_batch()
    for mode in ("stdnormsum", "evalnormsum"):
        opt = atlas_synth.make_opt(gold_score_mode=mode, temperature_gold=0.1, temperature_score=0.1,
                                   compute_crossattention_stats=(mode == "stdnormsum"))
        reader = FiD(T5ConfigLite(**T5_KW))
        sd, _ = model_synth.fill_state_dict(reader.state_dict(), seed=202)
        reader.load_state_dict(sd)
        reader.overwrite_forward_crossattention()          # what src/model_io.py:79-81 does for these modes
        reader.create_crossattention_storage()
        contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
        sd, _ = model_synth.fill_state_dict(contriever.state_dict(), seed=101)
        contriever.load_state_dict(sd)
        model = Atlas(opt, reader.to(dev), DualEncoderRetriever(opt, contriever.to(dev)), reader_tok, retriever_tok).eval()
        model.retrieve = lambda *a, **k: (passages, None)
        stats = {}
        reader_loss, retriever_loss = model(None, query, target, train_retriever=True, iter_stats=stats)
        assert torch.isfinite(reader_loss) and torch.isfinite(retriever_loss) and retriever_loss.requires_grad
        (reader_loss + retriever_loss).backward()
        assert contriever.encoder.layer[0].attention.self.query.weight.grad is not None
        if mode == "stdnormsum":
            assert any(k.startswith("corr/") for k in stats)
