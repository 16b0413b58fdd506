"""T5 v1.0 readers on the GPU: the ReLU epilogue of the wgmma linear layer (EPI_RELU, both schedules) and the ReLU
backward kernel, then a tied ReLU FiD against the unmodified reference (tests/golden/fid_relu_tiny.npz,
oracle/make_golden_t5v10.py) at t5-base and t5-small widths: forward logits / loss in every execution variant, gradients
(including `shared.weight`, which carries the embedding and the LM-head gradient), greedy and beam generation, and one
Atlas training step.  Bars as in test_gemm_pingpong_gpu.py, test_models_gpu.py and test_train_gpu.py."""
import math
import os

import numpy as np
import pytest
import torch

import beam_oracle as bo
import grad_oracle
import model_synth
from conftest import GOLDEN_DIR
from test_beam_search_gpu import EOS, L_TOK, LENS, MODE, N_CTX, PAD, _drive_oracle, _passages, _recorded_generate

pytestmark = pytest.mark.gpu

GEOMETRIES = {"base": dict(d_ff=3072), "small": dict(d_model=512, num_heads=8, d_ff=2048)}
DTYPES = [(torch.float16, "fp16"), (torch.bfloat16, "bf16")]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "fid_relu_tiny.npz"))


def _ref_logits16(golden, geom, key):
    """The reference's own 16-bit logits, stored as their 16-bit patterns."""
    dt = torch.float16 if key == "fp16" else torch.bfloat16
    return torch.from_numpy(golden[f"{geom}/logits_{key}_bits"]).view(dt).float().numpy()


# ------------------------------------------------------------------------------------------------------------------------
# 1. the GEMM epilogue
# ------------------------------------------------------------------------------------------------------------------------
def _close(got, ref, dtype):
    ref16 = ref.to(dtype).float()
    ulp = (torch.finfo(dtype).eps * ref16.abs()).clamp_min(torch.finfo(dtype).tiny * 1024)
    err = (got.float() - ref).abs()
    return bool((err <= 1.0 * ulp + 1e-3 * ref.abs() + 3e-5).all()), float(err.max())


def _inputs(dtype, dev, M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(M, K, generator=g) * 0.5).to(dtype).to(dev)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dtype).to(dev)
    bias = (torch.randn(N, generator=g) * 0.1).to(dtype).to(dev)
    return x, w, bias


def _ref(x, w, bias=None, scale=None):
    acc = x.float() @ w.float().T
    if scale is not None:
        acc = acc * scale[:, None]
    if bias is not None:
        acc = acc + bias.float()
    return torch.relu(acc)


def _shapes():
    """(M, N, K) that select the cooperative 128 x 128, the cooperative 128 x 256 and the ping-pong schedule (gemm.cu picks
    ping-pong from 2 x #SMs 128 x 128 tiles, 128 x 256 tiles once they fill the SMs)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m_wide = int(0.6 * sms)                      # N = 384: 2 m >= #SMs wide tiles, 3 m < 2 x #SMs narrow ones
    return {"coop128": (256 - 3, 1024, 768), "coop256": (128 * m_wide - 5, 384, 768), "pingpong": (20000, 3072, 768)}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("sched", ["coop128", "coop256", "pingpong"])
def test_relu_epilogue_matches_fp32_reference(dev, dtype, sched):
    from atlas_b200 import ops

    M, N, K = _shapes()[sched]
    x, w, bias = _inputs(dtype, dev, M, N, K, M + N)
    y = ops.linear(x, w, epilogue=ops.EPI_RELU)
    ok, err = _close(y, _ref(x, w), dtype)
    assert ok, f"max abs err {err}"
    assert float((y.float() < 0).sum()) == 0 and 0.3 < float((y == 0).float().mean()) < 0.7
    yb = ops.linear(x, w, bias, epilogue=ops.EPI_RELU)
    ok, err = _close(yb, _ref(x, w, bias), dtype)
    assert ok, f"max abs err {err} (bias)"
    # fused RMSNorm: rows scaled by rsqrt(ss / K + eps) before the ReLU
    ss = (x.float().pow(2).sum(-1) * 1.7).contiguous()
    eps = 1e-6
    ys = ops.linear(x, w, epilogue=ops.EPI_RELU, row_ss=ss, rs_eps=eps)
    ok, err = _close(ys, _ref(x, w, scale=torch.rsqrt(ss / K + eps)), dtype)
    assert ok, f"max abs err {err} (row_ss)"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("sched", ["coop128", "pingpong"])
def test_relu_epilogue_device_row_count(dev, dtype, sched):
    """Only the 128-row blocks below the device-side row count are computed; later rows keep their sentinel."""
    from atlas_b200 import ops

    M, N, K = _shapes()[sched]
    rows = M - 77 if sched == "pingpong" else 130
    x, w, _ = _inputs(dtype, dev, M, N, K, rows)
    out = torch.full((M, N), 7.0, dtype=dtype, device=dev)
    cnt = torch.tensor([rows], dtype=torch.int32, device=dev)
    ss = x.float().pow(2).sum(-1).contiguous()
    ops.linear(x, w, epilogue=ops.EPI_RELU, out=out, rows=cnt, row_ss=ss, rs_eps=1e-6)
    ok, err = _close(out[:rows], _ref(x[:rows], w, scale=torch.rsqrt(ss[:rows] / K + 1e-6)), dtype)
    assert ok, f"max abs err {err}"
    done = (rows + 127) // 128 * 128
    assert bool((out[done:] == 7.0).all())


@pytest.mark.parametrize("sched", ["coop128", "pingpong"])
def test_relu_epilogue_strided_output_view(dev, sched):
    """out[:, 768:768+N'] of a wider zero tensor with a ragged N': the TMA-clipped / guarded edges leave the columns
    outside the view and the rows after it untouched."""
    from atlas_b200 import ops

    M, _, K = _shapes()[sched]
    N = 712
    x, w, bias = _inputs(torch.float16, dev, M, N, K, 31)
    block = torch.zeros(2 * M + 64, 2304, dtype=torch.float16, device=dev)
    out, after = block[:M], block[M:]
    view = out[:, 768:768 + N]
    y = ops.linear(x, w, bias, epilogue=ops.EPI_RELU, out=view)
    assert y.data_ptr() == view.data_ptr()
    ok, err = _close(view, _ref(x, w, bias), torch.float16)
    assert ok, f"max abs err {err}"
    assert int(torch.count_nonzero(out[:, :768])) == 0 and int(torch.count_nonzero(out[:, 768 + N:])) == 0
    assert int(torch.count_nonzero(after)) == 0


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_relu_epilogue_pingpong_equals_cooperative(dev, dtype):
    """linear(x)[:256] (ping-pong) equals linear(x[:256]) (cooperative) bit for bit, with and without the fused norm."""
    from atlas_b200 import ops

    M, N, K = 20000, 3072, 2048
    x, w, bias = _inputs(dtype, dev, M, N, K, 77)
    assert torch.equal(ops.linear(x, w, bias, epilogue=ops.EPI_RELU)[:256],
                       ops.linear(x[:256], w, bias, epilogue=ops.EPI_RELU))
    ss = x.float().pow(2).sum(-1).contiguous()
    y = ops.linear(x, w, epilogue=ops.EPI_RELU, row_ss=ss, rs_eps=1e-6)
    assert torch.equal(y[:256], ops.linear(x[:256], w, epilogue=ops.EPI_RELU, row_ss=ss[:256].clone(), rs_eps=1e-6))


# ------------------------------------------------------------------------------------------------------------------------
# 2. the ReLU backward
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_relu_backward_bit_exact(dev, dtype):
    from atlas_b200 import grad_ops, ops

    gen = torch.Generator(device="cpu").manual_seed(3)
    u = torch.randn(1000, 3072, generator=gen).to(dtype)
    u[:, ::7] = 0.0
    u[::5, 1::11] = -0.0
    u, dg = u.to(dev), torch.randn(1000, 3072, generator=gen).to(dtype).to(dev)
    g = torch.relu(u)
    du = ops.relu_bwd(g, dg)
    assert torch.equal(du, dg * (g > 0))
    want = torch.where(g > 0, dg, torch.zeros_like(dg))
    assert torch.equal(du.view(torch.int16), want.view(torch.int16))
    # the autograd Function saves the output and masks with it
    x = u.clone().requires_grad_(True)
    y = grad_ops.relu(x)
    assert torch.equal(y, g)
    y.backward(dg)
    assert torch.equal(x.grad.view(torch.int16), want.view(torch.int16))
    # fused: relu(x W^T) with the ReLU in the GEMM epilogue, dx / dW from the masked gradient
    xs = (torch.randn(300, 768, generator=gen) * 0.5).to(dtype).to(dev).requires_grad_(True)
    w = (torch.randn(3072, 768, generator=gen) / math.sqrt(768)).to(dtype).to(dev).requires_grad_(True)
    out = grad_ops.linear_relu(xs, w)
    dout = torch.randn(300, 3072, generator=gen).to(dtype).to(dev)
    out.backward(dout)
    du = torch.where(out > 0, dout, torch.zeros_like(dout)).float()
    ref_dx, ref_dw = du @ w.detach().float(), du.T @ xs.detach().float()
    assert float((xs.grad.float() - ref_dx).norm() / ref_dx.norm()) < 1e-2
    assert float((w.grad.float() - ref_dw).norm() / ref_dw.norm()) < 1e-2


# ------------------------------------------------------------------------------------------------------------------------
# 3. - 6. the tied ReLU reader
# ------------------------------------------------------------------------------------------------------------------------
def _reader(geom, dtype=None, dev=None):
    from atlas_b200.fid import FiD, T5ConfigLite

    kw = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    kw.update(GEOMETRIES[geom], feed_forward_proj="relu", tie_word_embeddings=True)
    model = FiD(T5ConfigLite(**kw))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    sd["lm_head.weight"] = sd["shared.weight"].clone()             # one tied table, as in the golden
    model.load_state_dict(sd)
    assert model.lm_head.weight is model.shared.weight
    if dtype is not None:
        model = model.to(dtype).to(dev)
    return model


def _forward(model, dev, ids, mask, labels):
    with torch.no_grad():
        out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), decoder_input_ids=model._shift_right(labels.to(dev)),
                    labels=labels.to(dev), use_cache=False)
    return out


@pytest.mark.parametrize("geom", list(GEOMETRIES))
@pytest.mark.parametrize("dtype,key", DTYPES)
def test_fid_relu_matches_reference(dev, golden, geom, dtype, key, monkeypatch):
    """Logits / loss / encoder states against the reference (bars of test_models_gpu.test_fid_matches_reference) with the
    fused norm and CUDA graphs on and off; on inputs with dead 64-key tiles the packed encoder agrees with the padded one."""
    from atlas_b200 import ops

    model = _reader(geom, dtype, dev).eval()
    ids, mask, labels = model_synth.fid_inputs()
    model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
    ref32 = golden[f"{geom}/logits_fp32"]
    ref16_err = np.abs(_ref_logits16(golden, geom, key) - ref32).max()
    results = []
    for fuse in (True, False):
        for graphs in (True, False):
            model.fuse_norm, model.cuda_graphs = fuse, graphs
            out = _forward(model, dev, ids, mask, labels)
            logits = out[1].float().cpu().numpy()
            err = np.abs(logits - ref32).max()
            assert err <= 3.0 * ref16_err + 2e-4, (fuse, graphs, err, ref16_err)
            if dtype == torch.float16:
                assert err <= max(1e-3 * max(1.0, float(np.abs(ref32).max())), 1.5 * ref16_err), (fuse, graphs, err)
            assert abs(float(out[0]) - float(golden[f"{geom}/loss_fp32"])) <= 2e-2
            enc_ref = golden[f"{geom}/enc_fp32"].astype(np.float32)      # the first passage of the first query
            enc_err = np.abs(out.encoder_last_hidden_state[0, :64].float().cpu().numpy() - enc_ref).max()
            top = float(2.0 ** np.ceil(np.log2(np.abs(enc_ref).max())))
            assert enc_err <= 4.0 * top * (2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11) + 4e-3, enc_err
            results.append(logits)
    for r in results[1:]:
        assert np.abs(r - results[0]).max() <= 3.0 * ref16_err + 2e-4
    # padding-compacted encoder on and off: 2 passages of 128 tokens per query, several dead 64-key tiles
    model.fuse_norm, model.cuda_graphs = True, True
    model.encoder.config.n_context = N_CTX
    ids2, mask2 = _passages(2, N_CTX, L_TOK, LENS, 512, seed=4)
    lab2 = labels
    by_packed = {}
    for packed in (True, False):
        monkeypatch.setattr(ops, "_ENC_PACKED", packed)
        by_packed[packed] = _forward(model, dev, ids2, mask2, lab2)[1].float().cpu().numpy()
    assert np.abs(by_packed[True] - by_packed[False]).max() <= 3.0 * ref16_err + 2e-4


@pytest.mark.parametrize("geom", list(GEOMETRIES))
@pytest.mark.parametrize("dtype,tol", [(torch.bfloat16, 1.0), (torch.float16, 0.5), (torch.float32, 1.0)])
def test_fid_relu_gradients_match_reference(dev, golden, geom, dtype, tol):
    """Bars of test_train_gpu.py: 3 % on the norm, 15 % of the norm on the projection, 8 % relative L2 per small tensor
    (bf16; half of each for fp16), the last widened to 1.5x the reference's own bf16 error on that tensor where that is
    larger (the ReLU mask flips with 16-bit rounding: ~9 % on the feed-forward norm weights of the base geometry).  fp32
    parameters: bf16 compute, fp32 gradients."""
    model = _reader(geom, dtype, dev).train()
    model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
    ids, mask, labels = model_synth.fid_inputs()
    out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))
    out[0].backward()
    assert abs(float(out[0]) - float(golden[f"{geom}/grad_fp32/loss"])) <= 5e-2
    grads = {n: p.grad for n, p in model.named_parameters()}
    assert "lm_head.weight" not in grads and all(g is not None and g.dtype == dtype for g in grads.values())
    pre = f"{geom}/grad_fp32/"
    names = [k[len(pre) + 5:] for k in golden.files if k.startswith(pre + "norm/")]
    assert set(names) == set(grads), sorted(set(names) ^ set(grads))
    for n in names:
        g = grads[n].float().cpu().numpy()
        assert np.isfinite(g).all(), n
        ref_norm = float(golden[pre + "norm/" + n])
        assert abs(np.linalg.norm(g) - ref_norm) <= 3e-2 * tol * ref_norm, (n, np.linalg.norm(g), ref_norm)
        proj = float((g * grad_oracle.direction(n, g.shape)).sum())
        assert abs(proj - float(golden[pre + "proj/" + n])) <= 0.15 * tol * ref_norm, (n, proj)
        if pre + "full/" + n in golden.files:
            ref = golden[pre + "full/" + n]
            ref16_err = float(golden[f"{geom}/grad_bf16/relerr/{n}"])
            err = np.linalg.norm(g - ref) / np.linalg.norm(ref)
            assert err <= tol * max(8e-2, 1.5 * ref16_err), (n, err, ref16_err)


def test_fid_relu_gradient_checkpointing(dev):
    model = _reader("base", torch.bfloat16, dev).train()
    model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
    ids, mask, labels = model_synth.fid_inputs()
    runs = []
    for ckpt in (False, True):
        if ckpt:
            model.gradient_checkpointing_enable()
        model.zero_grad(set_to_none=True)
        out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))
        out[0].backward()
        runs.append((float(out[0]), {n: p.grad.float().clone() for n, p in model.named_parameters()}))
    model.gradient_checkpointing_disable()
    assert abs(runs[0][0] - runs[1][0]) <= 1e-3
    for n, g in runs[0][1].items():
        assert float((g - runs[1][1][n]).norm()) <= 2e-2 * float(g.norm()) + 1e-6, n


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_fid_relu_generate_greedy_cached_matches_prefix_rerun(dev, dtype):
    """The KV-cached decode step (the unfused feed-forward of the decode kernels) against the path that re-runs the decoder
    prefix: identical tokens wherever the teacher-forced top-2 gap exceeds the 16-bit noise (test_round2_gpu's rule)."""
    model = _reader("base", dtype, dev).eval()
    ids, mask, _ = model_synth.fid_inputs()
    model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
    with torch.no_grad():
        a = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), max_length=9, min_length=3)
        b = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), max_length=9, min_length=3, use_cache=False)
        tf = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), decoder_input_ids=b[:, :-1], use_cache=False).logits.float()
    top2 = tf.topk(2, dim=-1)[0]
    gap_ok = (top2[..., 0] - top2[..., 1]) > (0.02 if dtype == torch.bfloat16 else 0.005)
    n = min(a.shape[1], b.shape[1])
    compared = 0
    for bi in range(2):
        for t in range(1, n):
            if not bool(gap_ok[bi, t - 1]):
                break
            assert int(a[bi, t]) == int(b[bi, t]), (bi, t, a[bi].tolist(), b[bi].tolist())
            compared += 1
    assert compared >= 2


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fid_relu_generate_beams_match_oracle(dev, dtype):
    """num_beams=4: every selection equals oracle/beam_oracle.py's on the same step logits (exempt only below a 2-ulp
    margin) and the output equals the oracle's finalize; the graph-replayed generation equals the eager one."""
    model = _reader("small", dtype, dev).eval()
    model.fuse_norm = False
    nb, B, max_length, min_length, lp = 4, 2, 10, 3, 1.0
    model.encoder.config.n_context, model.encoder.config.bsz = N_CTX, B
    ids, mask = _passages(B, N_CTX, L_TOK, LENS, 512, seed=14)
    kw = dict(max_length=max_length, min_length=min_length, num_beams=nb, length_penalty=lp)
    model.cuda_graphs = False
    with torch.no_grad():
        seq, logits_of, sel, _ = _recorded_generate(model, ids.to(dev), mask.to(dev), **kw)
    orc = bo.BeamSearch(B, nb, model.config.vocab_size, max_length, min_length, lp, mode=MODE[dtype], eos=EOS, pad=PAD)
    exempt = _drive_oracle(orc, logits_of, sel, MODE[dtype])
    if not exempt:
        assert seq.cpu().numpy().tolist() == orc.finalize().tolist()
    model.cuda_graphs = True
    with torch.no_grad():
        g1 = model.generate(input_ids=ids.to(dev), attention_mask=mask.to(dev), **kw)
    assert torch.equal(g1, seq)


def test_atlas_step_with_tied_relu_reader(dev):
    """One `Atlas.forward(..., train_retriever=True)` step with a tied ReLU reader: finite losses, and backward() fills the
    gradient of the tied table and of every feed-forward matrix."""
    import atlas_synth
    from atlas_b200.atlas import Atlas
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    ret_ids = np.load(os.path.join(GOLDEN_DIR, "atlas_tiny.npz"))["ret_ids"]
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    corpus = atlas_synth.make_corpus()
    passages = [[corpus[int(i)] for i in row] for row in ret_ids]
    query, target = atlas_synth.make_batch()
    for mode in ("ppmean", "evalnormsum"):
        opt = atlas_synth.make_opt(gold_score_mode=mode, temperature_gold=0.1, temperature_score=0.1)
        reader = _reader("base")
        if mode == "evalnormsum":
            reader.overwrite_forward_crossattention()
            reader.create_crossattention_storage()
        contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
        sd, _ = model_synth.fill_state_dict(contriever.state_dict(), seed=101)
        contriever.load_state_dict(sd)
        model = Atlas(opt, reader.to(dev), DualEncoderRetriever(opt, contriever.to(dev)), reader_tok, retriever_tok).eval()
        model.retrieve = lambda *a, **k: (passages, None)
        reader_loss, retriever_loss = model(None, query, target, train_retriever=True, iter_stats={})
        assert torch.isfinite(reader_loss) and torch.isfinite(retriever_loss) and retriever_loss.requires_grad
        (reader_loss + retriever_loss).backward()
        assert reader.shared.weight.grad is not None and bool(torch.isfinite(reader.shared.weight.grad).all())
        ff = [m for n, m in reader.named_modules() if n.endswith("DenseReluDense")]
        assert len(ff) == 4
        for m in ff:
            for lin in (m.wi, m.wo):
                assert lin.weight.grad is not None and float(lin.weight.grad.norm()) > 0, mode
        assert contriever.encoder.layer[0].attention.self.query.weight.grad is not None
