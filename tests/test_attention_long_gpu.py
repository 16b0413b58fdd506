"""The K / V-streaming attention forward (`ops.attention_long`, attention_long_kernel of csrc/attention.cu) and the FiD reader
on passages longer than the 576 keys of the resident kernel.

Part A: the kernel against the float64 forward of oracle/attention_fwd_oracle.py, element by element within its bounds (the
        helpers and conventions of test_attention_fwd_gpu.py: NaN-filled input buffers, a strided output slice whose
        neighbouring columns must keep their NaN bits, block_live off and on bit-identical).  The oracle's C32 term was
        derived for at most 16 key blocks per CTA; at 64 blocks its worst-case fp32 chains (row sum, rescales, MMA
        accumulation) are 4x longer, which stays two orders of magnitude below the 16-bit rounding terms of the bound.
Part B: dropout on the probabilities, and `ops.attention_bwd` fed this forward's output and log-sum-exp, against
        oracle/attention_bwd_oracle.py.
Part C: the argument checks.
Part D: a synthetic FiD (oracle/model_synth) at text_maxlength 640 and 1024 against oracle/fid_cpu.py, its gradients against
        oracle/grad_oracle.py, generation, one Atlas training step, and the 4096-token limit."""
import os

import numpy as np
import pytest
import torch

import attention_bwd_oracle as abo
import attention_fwd_oracle as afo
import fid_cpu
import grad_oracle
import model_synth
from conftest import GOLDEN_DIR
from test_attention_fwd_gpu import _assert_sentinels, _assert_within, _bias, _inv_keep, _nan_filled, _qkv

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _holey_mask(B, L, seed):
    """Segment 0 full length; the others padded past a length in 40..100 % of L, with 10 % random holes among the live
    keys; segment 1 also has two wholly masked 64-key blocks inside its live range; the last segment has no live key at
    all (it keeps every block live, uniform-ish over the masked keys as in the reference's softmax)."""
    g = torch.Generator().manual_seed(seed)
    j = torch.arange(L)
    rows = []
    for b in range(B):
        n = L if b == 0 else int(torch.randint(max(1, L * 2 // 5), L + 1, (1,), generator=g))
        live = j < n
        if b > 0:
            live &= torch.rand(L, generator=g) >= 0.1
        if b == 1:
            live &= ~((j >= 64) & (j < 192))
        if b == B - 1 and B > 2:
            live[:] = False
        elif not bool(live.any()):
            live[0] = True
        rows.append(torch.where(live, 0.0, -10000.0))
    return torch.stack(rows)


def _run_long(dev, dtype, B, H, Lq, Lk, mask, bias, scale, causal, seed, qmul, what, dropout=None):
    """attention_long from NaN-guarded buffers into a strided output, block_live off and on, against the fp64 oracle."""
    from atlas_b200 import ops

    HD = H * 64
    qbuf, kvbuf, k_col0, v_col0, Q, K, V = _qkv(B, H, Lq, Lk, dtype, seed, qmul, dev)
    maskd = mask.to(dev) if mask is not None else None
    biasd = bias.to(dev) if bias is not None else None
    keep, inv = None, 1.0
    if dropout is not None:
        keep = ops.attention_dropout_mask(B, H, Lq, Lk, dropout[0], dropout[1], dropout[2], dev)
        inv = _inv_keep(dropout[0])
    O64, lse64, bo, bl = afo.forward_bound(Q, K, V, maskd, biasd, scale, causal, keep, inv, dtype=dtype)
    live = ops.key_block_live(maskd)
    outs = []
    for blk in ((None, live) if live is not None else (None,)):
        obuf = _nan_filled((B * Lq, HD + 64), dtype, dev)
        out, lse = ops.attention_long(qbuf, 8, kvbuf, k_col0, kvbuf, v_col0, B, H, Lq, Lk, add_mask=maskd, bias_delta=biasd,
                                      scale=scale, causal_value=causal, out=obuf[:, 32:32 + HD], return_lse=True,
                                      dropout=dropout, block_live=blk)
        tag = f"{what} {str(dtype)[6:]} block_live={blk is not None}"
        _assert_sentinels(obuf, 32, 32 + HD, dtype, tag)
        _assert_within(out, O64.reshape(B * Lq, HD), bo.reshape(B * Lq, HD), f"{tag} O", "L", dtype)
        _assert_within(lse, lse64, bl, f"{tag} lse", "L-lse", dtype)
        outs.append((out.clone(), lse.clone()))
    if len(outs) == 2:
        assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16)), f"{what}: O differs with block_live"
        assert torch.equal(outs[0][1], outs[1][1]), f"{what}: lse differs with block_live"
    return outs[0], (qbuf, kvbuf, k_col0, v_col0, Q, K, V, maskd, biasd)


# ------------------------------------------------------------------------------------------------------------------------
# Part A. the kernel against fp64
# ------------------------------------------------------------------------------------------------------------------------
LONG_LK = [577, 640, 1000, 1024, 2048, 4096]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", LONG_LK)
def test_t5_encoder_long(dev, dtype, L):
    """T5 encoder self-attention: relative-position bias, no scaling, key masks with holes, dead 64-key blocks and a
    segment without any live key; 577 and 1000 leave a ragged last key block."""
    S, H = (3, 4) if L <= 1024 else (3, 2)
    _run_long(dev, dtype, S, H, L, L, _holey_mask(S, L, seed=L), _bias(H, L, L, L), 1.0, 0.0, seed=L + 1, qmul=0.35,
              what=f"t5 L{L}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [577, 1024, 4096])
def test_bert_style_long(dev, dtype, L):
    """Scale 1/8 without a bias table, with and without a key mask."""
    B, H = 2, 2
    _run_long(dev, dtype, B, H, L, L, None, None, 0.125, 0.0, seed=L + 2, qmul=1.0, what=f"bert nomask L{L}")
    _run_long(dev, dtype, B, H, L, L, _holey_mask(B, L, seed=L + 3), None, 0.125, 0.0, seed=L + 4, qmul=1.0,
              what=f"bert L{L}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Lq,Lk", [(100, 1000), (1300, 700), (4096, 4096), (300, 4096)])
def test_rectangular_and_causal_long(dev, dtype, Lq, Lk):
    """Lq != Lk with the bias table indexed j - i + Lq - 1 (the CTA's slice of it starts at its last query row), and the
    causal rule j > i on top; (4096, 4096) fills the 8191-entry table."""
    H = 2
    _run_long(dev, dtype, 2, H, Lq, Lk, _holey_mask(2, Lk, seed=Lq), _bias(H, Lq, Lk, Lq + Lk), 1.0, 0.0, seed=Lq + Lk,
              qmul=0.35, what=f"rect Lq{Lq} Lk{Lk}")
    _run_long(dev, dtype, 2, H, Lq, Lk, None, _bias(H, Lq, Lk, Lq - Lk), 1.0, -10000.0, seed=Lq * 7 + Lk, qmul=0.35,
              what=f"rect causal Lq{Lq} Lk{Lk}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [64, 200, 576])
def test_boundary_both_kernels_meet_the_bound(dev, dtype, L):
    """At Lk <= 576 both kernels take the input: on the same inputs each meets the same fp64 bound, and since both run the
    same per-block functions on the same blocks in the same order, their O and lse are bit-identical, with dropout too."""
    from atlas_b200 import ops

    S, H = 3, 4
    mask, bias = _holey_mask(S, L, seed=L + 5), _bias(H, L, L, L + 5)
    for dropout in (None, (0.1, 4321, 64)):
        tag = f"boundary L{L} dropout={dropout is not None}"
        (o_long, lse_long), (qbuf, kvbuf, k_col0, v_col0, Q, K, V, maskd, biasd) = _run_long(
            dev, dtype, S, H, L, L, mask, bias, 1.0, 0.0, seed=L + 6, qmul=0.35, what=tag, dropout=dropout)
        out, lse = ops.attention(qbuf, 8, kvbuf, k_col0, kvbuf, v_col0, S, H, L, L, add_mask=maskd, bias_delta=biasd,
                                 scale=1.0, return_lse=True, dropout=dropout, block_live=ops.key_block_live(maskd))
        if dropout is None:
            O64, lse64, bo, bl = afo.forward_bound(Q, K, V, maskd, biasd, 1.0, 0.0, dtype=dtype)
            _assert_within(out, O64.reshape(S * L, H * 64), bo.reshape(S * L, H * 64), f"boundary resident L{L} O", "L", dtype)
            _assert_within(lse, lse64, bl, f"boundary resident L{L} lse", "L-lse", dtype)
        assert torch.equal(out.view(torch.int16), o_long.view(torch.int16)), f"{tag}: O differs between the kernels"
        assert torch.equal(lse, lse_long), f"{tag}: lse differs between the kernels"


# ------------------------------------------------------------------------------------------------------------------------
# Part B. dropout, and the backward fed this forward
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L,p_drop", [(1024, 0.1), (2048, 0.5)])
def test_dropout_long(dev, dtype, L, p_drop):
    """O against the fp64 forward with the keep mask `attention_dropout_mask` exports; the lse is that of the run without
    dropout."""
    S, H = 2, 2
    mask, bias = _holey_mask(S, L, seed=9), _bias(H, L, L, 9)
    (_, lse_d), _ = _run_long(dev, dtype, S, H, L, L, mask, bias, 1.0, 0.0, seed=21, qmul=0.35, what=f"dropout {p_drop} L{L}",
                              dropout=(p_drop, 4321, 64))
    (_, lse_0), _ = _run_long(dev, dtype, S, H, L, L, mask, bias, 1.0, 0.0, seed=21, qmul=0.35, what=f"no dropout L{L}")
    assert torch.equal(lse_d, lse_0), "dropout changed the log-sum-exp"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p_drop", [0.0, 0.1])
def test_backward_from_long_forward(dev, dtype, p_drop):
    """attention_bwd at L = 1024 on this forward's output and lse (its dropout key too): dQ, dK, dV and dbias within the
    bounds of oracle/attention_bwd_oracle.py evaluated on the same output."""
    from atlas_b200 import ops

    S, H, L = 2, 4, 1024
    mask, bias = _holey_mask(S, L, seed=31), _bias(H, L, L, 31)
    dkey = (p_drop, 777, 128) if p_drop else None
    (out, lse), (qbuf, kvbuf, k_col0, v_col0, Q, K, V, maskd, biasd) = _run_long(
        dev, dtype, S, H, L, L, mask, bias, 1.0, 0.0, seed=33, qmul=0.35, what=f"bwd-fwd p{p_drop}", dropout=dkey)
    keep, inv = None, 1.0
    if dkey is not None:
        keep = ops.attention_dropout_mask(S, H, L, L, p_drop, dkey[1], dkey[2], dev)
        inv = _inv_keep(p_drop)
    HD = H * 64
    g = torch.Generator().manual_seed(35)
    do16 = torch.randn(S * L, HD, generator=g).to(dtype).to(dev)
    ref = abo.attention_bwd(Q, K, V, out.double().view(S, L, H, 64), do16.double().view(S, L, H, 64), maskd, biasd, 1.0, 0.0,
                            keep, inv, dtype=dtype)
    dqkv = _nan_filled((S * L, 3 * HD), dtype, dev)
    dbias = ops.attention_bwd(qbuf, 8, kvbuf, k_col0, kvbuf, v_col0, out, do16, dqkv, 0, dqkv, HD, dqkv, 2 * HD, S, H, L, L,
                              add_mask=maskd, bias_delta=biasd, need_dbias=True, scale=1.0, lse=lse, dropout=dkey,
                              block_live=ops.key_block_live(maskd))
    tag = f"bwd L{L} p{p_drop} {str(dtype)[6:]}"
    assert bool(torch.isfinite(dqkv).all()), f"{tag}: non-finite gradient"
    for name, c0, n in (("dq", 0, L), ("dk", HD, L), ("dv", 2 * HD, L)):
        _assert_within(dqkv[:, c0:c0 + HD], ref[name].reshape(S * n, HD), ref[name + "_bound"].reshape(S * n, HD),
                       f"{tag} {name}", "L-bwd", dtype)
    _assert_within(dbias, ref["dbias"], ref["dbias_bound"], f"{tag} dbias", "L-bwd", dtype)


# ------------------------------------------------------------------------------------------------------------------------
# Part C. argument checks
# ------------------------------------------------------------------------------------------------------------------------
def test_attention_long_argument_checks(dev):
    """B = 0 is a no-op; every documented limit is an error before any launch and leaves the output untouched."""
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    H = 2
    buf = torch.zeros((8200, 3 * H * 64 + 8), dtype=torch.bfloat16, device=dev)
    out = ops.attention_long(buf, 0, buf, H * 64, buf, 2 * H * 64, 0, H, 1024, 1024,
                             out=torch.empty((0, H * 64), dtype=torch.bfloat16, device=dev))
    assert out.shape == (0, H * 64)
    cases = ((dict(Lq=64, Lk=4097), "Lk <= 4096"), (dict(Lq=4098, Lk=4096), "bias table"),
             (dict(Lq=8193, Lk=1), "bias table"), (dict(Lq=1024, Lk=1024, k_col0=H * 64 + 4), "multiples of 8"),
             (dict(Lq=1024, Lk=1024, ldq=3 * H * 64 + 4), "multiples of 8"))
    for kw, frag in cases:
        sentinel = torch.full((8200, H * 64), 3.0, dtype=torch.bfloat16, device=dev)
        q = torch.zeros((8200, kw["ldq"]), dtype=torch.bfloat16, device=dev) if "ldq" in kw else buf
        with pytest.raises(AtlasB200Error, match=frag):
            ops.attention_long(q, 0, buf, kw.get("k_col0", H * 64), buf, 2 * H * 64, 1, H, kw["Lq"], kw["Lk"], out=sentinel)
        torch.cuda.synchronize()
        assert bool((sentinel == 3.0).all()), frag


# ------------------------------------------------------------------------------------------------------------------------
# Part D. the FiD reader on long passages
# ------------------------------------------------------------------------------------------------------------------------
T5_KW = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}


def _reader(dtype, dev, **over):
    from atlas_b200.fid import FiD, T5ConfigLite

    model = FiD(T5ConfigLite(**dict(T5_KW, **over)))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    return model.to(dtype).to(dev), sd


def _long_inputs(B, n_ctx, L, T=8, seed=0):
    """Passages of 40..100 % of L tokens (one full), padded to L, and labels of up to T tokens."""
    ids, mask, labels = model_synth.fid_inputs(seed=seed + L, B=B, n_ctx=n_ctx, L=L, T=T)
    g = torch.Generator().manual_seed(seed + L)
    lens = torch.randint(L * 2 // 5, L + 1, (B, n_ctx), generator=g)
    lens[0, 0] = L
    m = torch.arange(L)[None, None, :] < lens[..., None]
    ids = (ids.view(B, n_ctx, L).clamp_min(2) * m).view(B, n_ctx * L)
    return ids, m.view(B, n_ctx * L), labels


def _logit_err(model, sd, dev, ids, mask, labels, n_ctx):
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, ids.shape[0]
    with torch.no_grad():
        out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), decoder_input_ids=model._shift_right(labels.to(dev)),
                    labels=labels.to(dev), use_cache=False)
    loss, ref, _ = fid_cpu.fid_forward({k: v.float() for k, v in sd.items()}, model_synth.T5_CFG, ids, mask,
                                       model._shift_right(labels), labels, n_context=n_ctx)
    return float((out[1].float().cpu() - ref).abs().max()), abs(float(out[0]) - float(loss)), float(ref.abs().max())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [640, 1024])
def test_fid_long_passages_match_cpu_oracle(dev, dtype, L):
    """Logits and loss against the fp32 restatement of the reference, with the fused norm and CUDA graphs on and off.  The
    bar is calibrated on the same model and inputs of the same size cut into 512-token passages (the resident kernel):
    the long passages may be at most 3x (+ 2e-4) as far from the oracle, and the loss within 2e-2."""
    model, sd = _reader(dtype, dev)
    model.eval()
    n_ctx = 2
    ids, mask, labels = _long_inputs(2, n_ctx, L)
    short_ctx = n_ctx * L // 512 if (n_ctx * L) % 512 == 0 else None
    cal_ids, cal_mask, _ = _long_inputs(2, 4, 512, seed=1) if short_ctx is None else (ids, mask, None)
    cal_err, _, _ = _logit_err(model, sd, dev, cal_ids, cal_mask, labels, short_ctx or 4)
    for fuse in (True, False):
        for graphs in (True, False):
            model.fuse_norm, model.cuda_graphs = fuse, graphs
            err, loss_err, top = _logit_err(model, sd, dev, ids, mask, labels, n_ctx)
            print(f"L{L} {str(dtype)[6:]} fuse={fuse} graphs={graphs}: max |logits - fp32| {err:.3g} "
                  f"(512-token passages: {cal_err:.3g}, max |logit| {top:.3g}), |loss - fp32| {loss_err:.3g}")
            assert err <= 3.0 * cal_err + 2e-4, (fuse, graphs, err, cal_err)
            assert loss_err <= 2e-2, (fuse, graphs, loss_err)


def _bias_table_errors(model, dev, sd, ids, mask, labels, n_ctx):
    """Relative L2 errors of the relative-position bias gradients of one backward against grad_oracle's."""
    _, ref = grad_oracle.fid_grads({k: v.float() for k, v in sd.items()}, model_synth.T5_CFG, ids, mask, labels, n_ctx,
                                   model._shift_right)
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, ids.shape[0]
    model.zero_grad(set_to_none=True)
    model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))[0].backward()
    return {n: float((p.grad.float().cpu() - ref[n]).norm() / ref[n].norm()) for n, p in model.named_parameters()
            if "relative_attention_bias" in n}


@pytest.mark.parametrize("dtype,tol", [(torch.bfloat16, 1.0), (torch.float16, 0.5)])
def test_fid_long_gradients_match_oracle(dev, dtype, tol):
    """A training step at text_maxlength 1024 (no dropout), with and without gradient checkpointing, against torch.autograd
    of oracle/fid_cpu.py: bars of test_train_gpu.py - 3 % on each gradient's norm and 15 % of the norm on its projection
    on a seeded direction (bf16; half of each for fp16), and 8 % relative L2 on the relative-position bias tables, which
    the attention backward produces from this forward's log-sum-exp, widened to 1.5x the error of the same tables when the
    same tokens run as 512-token passages on the resident kernel where that is larger.  The 8 % holds for fp16 too: its
    encoder table measured 4.5 % here against 2.5 % for 512-token passages, while the same backward at L = 1024 meets the
    per-element fp64 bounds of test_backward_from_long_forward."""
    n_ctx, L = 2, 1024
    ids, mask, labels = _long_inputs(1, n_ctx, L, seed=3)
    model, sd = _reader(dtype, dev)
    model.train()
    cal = _bias_table_errors(model, dev, sd, ids, mask, labels, n_ctx * L // 512)
    ref_loss, ref = grad_oracle.fid_grads({k: v.float() for k, v in sd.items()}, model_synth.T5_CFG, ids, mask, labels, n_ctx,
                                          model._shift_right)
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, 1
    names = [n for n, _ in model.named_parameters() if n in ref]
    assert len(names) >= 20 and any("relative_attention_bias" in n for n in names)
    for ckpt in (False, True):
        if ckpt:
            model.gradient_checkpointing_enable()
        model.zero_grad(set_to_none=True)
        out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))
        out[0].backward()
        assert abs(float(out[0]) - ref_loss) <= 5e-2, (ckpt, float(out[0]), ref_loss)
        for n, p in model.named_parameters():
            if n not in ref:
                continue
            g = p.grad.float().cpu()
            r = ref[n].float()
            assert bool(torch.isfinite(g).all()), n
            rn = float(r.norm())
            assert abs(float(g.norm()) - rn) <= 3e-2 * tol * rn, (ckpt, n, float(g.norm()), rn)
            d = torch.from_numpy(grad_oracle.direction(n, tuple(g.shape)))
            assert abs(float((g * d).sum()) - float((r * d).sum())) <= 0.15 * tol * rn, (ckpt, n)
            if n in cal:
                err = float((g - r).norm()) / rn
                print(f"{str(dtype)[6:]} ckpt={ckpt} {n}: relative L2 {err:.4f} (512-token passages: {cal[n]:.4f})")
                assert err <= max(8e-2, 1.5 * cal[n]), (ckpt, n, err, cal[n])
    model.gradient_checkpointing_disable()


def test_fid_long_checkpointing_rederives_dropout(dev):
    """With dropout on (text_maxlength 1024), the checkpointed backward recomputes each block under the same dropout keys:
    loss and gradients equal those of the run that keeps its activations."""
    n_ctx, L = 2, 1024
    ids, mask, labels = _long_inputs(1, n_ctx, L, seed=5)
    model, _ = _reader(torch.bfloat16, dev, dropout_rate=0.1)
    model.train()
    model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, 1
    runs = []
    for ckpt in (False, True):
        if ckpt:
            model.gradient_checkpointing_enable()
        model.zero_grad(set_to_none=True)
        torch.manual_seed(11)
        torch.cuda.manual_seed(11)
        out = model(input_ids=ids.to(dev), attention_mask=mask.to(dev), labels=labels.to(dev))
        out[0].backward()
        runs.append((float(out[0]), {n: p.grad.float().clone() for n, p in model.named_parameters()}))
    model.gradient_checkpointing_disable()
    assert abs(runs[0][0] - runs[1][0]) <= 1e-3
    for n, g in runs[0][1].items():
        assert float((g - runs[1][1][n]).norm()) <= 2e-2 * float(g.norm()) + 1e-6, n


@pytest.mark.parametrize("dtype", DTYPES)
def test_fid_long_generate_cached_matches_uncached(dev, dtype):
    """Greedy generation at text_maxlength 1024: the KV-cached decode equals the path that re-runs the decoder prefix,
    wherever the teacher-forced top-2 gap exceeds the 16-bit noise (the rule of test_round2_gpu)."""
    model, _ = _reader(dtype, dev)
    model.eval()
    ids, mask, _ = _long_inputs(2, 2, 1024, seed=7)
    model.encoder.config.n_context, model.encoder.config.bsz = 2, 2
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


def test_atlas_training_step_long_passages(dev):
    """One `Atlas.forward(..., train_retriever=True)` step with the ppmean gold scores at text_maxlength 1024: finite
    losses and reader / retriever gradients."""
    import atlas_synth
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever

    ret_ids = np.load(os.path.join(GOLDEN_DIR, "atlas_tiny.npz"))["ret_ids"]
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    corpus = atlas_synth.make_corpus()
    passages = [[corpus[int(i)] for i in row] for row in ret_ids]
    query, target = atlas_synth.make_batch()
    opt = atlas_synth.make_opt(gold_score_mode="ppmean", text_maxlength=1024, temperature_gold=0.1, temperature_score=0.1)
    reader = FiD(T5ConfigLite(**T5_KW))
    reader.load_state_dict(model_synth.fill_state_dict(reader.state_dict(), 202)[0])
    contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    contriever.load_state_dict(model_synth.fill_state_dict(contriever.state_dict(), seed=101)[0])
    model = Atlas(opt, reader.to(dev), DualEncoderRetriever(opt, contriever.to(dev)), reader_tok, retriever_tok).eval()
    model.retrieve = lambda *a, **k: (passages, None)
    reader_loss, retriever_loss = model(None, query, target, train_retriever=True, iter_stats={})
    assert torch.isfinite(reader_loss) and torch.isfinite(retriever_loss) and retriever_loss.requires_grad
    (reader_loss + retriever_loss).backward()
    rel = reader.encoder.block[0].layer[0].SelfAttention.relative_attention_bias.weight.grad
    assert rel is not None and bool(torch.isfinite(rel).all()) and float(rel.norm()) > 0
    assert contriever.encoder.layer[0].attention.self.query.weight.grad is not None


def test_fid_text_maxlength_limit(dev):
    """text_maxlength = 4097 raises the documented error, in evaluation and in training."""
    from atlas_b200._lib import AtlasB200Error

    model, _ = _reader(torch.bfloat16, dev, num_layers=1, num_decoder_layers=1)
    model.encoder.config.n_context, model.encoder.config.bsz = 1, 1
    ids = torch.full((1, 4097), 5, dtype=torch.long, device=dev)
    mask = torch.ones_like(ids, dtype=torch.bool)
    labels = torch.full((1, 4), 7, dtype=torch.long, device=dev)
    model.eval()
    with torch.no_grad(), pytest.raises(AtlasB200Error, match="at most 4096 tokens"):
        model(input_ids=ids, attention_mask=mask, labels=labels)
    model.train()
    with pytest.raises(AtlasB200Error, match="at most 4096 tokens"):
        model(input_ids=ids, attention_mask=mask, labels=labels)
