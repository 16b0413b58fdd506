"""GPU: the sharded optimizer and gradient wrapper (atlas_b200/sharded.py) against `AdamWFP32Copy` and the plain module.

At one rank, `OSS` + `ShardedDataParallel` must be bit for bit `AdamWFP32Copy` + `torch.nn.utils.clip_grad_norm_`.  The
gradients of that comparison are designed so that both clipping rules are exact: every element of a parameter's
gradient is +-u with u a power of two, the parameters hold 16^2, 24^2, 48^2 and 42^2 elements (norms 16u, 24u, 48u,
42u, total 70u), and the clip threshold makes the coefficient a power of two.  So torch's 16-bit norm and this fp32
norm agree, and so do the clipped gradients.

With more than one rank, tests/_sharded_worker.py runs under torchrun (NCCL, one GPU per rank; skipped with fewer
GPUs)."""
import copy
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import model_synth
import shard_oracle

pytestmark = pytest.mark.gpu

SIDES = (16, 42, 24, 48)                 # sqrt of each parameter's numel: 16^2 + 42^2 + 24^2 + 48^2 = 70^2


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


class Bag(torch.nn.Module):
    """Parameters whose gradient is whatever tensor the forward is given: loss = sum_i sum(p_i * c_i)."""

    def __init__(self, shapes, dtype, dev, seed=3):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.ps = torch.nn.ParameterList(
            [torch.nn.Parameter((torch.randn(*s, generator=g) * 0.1).to(dtype).to(dev)) for s in shapes])

    def forward(self, cs):
        return sum((p * c).sum() for p, c in zip(self.ps, cs))


def _groups(params, lrs=(3e-3, 1e-3), wds=(0.1, 0.0)):
    params = list(params)
    return [{"params": params[0::2], "lr": lrs[0], "weight_decay": wds[0]},
            {"params": params[1::2], "lr": lrs[1], "weight_decay": wds[1]}]


def _designed_grads(step, dtype, dev):
    """+-u per element, u = 2^-6, 2^-5, 2^-7 at steps 1, 2, 3."""
    u = 2.0 ** (-6, -5, -7)[step - 1]
    g = torch.Generator().manual_seed(100 + step)
    return [((torch.randint(0, 2, (s, s), generator=g) * 2 - 1) * u).to(dtype).to(dev) for s in SIDES]


def _pair(dtype, dev, **kw):
    from atlas_b200.optim import AdamWFP32Copy
    from atlas_b200.sharded import OSS, ShardedDataParallel

    ref = Bag([(s, s) for s in SIDES], dtype, dev)
    mod = copy.deepcopy(ref)
    ref_opt = AdamWFP32Copy(_groups(ref.parameters()), betas=(0.9, 0.98), eps=1e-6, **kw)
    opt = OSS(_groups(mod.parameters()), optim=AdamWFP32Copy, betas=(0.9, 0.98), eps=1e-6, force_broadcast_object=True,
              **kw)
    return ref, ref_opt, ShardedDataParallel(mod, opt, auto_refresh_trainable=False), opt


def _bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_one_rank_is_adamw_fp32copy_bit_for_bit(dev, dtype):
    ref, ref_opt, sdp, opt = _pair(dtype, dev)
    scale, clip = 4.0, 35 * 2.0 ** -6 / 4.0        # coefficients 1/2, 1/4 and 1 (not clipped) at steps 1, 2, 3
    for step in (1, 2, 3):
        cs = _designed_grads(step, dtype, dev)
        ref.zero_grad(set_to_none=True)
        ref(cs).backward()
        want = torch.nn.utils.clip_grad_norm_(ref.parameters(), scale * clip)
        ref_opt.step(scale=scale)
        sdp.zero_grad(set_to_none=True)
        sdp(cs).backward()
        got = opt.clip_grad_norm(scale * clip)
        opt.step(scale=scale)
        assert float(got) == float(want) == 70 * 2.0 ** (-6, -5, -7)[step - 1]
        for a, b in zip(ref.parameters(), sdp.module.parameters()):
            assert torch.equal(_bits(a), _bits(b)), step
    sd_ref, sd = ref_opt.state_dict(), opt.state_dict()
    assert sorted(sd["state"]) == sorted(sd_ref["state"]) == [0, 1, 2, 3]
    for i, st in sd_ref["state"].items():
        assert int(sd["state"][i]["step"]) == int(st["step"]) == 3
        for key in ("float32copy", "exp_avg", "exp_avg_sq"):
            assert sd["state"][i][key].shape == st[key].shape
            assert torch.equal(_bits(sd["state"][i][key]), _bits(st[key])), (i, key)
    assert [g["params"] for g in sd["param_groups"]] == [g["params"] for g in sd_ref["param_groups"]]
    for g, h in zip(sd["param_groups"], sd_ref["param_groups"]):
        assert all(g[k] == h[k] for k in ("lr", "betas", "eps", "weight_decay"))


def test_layout_is_the_oracles(dev):
    from atlas_b200.sharded import OSS

    shapes = [(768, 768), (5,), (1000, 33), (1,), (63,), (2048, 130)]
    bag = Bag(shapes, torch.bfloat16, dev)
    before = [p.detach().clone() for p in bag.parameters()]
    opt = OSS(bag.parameters(), lr=1e-3)
    offsets, padded, shard = shard_oracle.partition([int(np.prod(s)) for s in shapes], 1)
    assert opt._padded == padded and opt._shard_size == shard
    assert opt._segments == [shard_oracle.segments([int(np.prod(s)) for s in shapes], 1, 0)]
    base = opt._flat.data_ptr()
    for p, o, b in zip(bag.parameters(), offsets.tolist(), before):
        assert p.data_ptr() == base + 2 * o and torch.equal(p, b)
    assert float(opt._flat[int(offsets[-1]) + 2048 * 130:].abs().sum()) == 0.0


def test_accumulation_equals_one_backward_of_the_sum(dev):
    from atlas_b200.optim import AdamWFP32Copy
    from atlas_b200.sharded import OSS, ShardedDataParallel

    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(96, 160), torch.nn.GELU(), torch.nn.Linear(160, 40)).to(dev)
    net = net.to(torch.bfloat16)
    ref = copy.deepcopy(net)
    ref_opt = AdamWFP32Copy(ref.parameters(), lr=1e-3)
    opt = OSS(net.parameters(), lr=1e-3)
    sdp = ShardedDataParallel(net, opt)
    x1, x2 = (torch.randn(33, 96, device=dev).to(torch.bfloat16) for _ in range(2))
    sdp(x1).float().square().mean().backward()
    sdp(x2).float().square().mean().backward()
    (ref(x1).float().square().mean() + ref(x2).float().square().mean()).backward()
    for p, q in zip(net.parameters(), ref.parameters()):
        assert p.grad.data_ptr() >= opt._grad_flat.data_ptr()          # a view of the flat buffer
        torch.testing.assert_close(p.grad.float(), q.grad.float(), rtol=2e-2, atol=2e-2 * float(q.grad.abs().max()))
    opt.step()
    ref_opt.step()
    for p, q in zip(net.parameters(), ref.parameters()):
        torch.testing.assert_close(p.float(), q.float(), rtol=2e-2, atol=3e-3)   # a sign flip of a tiny gradient moves 2 lr


def test_zero_grad_then_skipped_step_leaves_no_stale_gradient(dev):
    ref, ref_opt, sdp, opt = _pair(torch.bfloat16, dev)
    sdp(_designed_grads(1, torch.bfloat16, dev)).backward()       # an example whose statistics say "skip"
    sdp.zero_grad()
    assert all(p.grad is None for p in sdp.parameters())
    cs = _designed_grads(2, torch.bfloat16, dev)
    sdp(cs).backward()
    opt.step(scale=2.0)
    ref(cs).backward()
    ref_opt.step(scale=2.0)
    for a, b in zip(ref.parameters(), sdp.module.parameters()):
        assert torch.equal(_bits(a), _bits(b))


def test_state_dict_round_trips_with_adamw_fp32copy(dev):
    from atlas_b200.optim import AdamWFP32Copy
    from atlas_b200.sharded import OSS, ShardedDataParallel

    ref, ref_opt, sdp, opt = _pair(torch.bfloat16, dev)
    for step in (1, 2):
        cs = _designed_grads(step, torch.bfloat16, dev)
        ref.zero_grad(set_to_none=True)
        ref(cs).backward()
        ref_opt.step(scale=2.0)
        sdp.zero_grad(set_to_none=True)
        sdp(cs).backward()
        opt.step(scale=2.0)
    buf = io.BytesIO()
    torch.save({"ref": ref_opt.state_dict(), "oss": opt.state_dict()}, buf)
    buf.seek(0)
    saved = torch.load(buf, weights_only=False)
    cs = _designed_grads(3, torch.bfloat16, dev)

    # AdamWFP32Copy -> OSS: the resumed OSS run is the uninterrupted AdamWFP32Copy run
    mod2 = copy.deepcopy(ref)
    opt2 = OSS(_groups(mod2.parameters(), lrs=(9.0, 9.0)), lr=9.0, betas=(0.9, 0.98), eps=1e-6)
    opt2.load_state_dict(saved["ref"])
    assert [g["lr"] for g in opt2.param_groups] == [3e-3, 1e-3]
    sdp2 = ShardedDataParallel(mod2, opt2)
    sdp2(cs).backward()
    opt2.step(scale=2.0)
    ref.zero_grad(set_to_none=True)
    ref(cs).backward()
    ref_opt.step(scale=2.0)
    for a, b in zip(ref.parameters(), mod2.parameters()):
        assert torch.equal(_bits(a), _bits(b))

    # OSS -> AdamWFP32Copy: loads and resumes (torch's load casts the state to the parameters' dtype)
    mod3 = copy.deepcopy(sdp.module)
    opt3 = AdamWFP32Copy(_groups(mod3.parameters()), betas=(0.9, 0.98), eps=1e-6)
    opt3.load_state_dict(saved["oss"])
    assert all(int(opt3.state[p]["step"]) == 2 for p in mod3.parameters())
    mod3(cs).backward()
    opt3.step(scale=2.0)
    assert all(int(opt3.state[p]["step"]) == 3 for p in mod3.parameters())
    for a, b in zip(ref.parameters(), mod3.parameters()):
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-2, atol=1e-3)

    opt._all_states = []            # src/model_io.py:244
    assert opt.state_dict()["state"][0]["step"] == 2


def test_compute_grad_stats_over_a_wrapped_reader(dev):
    from types import SimpleNamespace

    from atlas_b200.optim import compute_grad_stats
    from atlas_b200.sharded import OSS, ShardedDataParallel

    torch.manual_seed(1)
    reader = torch.nn.Sequential(torch.nn.Linear(64, 64), torch.nn.Linear(64, 8)).to(dev).to(torch.bfloat16)
    plain = copy.deepcopy(reader)
    x = torch.randn(16, 64, device=dev).to(torch.bfloat16)
    wrapped = ShardedDataParallel(reader, OSS(reader.parameters(), lr=1e-3))
    wrapped(x).float().sum().backward()
    plain(x).float().sum().backward()
    got = compute_grad_stats(SimpleNamespace(reader=wrapped))
    want = compute_grad_stats(SimpleNamespace(reader=plain))
    assert got == want


def test_fid_cuda_graph_forward_survives_repointing(dev):
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.sharded import OSS

    kw = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    model = FiD(T5ConfigLite(**kw))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    model = model.to(torch.bfloat16).to(dev).eval()
    model.encoder.config.n_context, model.encoder.config.bsz = 3, 2
    assert model.cuda_graphs
    ids, mask, labels = (t.to(dev) for t in model_synth.fid_inputs())

    def logits():
        with torch.no_grad():
            return model(input_ids=ids, attention_mask=mask, labels=labels).logits.clone()

    # the FiD forward is not bitwise reproducible from run to run (its logits move by up to ~0.016 between replays and
    # eager calls on an H100), so "the same logits" is: within that spread, while a real weight change moves them far more
    before = logits()
    ptrs = [p.data_ptr() for p in model.parameters()]
    opt = OSS(model.parameters(), lr=1e-3)
    assert all(p.data_ptr() != q for p, q in zip(model.parameters(), ptrs))
    for _ in range(3):                                 # capture on the new weight buffers, then replays
        torch.testing.assert_close(logits(), before, rtol=0, atol=5e-2)
    with torch.no_grad():                              # the replayed graph reads the re-pointed weights
        opt._flat.mul_(0.5)
    from atlas_b200.retrievers import _bump_weights_epoch

    _bump_weights_epoch()
    logits()
    assert float((logits().float() - before.float()).abs().max()) > 0.25


def test_atlas_training_step_with_wrapped_reader_and_retriever(dev):
    import atlas_synth
    from atlas_b200.atlas import Atlas
    from atlas_b200.fid import FiD, T5ConfigLite
    from atlas_b200.optim import compute_grad_stats
    from atlas_b200.retrievers import BertConfigLite, Contriever, DualEncoderRetriever
    from atlas_b200.sharded import OSS, ShardedDataParallel
    from conftest import GOLDEN_DIR

    ret_ids = np.load(os.path.join(GOLDEN_DIR, "atlas_tiny.npz"))["ret_ids"]
    opt = atlas_synth.make_opt(temperature_gold=0.1, temperature_score=0.1, gold_score_mode="ppmean")
    reader_tok, retriever_tok = atlas_synth.tokenizers()
    kw = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    reader = FiD(T5ConfigLite(**kw))
    reader.load_state_dict(model_synth.fill_state_dict(reader.state_dict(), seed=202)[0])
    contriever = Contriever(BertConfigLite(**model_synth.CONTRIEVER_CFG))
    contriever.load_state_dict(model_synth.fill_state_dict(contriever.state_dict(), seed=101)[0])
    retriever = DualEncoderRetriever(opt, contriever.to(dev))
    model = Atlas(opt, reader.to(dev), retriever, reader_tok, retriever_tok).eval()
    reader_opt = OSS(model.reader.parameters(), lr=1e-4, weight_decay=0.01, betas=(0.9, 0.999), eps=1e-6)
    retr_opt = OSS(model.retriever.parameters(), lr=1e-5, weight_decay=0.01, betas=(0.9, 0.999), eps=1e-6)
    model.reader = ShardedDataParallel(model.reader, reader_opt, auto_refresh_trainable=False)
    model.retriever = ShardedDataParallel(model.retriever, retr_opt, auto_refresh_trainable=False)
    corpus = atlas_synth.make_corpus()
    passages = [[corpus[int(i)] for i in row] for row in ret_ids]
    query, target = atlas_synth.make_batch()
    model.retrieve = lambda *a, **k: (passages, None)
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    losses = []
    for _ in range(2):
        reader_loss, retriever_loss = model(None, query, target, train_retriever=True, iter_stats={})
        (reader_loss + retriever_loss).backward()
        losses.append(float(reader_loss))
        stats = compute_grad_stats(model)
        assert not stats["skip_example"] and stats["max"] > 0
        for o in (reader_opt, retr_opt):
            assert torch.isfinite(o.clip_grad_norm(1.0))
            o.step(scale=1.0)
        model.zero_grad()
    assert all(np.isfinite(losses))
    moved = [n for n, p in model.named_parameters() if not torch.equal(p, before[n])]
    assert any(n.startswith("reader.") for n in moved) and any(n.startswith("retriever.") for n in moved)


def _torchrun(world, backend, tmp_path):
    from conftest import ROOT

    res = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
         "127.0.0.1", "--master-port", str(29881 + world), ROOT + "/tests/_sharded_worker.py", backend, str(tmp_path)],
        capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_ranks_nccl(world, tmp_path):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    _torchrun(world, "nccl", tmp_path)
