"""T5 v1.0 readers (t5-small / -base / -large) on the host: the golden of the unmodified reference
(tests/golden/fid_relu_tiny.npz, oracle/make_golden_t5v10.py) is self-consistent, `FiD.from_pretrained` reads the original
t5 checkpoint layout as a tied ReLU model while v1.1 checkpoints keep loading as before, and head dimension 128
(t5-3b / t5-11b) is refused with a clear message."""
import json
import os

import numpy as np
import pytest
import torch

import model_synth
from conftest import GOLDEN_DIR

GEOMETRIES = {"base": (768, 12, 3072), "small": (512, 8, 2048)}       # d_model, heads, d_ff


def _cfg(**over):
    from atlas_b200.fid import T5ConfigLite

    kw = {k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    kw.update(over)
    return T5ConfigLite(**kw)


def test_golden_self_consistent():
    g = np.load(os.path.join(GOLDEN_DIR, "fid_relu_tiny.npz"))
    for tag, (d, _, d_ff) in GEOMETRIES.items():
        assert g[f"{tag}/logits_fp32"].shape == (2, 8, 512)
        assert g[f"{tag}/enc_fp32"].shape == (64, d)                # the first passage of the first query
        for dt, tdt in (("fp16", torch.float16), ("bf16", torch.bfloat16)):
            bits = g[f"{tag}/logits_{dt}_bits"]
            assert bits.shape == (2, 8, 512) and bits.dtype == np.int16
            logits16 = torch.from_numpy(bits).view(tdt).float().numpy()
            assert 0 < np.abs(logits16 - g[f"{tag}/logits_fp32"]).max() < 0.1
            assert abs(float(g[f"{tag}/loss_{dt}"]) - float(g[f"{tag}/loss_fp32"])) < 2e-2
        # the reference's no-grad and with-grad fp32 runs give the same loss
        assert abs(float(g[f"{tag}/grad_fp32/loss"]) - float(g[f"{tag}/loss_fp32"])) < 1e-4
        # the tie: one fingerprint for the table, none for lm_head; ReLU feed-forward parameter names
        assert f"{tag}/grad_fp32/norm/shared.weight" in g.files
        assert not any("lm_head" in k for k in g.files if k.startswith(tag + "/"))
        assert f"{tag}/grad_fp32/norm/encoder.block.1.layer.1.DenseReluDense.wi.weight" in g.files
        assert not any("wi_0" in k for k in g.files)
        assert g[f"{tag}/grad_fp32/full/encoder.final_layer_norm.weight"].shape == (d,)
        # every full small tensor has the reference's own bf16 relative error beside it
        full = [k.split("/full/")[1] for k in g.files if k.startswith(f"{tag}/grad_fp32/full/")]
        assert full and all(0 <= float(g[f"{tag}/grad_bf16/relerr/{n}"]) < 0.2 for n in full)
    # the same model: the weights of our FiD filled like the golden's
    from atlas_b200.fid import FiD

    for tag, (d, h, d_ff) in GEOMETRIES.items():
        m = FiD(_cfg(feed_forward_proj="relu", tie_word_embeddings=True, d_model=d, num_heads=h, d_ff=d_ff))
        _, sha = model_synth.fill_state_dict(m.state_dict(), 202)
        assert sha == str(g[f"{tag}/weights_sha256"]), tag


def _write_checkpoint(path, relu, with_head):
    from atlas_b200.fid import FiD

    model = FiD(_cfg(feed_forward_proj="relu" if relu else "gated-gelu", tie_word_embeddings=relu))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 5)
    if not with_head:
        del sd["lm_head.weight"]
    torch.save(sd, os.path.join(path, "pytorch_model.bin"))
    # the original t5-base config.json states neither feed_forward_proj nor tie_word_embeddings
    cfg = {k: v for k, v in model_synth.T5_CFG.items()
           if k not in ("feed_forward_proj", "tie_word_embeddings", "dropout_rate", "is_encoder_decoder", "use_cache")}
    cfg["model_type"] = "t5"
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f)
    return sd


def test_from_pretrained_t5_v10_layout(tmp_path):
    from atlas_b200.fid import FiD

    sd = _write_checkpoint(str(tmp_path), relu=True, with_head=False)
    model = FiD.from_pretrained(str(tmp_path))
    assert model.config.feed_forward_proj == "relu" and model.config.tie_word_embeddings is True
    assert model.lm_head.weight is model.shared.weight
    ff = model.encoder.block[0].layer[1].DenseReluDense
    assert hasattr(ff, "wi") and not hasattr(ff, "wi_0")
    assert torch.equal(ff.wi.weight, sd["encoder.block.0.layer.1.DenseReluDense.wi.weight"].float())
    assert torch.equal(model.lm_head.weight, sd["shared.weight"].float())
    # an explicit tie_word_embeddings in config.json is honoured
    with open(tmp_path / "config.json") as f:
        cfg = json.load(f)
    cfg["tie_word_embeddings"] = False
    with open(tmp_path / "config.json", "w") as f:
        json.dump(cfg, f)
    with pytest.raises(Exception, match="lm_head"):           # untied: the checkpoint really lacks the head now
        FiD.from_pretrained(str(tmp_path))


def test_from_pretrained_v11_layout_unchanged(tmp_path):
    from atlas_b200.fid import FiD

    _write_checkpoint(str(tmp_path), relu=False, with_head=True)
    model = FiD.from_pretrained(str(tmp_path))
    assert model.config.feed_forward_proj == "gated-gelu" and model.config.tie_word_embeddings is False
    assert model.lm_head.weight is not model.shared.weight
    assert hasattr(model.decoder.block[1].layer[2].DenseReluDense, "wi_1")


def test_constructor_ties_and_refuses_d_kv_128():
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.fid import FiD

    m = FiD(_cfg(feed_forward_proj="relu", tie_word_embeddings=True))
    assert m.lm_head.weight is m.shared.weight
    assert [n for n, _ in m.named_parameters() if n in ("shared.weight", "lm_head.weight")] == ["shared.weight"]
    assert m.to(torch.bfloat16).lm_head.weight is m.shared.weight
    assert FiD(_cfg()).lm_head.weight is not FiD(_cfg()).shared.weight
    for d_model, heads in ((1024, 32), (1024, 128)):          # t5-3b, t5-11b
        with pytest.raises(AtlasB200Error, match="t5-3b") as e:
            FiD(_cfg(feed_forward_proj="relu", tie_word_embeddings=True, d_model=d_model, num_heads=heads, d_kv=128))
        assert "128" in str(e.value)
    with pytest.raises(AtlasB200Error, match="feed_forward_proj"):
        FiD(_cfg(feed_forward_proj="gated-silu"))
