"""Generate tests/golden/fid_relu_tiny.npz: the UNMODIFIED reference `src.fid.FiD` built as a T5 v1.0 reader
(feed_forward_proj="relu" -> T5DenseReluDense, LM head tied to `shared` and fed the final hidden state scaled by
d_model^-0.5), run on CPU under oracle/ref_shims.py with seeded weights / inputs (oracle/model_synth.py).

TEST INFRASTRUCTURE.  Two geometries, each under its own key prefix:
  base   model_synth.T5_CFG with d_ff 3072 (t5-base proportions: d_model 768, 12 heads)
  small  t5-small proportions: d_model 512, 8 heads, d_ff 2048, 2 + 2 layers
Stored per geometry, as make_golden_models.py / make_golden_grads.py store them for T5 v1.1: the fp32 loss and logits,
the fp32 encoder states of the first passage of the first query (`enc_fp32`, [64, d] in fp16: the whole [2, 192, d] tensor
would make up most of the file), the reference's own fp16 / bf16 logits (`logits_{fp16,bf16}_bits`, their 16-bit patterns
as int16) and losses (the accuracy budget), and the gradient fingerprints of the fp32 run (L2 norm, seeded projection, full
small tensors) and of the bf16-parameter run, dropout off.  For the small tensors the bf16 run also stores its relative L2
distance from the fp32 run (`grad_bf16/relerr/<name>`): the ReLU's hard mask flips with 16-bit rounding, and the
reference's own bf16 run sits up to ~9 % from its fp32 run on the feed-forward norm weights' gradients.
`shared.weight` carries the embedding AND the LM-head gradient (one tied parameter)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_grads  # noqa: E402
import model_synth  # noqa: E402
import ref_shims  # noqa: E402

GOLDEN_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")
SEED = 202

GEOMETRIES = {
    "base": dict(model_synth.T5_CFG, feed_forward_proj="relu", tie_word_embeddings=True, d_ff=3072),
    "small": dict(model_synth.T5_CFG, feed_forward_proj="relu", tie_word_embeddings=True, d_model=512, num_heads=8,
                  d_ff=2048),
}


def tied_state_dict(sd_keys_model):
    """Seeded weights with the LM head equal to the embedding (the two names of one tied parameter)."""
    sd, sha = model_synth.fill_state_dict(sd_keys_model.state_dict(), SEED)
    sd["lm_head.weight"] = sd["shared.weight"].clone()
    return sd, sha


def build(cfg_kw, sd, dt):
    from transformers import T5Config
    from src.fid import FiD

    model = FiD(T5Config(**cfg_kw))
    # transformers 5.x does not tie on a flag set after construction, nor always from the kwarg: tie explicitly
    model.lm_head.weight = model.shared.weight
    assert model.lm_head.weight.data_ptr() == model.shared.weight.data_ptr()
    assert type(model.encoder.block[0].layer[1].DenseReluDense).__name__ == "T5DenseReluDense"
    assert model.config.tie_word_embeddings
    if sd is not None:
        model.load_state_dict(sd)
    model = model.to(dt).eval()                     # eval: dropout off (gradients stay enabled where asked)
    assert model.lm_head.weight.data_ptr() == model.shared.weight.data_ptr()
    model.encoder.config.n_context = 3
    model.encoder.config.bsz = 2
    return model


def geometry(tag, cfg_kw, out):
    ids, mask, labels = model_synth.fid_inputs(vocab=cfg_kw["vocab_size"])
    sd, sha = tied_state_dict(build(cfg_kw, None, torch.float32))
    out[f"{tag}/weights_sha256"] = np.array(sha)
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16), ("fp16", torch.float16)):
        model = build(cfg_kw, sd, dt)
        with torch.no_grad():
            res = model(input_ids=ids, attention_mask=mask, decoder_input_ids=model._shift_right(labels), labels=labels,
                        use_cache=False)
        out[f"{tag}/loss_{name}"] = np.array(float(res[0]))
        if name == "fp32":                          # encoder states in fp16 to keep the fixture small (values are O(1))
            out[f"{tag}/logits_fp32"] = res[1].numpy()
            out[f"{tag}/enc_fp32"] = res.encoder_last_hidden_state[0, :64].numpy().astype(np.float16)
        else:
            out[f"{tag}/logits_{name}_bits"] = res[1].view(torch.int16).numpy()
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        model = build(cfg_kw, sd, dt)
        res = model(input_ids=ids, attention_mask=mask, decoder_input_ids=model._shift_right(labels), labels=labels,
                    use_cache=False)
        res[0].backward()
        assert torch.isfinite(res[0]) and torch.isfinite(model.shared.weight.grad).all()
        out[f"{tag}/grad_{name}/loss"] = np.float32(float(res[0]))
        make_golden_grads.fingerprints(model, f"{tag}/grad_{name}", out, full=(name == "fp32"))
        if name == "bf16":
            for n, p in model.named_parameters():
                ref = out.get(f"{tag}/grad_fp32/full/{n}")
                if ref is not None:
                    err = np.linalg.norm(p.grad.float().numpy() - ref) / np.linalg.norm(ref)
                    out[f"{tag}/grad_bf16/relerr/{n}"] = np.float32(err)
    for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
        logits16 = torch.from_numpy(out[f"{tag}/logits_{name}_bits"]).view(dt).float().numpy()
        print(f"{tag}: reference {name} vs fp32 logits max abs diff", float(np.abs(logits16 - out[f"{tag}/logits_fp32"]).max()),
              "loss", float(out[f"{tag}/loss_{name}"]), float(out[f"{tag}/loss_fp32"]))


if __name__ == "__main__":
    ref_shims.install()
    torch.manual_seed(0)
    out = {}
    for tag, kw in GEOMETRIES.items():
        geometry(tag, kw, out)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "fid_relu_tiny.npz"), **out)
    print(len(out), "entries")
