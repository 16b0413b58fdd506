"""Gradients of the CPU restatements (oracle/fid_cpu.py) by torch.autograd: the checker for the GPU training path.

TEST INFRASTRUCTURE (only tests/, smoke() and bench.py's CPU legs may import oracle/).  Pinned against the UNMODIFIED
reference's own gradients in tests/test_oracle_golden.py (tests/golden/grads_tiny.npz, oracle/make_golden_grads.py):
reference = `loss.backward()` through src/fid.py / src/modeling_t5.py / src/retrievers.py / src/modeling_bert.py."""
import zlib

import numpy as np
import torch

import fid_cpu


def direction(name, shape):
    """The seeded random direction make_golden_grads.py projects every gradient on."""
    rng = np.random.default_rng([7, zlib.crc32(name.encode())])
    return rng.standard_normal(shape, dtype=np.float32)


def _leafs(sd):
    out = {}
    for k, v in sd.items():
        if torch.is_floating_point(v) and not k.endswith("embed_tokens.weight"):
            out[k] = v.detach().float().clone().requires_grad_()
    full = dict(out)
    for k in sd:                                  # tied aliases share the leaf of `shared.weight`
        if k.endswith("embed_tokens.weight"):
            full[k] = out["shared.weight"]
    return out, full


def fid_grads(sd, cfg, input_ids, attention_mask, labels, n_context, shift_right):
    """-> (loss float, {parameter name: fp32 gradient})."""
    leafs, full = _leafs(sd)
    loss, _, _ = fid_cpu.fid_forward(full, cfg, input_ids, attention_mask, shift_right(labels), labels, n_context=n_context)
    loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in leafs.items() if v.grad is not None}


def contriever_grads(sd, cfg, input_ids, attention_mask):
    """Loss = the fixed linear functional of the embeddings used by make_golden_grads.py."""
    leafs, full = _leafs(sd)
    emb = fid_cpu.contriever_forward(full, cfg, input_ids, attention_mask)
    w = torch.from_numpy(direction("emb", tuple(emb.shape)))
    loss = (emb.float() * w).sum() / emb.shape[0]
    loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in leafs.items() if v.grad is not None}
