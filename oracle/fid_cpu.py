"""CPU restatement (plain torch, fp32) of the reference's Fusion-in-Decoder forward and Contriever forward.

TEST INFRASTRUCTURE: the checker for the CUDA path and the timed CPU baseline of bench.py - never imported by
`atlas_b200/`.  `/root/reference` does not exist on the GPU box, so this module restates the algorithm from the
reference sources; it is PINNED against outputs of the unmodified reference (tests/golden/fid_tiny.npz,
contriever_tiny.npz, produced by oracle/make_golden_models.py) in tests/test_oracle_golden.py.

Follows (file:line under /root/reference/src):
  FiDStack.forward                fid.py:32-78        [B, n*L] -> [B*n, L] -> T5 encoder -> [B, n*L, d]
  T5Stack.forward                 modeling_t5.py:875-1083   embed, blocks, final RMSNorm; layer-0 position bias reused
  T5LayerNorm                     modeling_t5.py:235-253    x * rsqrt(mean(x^2) + eps) * w      (no mean subtraction)
  T5Attention.forward             modeling_t5.py:418-531    scores = q k^T (NO 1/sqrt(d)) + position_bias + mask; fp32 softmax
  _relative_position_bucket       modeling_t5.py:352-397    32 buckets, bidirectional (encoder) / unidirectional (decoder)
  T5DenseGatedGeluDense           modeling_t5.py:272-289    gelu_new(x W0) * (x W1) -> Wo
  T5ForConditionalGeneration.forward  modeling_t5.py:1523-1669   lm_head (untied for v1.1), CE(ignore_index=-100)
  masks: transformers==4.18 get_extended_attention_mask ((1-m)*-10000; causal product for the decoder) and
         invert_attention_mask ((1-m)*-1e9 in fp32).
  Contriever.forward              retrievers.py:22-60; BertLayerNorm modeling_bert.py:104-114 (UNCENTRED 2nd moment);
  BertSelfAttention               modeling_bert.py:328-366  (1/sqrt(64), additive mask, fp32 softmax); erf-GELU.
"""
import math

import torch
import torch.nn.functional as F


def gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def rms_norm(x, w, eps):
    var = x.float().pow(2).mean(-1, keepdim=True)
    return w * (x * torch.rsqrt(var + eps))


def relative_position_bucket(rel, bidirectional, num_buckets=32, max_distance=128):
    out = torch.zeros_like(rel)
    if bidirectional:
        num_buckets //= 2
        out = out + (rel > 0).long() * num_buckets
        rel = rel.abs()
    else:
        rel = -torch.min(rel, torch.zeros_like(rel))
    max_exact = num_buckets // 2
    small = rel < max_exact
    large = max_exact + (torch.log(rel.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).long()
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return out + torch.where(small, rel, large)


def position_bias(weight, lq, lk, bidirectional, num_buckets):
    ctx = torch.arange(lq)[:, None]
    mem = torch.arange(lk)[None, :]
    buckets = relative_position_bucket(mem - ctx, bidirectional, num_buckets)
    return weight[buckets].permute(2, 0, 1)[None]          # [1, H, lq, lk]


def _heads(x, H):
    B, L, _ = x.shape
    return x.view(B, L, H, -1).transpose(1, 2)


def t5_attention(sd, prefix, x, kv, bias, H):
    q = _heads(x @ sd[prefix + "q.weight"].T, H)
    k = _heads(kv @ sd[prefix + "k.weight"].T, H)
    v = _heads(kv @ sd[prefix + "v.weight"].T, H)
    scores = q @ k.transpose(-1, -2) + bias
    p = torch.softmax(scores.float(), dim=-1)
    o = (p @ v).transpose(1, 2).reshape(x.shape[0], x.shape[1], -1)
    return o @ sd[prefix + "o.weight"].T


def t5_ff(sd, prefix, h, eps):
    n = rms_norm(h, sd[prefix + "layer_norm.weight"], eps)
    g = gelu_new(n @ sd[prefix + "DenseReluDense.wi_0.weight"].T) * (n @ sd[prefix + "DenseReluDense.wi_1.weight"].T)
    return h + g @ sd[prefix + "DenseReluDense.wo.weight"].T


def fid_forward(sd, cfg, input_ids, attention_mask, decoder_input_ids, labels=None, n_context=1):
    """sd: HF-named fp32 state dict; cfg: dict with d_model, num_heads, num_layers, num_decoder_layers,
    relative_attention_num_buckets, layer_norm_epsilon.  Returns (loss or None, logits [B, T, V], enc [B, n*L, d])."""
    H, eps, nb = cfg["num_heads"], cfg["layer_norm_epsilon"], cfg["relative_attention_num_buckets"]
    B = input_ids.shape[0]
    ids = input_ids.reshape(B * n_context, -1)
    mask = attention_mask.reshape(B * n_context, -1).float()
    L = ids.shape[1]
    emb = sd["shared.weight"]
    h = emb[ids]
    ext = (1.0 - mask)[:, None, None, :] * -10000.0
    bias = position_bias(sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], L, L, True, nb) + ext
    for i in range(cfg["num_layers"]):
        p = f"encoder.block.{i}.layer.0."
        n = rms_norm(h, sd[p + "layer_norm.weight"], eps)
        h = h + t5_attention(sd, p + "SelfAttention.", n, n, bias, H)
        h = t5_ff(sd, f"encoder.block.{i}.layer.1.", h, eps)
    enc = rms_norm(h, sd["encoder.final_layer_norm.weight"], eps).reshape(B, n_context * L, -1)

    T = decoder_input_ids.shape[1]
    d = emb[decoder_input_ids]
    causal = (torch.arange(T)[None, :] <= torch.arange(T)[:, None]).float()
    self_bias = position_bias(sd["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], T, T, False, nb) \
        + (1.0 - causal)[None, None] * -10000.0
    cross_bias = (1.0 - attention_mask.reshape(B, -1).float())[:, None, None, :] * -1e9
    for i in range(cfg["num_decoder_layers"]):
        p = f"decoder.block.{i}.layer.0."
        n = rms_norm(d, sd[p + "layer_norm.weight"], eps)
        d = d + t5_attention(sd, p + "SelfAttention.", n, n, self_bias, H)
        p = f"decoder.block.{i}.layer.1."
        n = rms_norm(d, sd[p + "layer_norm.weight"], eps)
        d = d + t5_attention(sd, p + "EncDecAttention.", n, enc, cross_bias, H)
        d = t5_ff(sd, f"decoder.block.{i}.layer.2.", d, eps)
    d = rms_norm(d, sd["decoder.final_layer_norm.weight"], eps)
    logits = d @ sd["lm_head.weight"].T                       # untied head (T5 v1.1): no d^-0.5 rescale
    loss = None
    if labels is not None:
        loss = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), labels.reshape(-1), ignore_index=-100)
    return loss, logits, enc


def bert_layer_norm(x, w, b, eps):
    u = x.mean(-1, keepdim=True)
    s = x.pow(2).mean(-1, keepdim=True)            # E[x^2], NOT the variance (modeling_bert.py:108-112)
    return w * ((x - u) * torch.rsqrt(s + eps)) + b


def contriever_forward(sd, cfg, input_ids, attention_mask):
    """Contriever (BERT + masked mean pooling) in fp32.  Returns [B, hidden]."""
    H, eps = cfg["num_attention_heads"], cfg["layer_norm_eps"]
    B, L = input_ids.shape
    x = sd["embeddings.word_embeddings.weight"][input_ids] + sd["embeddings.token_type_embeddings.weight"][0] \
        + sd["embeddings.position_embeddings.weight"][:L][None]
    x = bert_layer_norm(x, sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], eps)
    ext = (1.0 - attention_mask.float())[:, None, None, :] * -10000.0
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        lin = lambda t, name: t @ sd[p + name + ".weight"].T + sd[p + name + ".bias"]
        q, k, v = (_heads(lin(x, "attention.self." + n), H) for n in ("query", "key", "value"))
        pr = torch.softmax((q @ k.transpose(-1, -2) / math.sqrt(q.shape[-1]) + ext).float(), dim=-1)
        ctx = (pr @ v).transpose(1, 2).reshape(B, L, -1)
        x = bert_layer_norm(lin(ctx, "attention.output.dense") + x, sd[p + "attention.output.LayerNorm.weight"],
                            sd[p + "attention.output.LayerNorm.bias"], eps)
        inter = F.gelu(lin(x, "intermediate.dense"))
        x = bert_layer_norm(lin(inter, "output.dense") + x, sd[p + "output.LayerNorm.weight"],
                            sd[p + "output.LayerNorm.bias"], eps)
    m = attention_mask[..., None].bool()
    x = x.masked_fill(~m, 0.0)
    return x.sum(dim=1) / attention_mask.sum(dim=1)[..., None]


# ---------------------------------------------------------------------------------------------
# random-init fp32 state dicts under the HF parameter names (bench.py's CPU baseline / reference arm)
# ---------------------------------------------------------------------------------------------
T5_BASE = dict(vocab_size=32128, d_model=768, d_kv=64, d_ff=2048, num_layers=12, num_decoder_layers=12, num_heads=12,
               relative_attention_num_buckets=32, layer_norm_epsilon=1e-6)
BERT_BASE = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)


def t5_random_state(cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    d, dff, inner, V = cfg["d_model"], cfg["d_ff"], cfg["num_heads"] * cfg["d_kv"], cfg["vocab_size"]
    rn = lambda *shape, std=1.0: torch.randn(*shape, generator=g) * std
    sd = {"shared.weight": rn(V, d), "lm_head.weight": rn(V, d, std=d ** -0.5)}
    for stack, n in (("encoder", cfg["num_layers"]), ("decoder", cfg["num_decoder_layers"])):
        for i in range(n):
            blk = f"{stack}.block.{i}.layer."
            attn = [("0.SelfAttention.", i == 0)] + ([("1.EncDecAttention.", False)] if stack == "decoder" else [])
            for name, has_bias in attn:
                sd[blk + name + "q.weight"] = rn(inner, d, std=(d * cfg["d_kv"]) ** -0.5)
                sd[blk + name + "k.weight"] = rn(inner, d, std=d ** -0.5)
                sd[blk + name + "v.weight"] = rn(inner, d, std=d ** -0.5)
                sd[blk + name + "o.weight"] = rn(d, inner, std=inner ** -0.5)
                if has_bias:
                    sd[blk + name + "relative_attention_bias.weight"] = rn(cfg["relative_attention_num_buckets"],
                                                                           cfg["num_heads"], std=d ** -0.5)
                sd[blk + name[:2] + "layer_norm.weight"] = torch.ones(d)
            ff = blk + ("2." if stack == "decoder" else "1.")
            sd[ff + "DenseReluDense.wi_0.weight"] = rn(dff, d, std=d ** -0.5)
            sd[ff + "DenseReluDense.wi_1.weight"] = rn(dff, d, std=d ** -0.5)
            sd[ff + "DenseReluDense.wo.weight"] = rn(d, dff, std=dff ** -0.5)
            sd[ff + "layer_norm.weight"] = torch.ones(d)
        sd[f"{stack}.final_layer_norm.weight"] = torch.ones(d)
    return sd


def bert_random_state(cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    h, inter = cfg["hidden_size"], cfg["intermediate_size"]
    rn = lambda *shape: torch.randn(*shape, generator=g) * 0.02
    sd = {"embeddings.word_embeddings.weight": rn(cfg["vocab_size"], h),
          "embeddings.position_embeddings.weight": rn(cfg["max_position_embeddings"], h),
          "embeddings.token_type_embeddings.weight": rn(cfg["type_vocab_size"], h),
          "embeddings.LayerNorm.weight": torch.ones(h), "embeddings.LayerNorm.bias": torch.zeros(h)}
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        for name, (o, k) in {"attention.self.query": (h, h), "attention.self.key": (h, h), "attention.self.value": (h, h),
                             "attention.output.dense": (h, h), "intermediate.dense": (inter, h),
                             "output.dense": (h, inter)}.items():
            sd[p + name + ".weight"], sd[p + name + ".bias"] = rn(o, k), torch.zeros(o)
        for name in ("attention.output.LayerNorm", "output.LayerNorm"):
            sd[p + name + ".weight"], sd[p + name + ".bias"] = torch.ones(h), torch.zeros(h)
    return sd
