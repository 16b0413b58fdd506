"""CPU restatement of the opt-in FP8 (e4m3) cross K|V cache of KV-cached generation (csrc/kv_fp8.cu) and a teacher-forced
FiD decoder that attends over the dequantized cache.

TEST INFRASTRUCTURE, never imported by `atlas_b200/`.

  quantize_e4m3      the quantizer's rule in torch-CPU fp32 (IEEE division and multiplication, as __fdiv_rn / __fmul_rn),
                     then clamp(+-448) and a cast to torch.float8_e4m3fn (round to nearest even): the codes and scales the
                     kernel must produce bit for bit.
  dequantize_e4m3    float(e4m3(code)) * scale, in float64 (the product of a 4-bit significand and an fp32 scale is exact).
  decoder_logits     fid_cpu's decoder (self-attention through fid_cpu.t5_attention, the same RMSNorm / feed-forward / head)
                     with each layer's cross K and V given instead of projected from the encoder output: the reference a
                     kernel-level comparison of the fp8 decode steps needs, free of the quantization loss itself.
"""
import torch

import fid_cpu

E4M3_MAX = 448.0


def quantize_e4m3(x):
    """x [rows, C*64] (fp16 / bf16 / fp32 values) -> (codes uint8 [rows, C*64], scales fp32 [rows, C]).
    Per 64-value block: amax = max|x|, inv = 448 / amax, code = e4m3(x * inv), scale = amax / 448; amax == 0 -> scale 0 and
    codes 0; a NaN or inf in the block -> scale NaN and codes 0."""
    rows, n = x.shape
    C = n // 64
    xf = x.float().reshape(rows, C, 64)
    bad = ~torch.isfinite(xf).all(-1)
    amax = xf.abs().amax(-1)
    zero = amax == 0
    safe = torch.where(bad | zero, torch.ones_like(amax), amax)
    inv = torch.tensor(E4M3_MAX, dtype=torch.float32) / safe
    y = (xf * inv[..., None]).clamp(-E4M3_MAX, E4M3_MAX)
    codes = y.to(torch.float8_e4m3fn).view(torch.uint8)
    codes = torch.where((bad | zero)[..., None], torch.zeros_like(codes), codes)
    scale = amax / torch.tensor(E4M3_MAX, dtype=torch.float32)
    scale = torch.where(zero, torch.zeros_like(scale), scale)
    scale = torch.where(bad, torch.full_like(scale, float("nan")), scale)
    return codes.reshape(rows, C * 64), scale


def dequantize_e4m3(codes, scale):
    """codes uint8 [rows, C*64], scales fp32 [rows, C] -> float64 [rows, C*64]."""
    rows, n = codes.shape
    v = codes.contiguous().view(torch.float8_e4m3fn).double().reshape(rows, n // 64, 64)
    return (v * scale.double()[..., None]).reshape(rows, n)


def _cross_attention_given_kv(sd, prefix, x, k, v, bias, H):
    """fid_cpu.t5_attention with the key / value projections replaced by given per-head K, V [B, Lk, H*64]."""
    q = fid_cpu._heads(x @ sd[prefix + "q.weight"].T, H)
    scores = q @ fid_cpu._heads(k, H).transpose(-1, -2) + bias
    p = torch.softmax(scores.float(), dim=-1)
    o = (p @ fid_cpu._heads(v, H)).transpose(1, 2).reshape(x.shape[0], x.shape[1], -1)
    return o @ sd[prefix + "o.weight"].T


def decoder_logits(sd, cfg, enc_mask, decoder_input_ids, cross_k, cross_v):
    """Teacher-forced decoder logits [B, T, V] in fp32 from the per-layer cross K / V ([B, Lk, H*64] each) and the encoder
    mask [B, Lk]; the rest as fid_cpu.fid_forward (untied T5 v1.1 head)."""
    H, eps, nb = cfg["num_heads"], cfg["layer_norm_epsilon"], cfg["relative_attention_num_buckets"]
    B, T = decoder_input_ids.shape
    d = sd["shared.weight"][decoder_input_ids]
    causal = (torch.arange(T)[None, :] <= torch.arange(T)[:, None]).float()
    self_bias = fid_cpu.position_bias(sd["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], T, T, False,
                                      nb) + (1.0 - causal)[None, None] * -10000.0
    cross_bias = (1.0 - enc_mask.reshape(B, -1).float())[:, None, None, :] * -1e9
    for i in range(cfg["num_decoder_layers"]):
        p = f"decoder.block.{i}.layer.0."
        n = fid_cpu.rms_norm(d, sd[p + "layer_norm.weight"], eps)
        d = d + fid_cpu.t5_attention(sd, p + "SelfAttention.", n, n, self_bias, H)
        p = f"decoder.block.{i}.layer.1."
        n = fid_cpu.rms_norm(d, sd[p + "layer_norm.weight"], eps)
        d = d + _cross_attention_given_kv(sd, p + "EncDecAttention.", n, cross_k[i].float(), cross_v[i].float(), cross_bias, H)
        d = fid_cpu.t5_ff(sd, f"decoder.block.{i}.layer.2.", d, eps)
    d = fid_cpu.rms_norm(d, sd["decoder.final_layer_norm.weight"], eps)
    return d @ sd["lm_head.weight"].T
