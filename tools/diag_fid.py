import os, sys, math
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import model_synth
from atlas_b200 import ops
from atlas_b200.fid import FiD, T5ConfigLite, bias_by_delta
dev = torch.device("cuda:0")
g = np.load(os.path.join(ROOT, "tests/golden/fid_tiny.npz"))
dt = torch.float16
cfg = T5ConfigLite(**{k: v for k, v in model_synth.T5_CFG.items() if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")})
model = FiD(cfg)
sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
model.load_state_dict(sd); model = model.to(dt).to(dev).eval()
ids, mask, labels = model_synth.fid_inputs()
ids, mask, labels = ids.to(dev), mask.to(dev), labels.to(dev)
B, n_ctx = 2, 3
model.encoder.config.n_context, model.encoder.config.bsz = n_ctx, B
with torch.no_grad():
    enc = model.encode(ids, mask)
print("enc err vs golden fp32:", float((enc.float().cpu() - torch.from_numpy(g["enc_fp32"].astype(np.float32))).abs().max()))
# ---- fp32 torch reference of the decoder using the same weights, fed with OUR encoder output ----
W = {k: v.float().to(dev) for k, v in sd.items()}
H, d = 12, 768
dec_in = model._shift_right(labels)
T = dec_in.shape[1]
encf = enc.float()
Lk = encf.shape[1]
def rms(x, w): return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6))
def heads(x, L): return x.view(B, L, H, 64).permute(0, 2, 1, 3)
h = W["shared.weight"][dec_in]                       # [B,T,d]
bias = bias_by_delta(W["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], T, T, False, 32)  # [H, 2T-1]
i = torch.arange(T, device=dev)
idx = i[None, :] - i[:, None] + (T - 1)
pos_bias = bias[:, idx][None]                         # [1,H,T,T]
causal = (i[None, :] > i[:, None]).float() * -10000.0
cross_mask = (1.0 - mask.view(B, Lk).float()) * -1e4
# ours, stage by stage
Wh, G, _ = model._weights()
with torch.no_grad():
    hh = Wh["shared.weight"][dec_in.reshape(-1)]
    for L_ in range(2):
        p = f"decoder.block.{L_}.layer.0."
        # reference self-attn
        n = rms(h, W[p + "layer_norm.weight"])
        q, k, v = [heads(n @ W[p + f"SelfAttention.{x}.weight"].T, T) for x in "qkv"]
        s = q @ k.transpose(-1, -2) + pos_bias + causal
        a = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B, T, d)
        h = h + a @ W[p + "SelfAttention.o.weight"].T
        # ours self-attn
        nn_ = ops.layernorm(hh, Wh[p + "layer_norm.weight"], None, 1e-6, kind=1)
        qkv = torch.empty((B * T, 3 * d), dtype=dt, device=dev)
        ops.linear(nn_, Wh[p + "SelfAttention.q.weight"], out=qkv[:, :d]); ops.linear(nn_, Wh[p + "SelfAttention.k.weight"], out=qkv[:, d:2*d]); ops.linear(nn_, Wh[p + "SelfAttention.v.weight"], out=qkv[:, 2*d:])
        ctx = ops.attention(qkv, 0, qkv, d, qkv, 2 * d, B, H, T, T, bias_delta=bias, scale=1.0, causal_value=-10000.0)
        print(f"layer {L_} self-attn ctx err", float((ctx.float().view(B, T, d) - a).abs().max()))
        hh = ops.linear(ctx, Wh[p + "SelfAttention.o.weight"], None, residual=hh, epilogue=ops.EPI_RESIDUAL)
        print(f"layer {L_} after self-attn err", float((hh.float().view(B, T, d) - h).abs().max()))
        p = f"decoder.block.{L_}.layer.1."
        n = rms(h, W[p + "layer_norm.weight"])
        q = heads(n @ W[p + "EncDecAttention.q.weight"].T, T)
        k = (encf @ W[p + "EncDecAttention.k.weight"].T).view(B, Lk, H, 64).permute(0, 2, 1, 3)
        v = (encf @ W[p + "EncDecAttention.v.weight"].T).view(B, Lk, H, 64).permute(0, 2, 1, 3)
        s = q @ k.transpose(-1, -2) + cross_mask[:, None, None, :]
        a = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B, T, d)
        h = h + a @ W[p + "EncDecAttention.o.weight"].T
        nn_ = ops.layernorm(hh, Wh[p + "layer_norm.weight"], None, 1e-6, kind=1)
        qq = ops.linear(nn_, Wh[p + "EncDecAttention.q.weight"])
        kv = torch.empty((B * Lk, 2 * d), dtype=dt, device=dev)
        flat = enc.reshape(-1, d)
        ops.linear(flat, Wh[p + "EncDecAttention.k.weight"], out=kv[:, :d]); ops.linear(flat, Wh[p + "EncDecAttention.v.weight"], out=kv[:, d:])
        print(f"layer {L_} cross k proj err", float((kv[:, :d].float().view(B, Lk, H, 64).permute(0, 2, 1, 3) - k).abs().max()))
        split = next(s_ for s_ in range(min(512, Lk), 0, -1) if Lk % s_ == 0)
        ctx = ops.cross_attention_split(qq, 0, kv, 0, d, B, H, T, Lk, add_mask=cross_mask, scale=1.0, split=split)
        print(f"layer {L_} cross ctx err (split {split})", float((ctx.float().view(B, T, d) - a).abs().max()))
        hh = ops.linear(ctx, Wh[p + "EncDecAttention.o.weight"], None, residual=hh, epilogue=ops.EPI_RESIDUAL)
        p = f"decoder.block.{L_}.layer.2."
        n = rms(h, W[p + "layer_norm.weight"])
        ff = torch.nn.functional.gelu(n @ W[p + "DenseReluDense.wi_0.weight"].T, approximate="tanh") * (n @ W[p + "DenseReluDense.wi_1.weight"].T)
        h = h + ff @ W[p + "DenseReluDense.wo.weight"].T
        hh = model._residual(model._ff_in(Wh, G, p, hh), Wh[p + "DenseReluDense.wo.weight"], hh)
        print(f"layer {L_} after FF err", float((hh.float().view(B, T, d) - h).abs().max()))
    h = rms(h, W["decoder.final_layer_norm.weight"])
    logits_ref = h @ W["lm_head.weight"].T
    lg = model.decode(dec_in, enc, mask.view(B, -1))
    print("logits: ours vs inline-ref", float((lg.float() - logits_ref).abs().max()), " inline-ref vs golden", float((logits_ref.cpu() - torch.from_numpy(g["logits_fp32"])).abs().max()))
