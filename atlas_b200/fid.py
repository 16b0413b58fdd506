"""Drop-in for `src.fid.FiD` (reference src/fid.py:28-357 over the vendored T5, src/modeling_t5.py; v1.1 and v1.0):
Fusion-in-Decoder on B200 kernels: the no-grad forward (evaluation / scoring / greedy generation, replayed from a
CUDA graph), the with-grad forward + hand-written backward kernels of the training step (`_forward_train`, grad_ops.py),
and the cross-attention score capture used for retriever distillation (src/fid.py:126-235,333-343).

Surface kept: `FiD(config)`, `forward(input_ids [B, n*L], attention_mask, decoder_input_ids,
labels, encoder_outputs=None, use_cache=False)` -> output indexable as `out[0]` = loss, `out[1]` = logits with
`.logits`, `.loss`, `.encoder_last_hidden_state`; `encoder.config.{n_context,bsz}` are read like the reference's
`FiDStack` (src/fid.py:47-49,66-76); `_shift_right`; `generate` (greedy); parameter names identical to HF T5
(`shared`, `encoder.block.N.layer.0.SelfAttention.{q,k,v,o}`, `relative_attention_bias` on block 0,
`layer.1.EncDecAttention`, `DenseReluDense.{wi_0,wi_1,wo}` (v1.1) or `DenseReluDense.{wi,wo}` (v1.0), `lm_head`) so
reference checkpoints load.  T5 v1.0 (t5-small / -base / -large: `feed_forward_proj="relu"`, LM head tied to `shared` and
applied to the final hidden state scaled by d_model^-0.5) runs the same kernels with the ReLU fused into the wi GEMM.

What runs where (all in csrc/): RMSNorm (T5LayerNorm, modeling_t5.py:244-253); q/k/v/o and FF projections on the
wgmma GEMM with fused residual, gated-GELU and ReLU epilogues (modeling_t5.py:256-289); encoder self-attention as
B*n independent L-token segments with the relative-position bias added on the fly from a [H, 2L-1] table
(modeling_t5.py:352-416,478-524) - the [B*n, H, L, L] bias / probability tensors are never materialised;
decoder cross-attention over the n*L concatenated keys as split-KV + combine (fid.py:298-349).
Dropout: counter-based masks inside the kernels (csrc/dropout.cuh).  The fp16 `isinf` clamps of every sub-layer
(modeling_t5.py:657-708, three host syncs per block in the reference) are decided on the device (ops.clamp_inf_).
"""
import copy
import math
import os
from types import SimpleNamespace

import torch
from torch import nn

from . import grad_ops, ops
from ._lib import AtlasB200Error
from .retrievers import HalfCache


class T5ConfigLite(SimpleNamespace):
    """The T5Config fields this path reads (defaults = google/t5-base-lm-adapt, i.e. T5 v1.1 base)."""

    def __init__(self, **kw):
        d = dict(vocab_size=32128, d_model=768, d_kv=64, d_ff=2048, num_layers=12, num_decoder_layers=12, num_heads=12,
                 relative_attention_num_buckets=32, layer_norm_epsilon=1e-6, feed_forward_proj="gated-gelu",
                 tie_word_embeddings=False, decoder_start_token_id=0, pad_token_id=0, eos_token_id=1)
        d.update(kw)
        super().__init__(**d)


class _Norm(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d))


class _Attn(nn.Module):
    def __init__(self, c, has_bias):
        super().__init__()
        inner = c.num_heads * c.d_kv
        self.q = nn.Linear(c.d_model, inner, bias=False)
        self.k = nn.Linear(c.d_model, inner, bias=False)
        self.v = nn.Linear(c.d_model, inner, bias=False)
        self.o = nn.Linear(inner, c.d_model, bias=False)
        if has_bias:
            self.relative_attention_bias = nn.Embedding(c.relative_attention_num_buckets, c.num_heads)


class _SelfAttnLayer(nn.Module):
    def __init__(self, c, has_bias):
        super().__init__()
        self.SelfAttention = _Attn(c, has_bias)
        self.layer_norm = _Norm(c.d_model)


class _CrossAttnLayer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.EncDecAttention = _Attn(c, False)
        self.layer_norm = _Norm(c.d_model)


class _FF(nn.Module):
    """T5DenseGatedGeluDense (wi_0, wi_1, wo) or, for feed_forward_proj="relu", T5DenseReluDense (wi, wo)."""

    def __init__(self, c):
        super().__init__()
        if c.feed_forward_proj == "relu":
            self.wi = nn.Linear(c.d_model, c.d_ff, bias=False)
        else:
            self.wi_0 = nn.Linear(c.d_model, c.d_ff, bias=False)
            self.wi_1 = nn.Linear(c.d_model, c.d_ff, bias=False)
        self.wo = nn.Linear(c.d_ff, c.d_model, bias=False)


class _FFLayer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.DenseReluDense = _FF(c)
        self.layer_norm = _Norm(c.d_model)


class _Block(nn.Module):
    def __init__(self, c, is_decoder, has_bias):
        super().__init__()
        layers = [_SelfAttnLayer(c, has_bias)]
        if is_decoder:
            layers.append(_CrossAttnLayer(c))
        layers.append(_FFLayer(c))
        self.layer = nn.ModuleList(layers)


class FiDStack(nn.Module):
    def __init__(self, config, embed_tokens, is_decoder):
        super().__init__()
        self.config = copy.copy(config)
        self.config.is_decoder = is_decoder
        self.is_decoder = is_decoder
        self.embed_tokens = embed_tokens
        n = config.num_decoder_layers if is_decoder else config.num_layers
        self.block = nn.ModuleList([_Block(config, is_decoder, i == 0) for i in range(n)])
        self.final_layer_norm = _Norm(config.d_model)


def relative_position_bucket(relative_position, bidirectional=True, num_buckets=32, max_distance=128):
    """T5's bucket function restated with the same torch ops and rounding as src/modeling_t5.py:352-397."""
    relative_buckets = 0
    if bidirectional:
        num_buckets //= 2
        relative_buckets += (relative_position > 0).to(torch.long) * num_buckets
        relative_position = torch.abs(relative_position)
    else:
        relative_position = -torch.min(relative_position, torch.zeros_like(relative_position))
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    if_large = max_exact + (
        torch.log(relative_position.float() / max_exact) / math.log(max_distance / max_exact) * (num_buckets - max_exact)
    ).to(torch.long)
    if_large = torch.min(if_large, torch.full_like(if_large, num_buckets - 1))
    relative_buckets += torch.where(is_small, relative_position, if_large)
    return relative_buckets


def bias_by_delta(weight, lq, lk, bidirectional, num_buckets):
    """[H, lq+lk-1] fp32 table: entry (j - i) + (lq - 1) holds the head's bias for key j / query i
    (`compute_bias`, src/modeling_t5.py:399-416, indexed by offset instead of a [lq, lk] matrix)."""
    delta = torch.arange(-(lq - 1), lk, device=weight.device, dtype=torch.long)
    buckets = relative_position_bucket(delta, bidirectional=bidirectional, num_buckets=num_buckets)
    return weight[buckets].t().float().contiguous()


def _capture(fn):
    """(CUDA graph of `fn()`, what the captured call returned), after one eager warm-up call on a side stream (lazy kernel
    attributes, allocator, weight caches).  The warm-up really runs: state it writes is the caller's to reset."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    return graph, out


class _GraphRunner:
    """One captured CUDA graph of a static-shape function of device tensors.  Every kernel of this package is
    launched through the C ABI on `torch.cuda.current_stream()`, so capturing the whole forward removes the ~150
    host launches of the decoder stack (launch-bound at T = 32 target tokens) from the critical path."""

    def __init__(self, fn, example_inputs):
        self.static_in = [t.clone() for t in example_inputs]
        self.graph, self.static_out = _capture(lambda: fn(*self.static_in))

    def __call__(self, *inputs):
        for dst, src in zip(self.static_in, inputs):
            dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_out


def _check_passage_length(L):
    if L > ops.ATTENTION_LONG_MAX_LK:
        raise AtlasB200Error(f"text_maxlength = {L} is not supported: the encoder self-attention takes passages of at most "
                             f"{ops.ATTENTION_LONG_MAX_LK} tokens")


def _cross_split(Lk, dropout=False, force_pad=False):
    """(split, Lk_pad): key segment and padded key range of the split-KV cross-attention over Lk keys.

    Segments: the largest divisor of Lk up to 384 keys, else up to 512 (the attention kernel keeps a whole segment's K / V
    in shared memory).  dropout: the training forward's dropout mask is addressed in 32-key groups (csrc/dropout.cuh), so a
    multiple of 32 in [64, 512] comes first.  Lk_pad = Lk then.
    A key range without such a divisor (Lk > 512 with none in [64, 512]; with dropout, none that is a multiple of 32) is
    padded instead: ceil(Lk / 384) segments (one up to 512 keys) of equal length rounded up to a multiple of 64, so
    Lk_pad - Lk < 384 dead keys (< 64 up to 512 keys), which _pad_keys / _cross_mask add and mask.
    force_pad: the padded plan even where a divisor exists (tests)."""
    if not force_pad:
        split = None
        if dropout:
            split = next((s for s in range(min(512, Lk) // 32 * 32, 63, -32) if Lk % s == 0), None)
        split = split or next((s for s in range(min(384, Lk), 63, -1) if Lk % s == 0), None) or \
            next(s for s in range(min(512, Lk), 0, -1) if Lk % s == 0)
        if (split >= 64 or Lk <= 512) and (not dropout or split % 32 == 0 or split == Lk):
            return split, Lk
    n = 1 if Lk <= 512 else -(-Lk // 384)
    split = (-(-Lk // n) + 63) // 64 * 64
    return split, n * split


def _pad_keys(x, B, Lk, Lk_pad):
    """[B * Lk, C] rows -> [B * Lk_pad, C]: each batch element's Lk rows followed by Lk_pad - Lk zero rows (x itself when
    Lk_pad == Lk).  Differentiable: the backward is the slice of the real rows."""
    if Lk_pad == Lk:
        return x
    return torch.nn.functional.pad(x.reshape(B, Lk, -1), (0, 0, 0, Lk_pad - Lk)).reshape(B * Lk_pad, -1)


def _cross_mask(enc_mask, B, Lk, dt, Lk_pad=None):
    """The additive cross-attention mask [B, Lk] fp32 of `invert_attention_mask` (4.18): -1e4 for fp16, -1e9 otherwise
    (src/modeling_t5.py:950).  Lk_pad: extended to [B, Lk_pad] with twice that value on the pad keys, so that they weigh
    exactly 0 even next to a batch element whose real keys are all masked."""
    neg = -1e4 if dt == torch.float16 else -1e9
    m = (1.0 - enc_mask.reshape(B, Lk).to(torch.float32)) * neg
    if Lk_pad is not None and Lk_pad != Lk:
        m = torch.nn.functional.pad(m, (0, Lk_pad - Lk), value=2.0 * neg)
    return m


def _norm_sums(n_sub, M, device, fused):
    """Row sums of squares for a stack of n_sub normed sub-layers of M rows (fused RMSNorm, see _norm_in): entry j is what
    sub-layer j's norm reads, entry j + 1 what its residual GEMM writes.  Entry 0 (the first norm has no producing GEMM) and
    every entry of an unfused stack are None: that norm runs as a kernel."""
    if not fused:
        return [None] * (n_sub + 1)
    return [None] + list(torch.zeros((n_sub, M), dtype=torch.float32, device=device).unbind(0))


class FiDOutput(tuple):
    """(loss, logits, encoder_last_hidden_state) with the attribute names Atlas reads (src/atlas.py:292-300,583-590)."""

    def __new__(cls, loss, logits, enc):
        o = super().__new__(cls, (loss, logits, enc))
        o.loss, o.logits, o.encoder_last_hidden_state = loss, logits, enc
        return o


class FiD(nn.Module):
    def __init__(self, config=None):
        super().__init__()
        config = config or T5ConfigLite()
        if config.d_kv != 64:
            raise AtlasB200Error(f"head dimension d_kv = {config.d_kv} is not implemented: the attention kernels need d_kv = 64 "
                                 "(t5-small / -base / -large and every T5 v1.1 size; t5-3b and t5-11b have d_kv = 128)")
        if not hasattr(config, "feed_forward_proj"):
            config.feed_forward_proj = "gated-gelu"
        if config.feed_forward_proj not in ("gated-gelu", "relu"):
            raise AtlasB200Error(f"feed_forward_proj={config.feed_forward_proj!r} is not implemented (gated-gelu: T5 v1.1, "
                                 "relu: T5 v1.0)")
        self.config = config
        self.model_dim = config.d_model
        self.shared = nn.Embedding(config.vocab_size, config.d_model)
        self.encoder = FiDStack(config, self.shared, is_decoder=False)
        self.decoder = FiDStack(config, self.shared, is_decoder=True)
        self.lm_head = nn.Linear(config.d_model, config.vocab_size, bias=False)
        if getattr(config, "tie_word_embeddings", False):
            self.lm_head.weight = self.shared.weight            # T5 v1.0: one table for the embedding and the LM head
        self.encoder.config.n_context = 1
        self.encoder.config.bsz = 1
        self._half = HalfCache()
        # CUDA-graph replay of the static-shape forward (eval / scoring); ATLAS_B200_CUDA_GRAPH=0 or
        # `model.cuda_graphs = False` runs every kernel launch eagerly (needed under profilers' event bracketing)
        self.cuda_graphs = os.environ.get("ATLAS_B200_CUDA_GRAPH", "1") != "0"
        self.fuse_norm = os.environ.get("ATLAS_B200_FUSE_NORM", "1") != "0"   # RMSNorm folded into the encoder GEMMs
        self._graphs = {}

    @classmethod
    def from_pretrained(cls, path, **kw):
        """Local HF-layout directory (config.json + weights) of a T5 checkpoint, src/model_io.py:77.  A config.json without
        `feed_forward_proj` (the original t5-small / -base / -large) is read as T5 v1.0 when the weights hold
        `DenseReluDense.wi` instead of `wi_0` / `wi_1`: ReLU feed-forward and, unless stated, a tied LM head
        (transformers' defaults for those fields)."""
        from ._pretrained import load_pretrained

        def infer(raw, sd):
            if "feed_forward_proj" in raw or not any(k.endswith("DenseReluDense.wi.weight") for k in sd):
                return {}
            return {"feed_forward_proj": "relu", "tie_word_embeddings": raw.get("tie_word_embeddings", True)}

        return load_pretrained(cls, T5ConfigLite, path, infer_config=infer, **kw)

    # ---- reference surface that is configuration only -------------------------------------
    def set_checkpoint(self, use_checkpoint):
        pass

    def gradient_checkpointing_enable(self):
        """Recompute each block in the backward instead of keeping its activations (torch.utils.checkpoint around the
        autograd Functions of grad_ops.py), `--use_gradient_checkpoint_reader` (src/model_io.py:86-87)."""
        self._grad_ckpt = True

    def gradient_checkpointing_disable(self):
        self._grad_ckpt = False

    # ---- cross-attention score capture (src/fid.py:126-235,333-343) -------------------------------------
    def reset_score_storage(self):
        self._xattn = []

    def overwrite_forward_crossattention(self):
        """From now on every forward also records, per decoder layer, the head-means of the cross-attention logits,
        probabilities and ||V||-weighted probabilities (src/model_io.py:79-81 calls this for the eval* / std* gold score
        modes and `compute_crossattention_stats`).  The recording forward runs eagerly (no CUDA graph)."""
        self._capture = True

    def create_crossattention_storage(self):
        self._xattn = []

    def _record_xattn(self, q, kv, B, H, T, Lk, lse, mask, layer=None, keys=None):
        """Keep ONE record per decoder layer, overwritten by every forward (the reference keeps one buffer per attention
        module, src/fid.py:333-343): constant memory however many forwards run between two `reset_score_storage()` calls.
        The statistics kernel takes at most 128 target tokens: longer targets run as 128-token slices of q and lse
        (every row's statistics depend on its own query only).  keys: the real keys of a padded range of Lk (_cross_split),
        the records keep those."""
        if getattr(self, "_capture", False):
            n = self.config.num_decoder_layers
            if not isinstance(getattr(self, "_xattn", None), list):
                self._xattn = []
            q, kv = q.detach(), kv.detach()
            parts = []
            for t0 in range(0, T, 128):
                t = min(128, T - t0)
                qs = q if t == T else q.view(B, T, -1)[:, t0:t0 + t].reshape(B * t, -1)
                parts.append(ops.cross_attention_stats(qs, 0, kv, 0, H * 64, B, H, t, Lk, lse[:, :, t0:t0 + t],
                                                       add_mask=mask, scale=1.0))
            rec = parts[0] if len(parts) == 1 else tuple(torch.cat(r, 1) for r in zip(*parts))
            if keys is not None and keys != Lk:
                rec = tuple(r[..., :keys] for r in rec)
            if layer is None:                       # sequential recording: a new forward starts after n records
                if len(self._xattn) >= n:
                    self._xattn = []
                self._xattn.append(rec)
            else:
                if len(self._xattn) != n:
                    self._xattn = [None] * n
                self._xattn[layer] = rec

    @torch.no_grad()
    def get_crossattention_scores(self, n_passages, mask, labels, ids, mode="all", mask_query=None):
        """One scalar per (query, passage) from the recorded cross-attention maps: `FiD.get_crossattention_scores`
        (src/fid.py:136-164) -> dict of [B, n_passages] tensors named {scores,probs,norms}{top5,top10,top20,nosep,first,
        sum,avg,woquery}."""
        rec = getattr(self, "_xattn", None)
        if not rec or len(rec) < self.config.num_decoder_layers or any(r is None for r in rec):
            raise AtlasB200Error("get_crossattention_scores: no recorded forward (call overwrite_forward_crossattention() "
                                 "and run a forward first)")
        rec = rec[-self.config.num_decoder_layers:]
        output = {}
        for idx, prefix in ((0, "scores"), (2, "norms"), (1, "probs")):
            if prefix in mode or "all" in mode:
                self.aggregate_value(torch.stack([r[idx] for r in rec]), mask, labels, n_passages, ids, mask_query, output,
                                     prefix=prefix)
        return output

    def aggregate_value(self, scores, mask, labels, n_passages, ids, mask_query=None, output=None, prefix=""):
        """src/fid.py:166-203, same reductions and the same (hard-coded 256) normalisers."""
        output = {} if output is None else output
        n_layers, bsz, n_tokens, _ = scores.size()
        ids = ids.view(bsz, n_passages, -1)
        scores = scores.view(n_layers, bsz, n_tokens, n_passages, -1)
        mask = mask.view(bsz, n_passages, -1).bool()
        scores = scores.masked_fill(~mask[None, :, None], 0.0)
        valid = ~(labels == -100)
        ntokens_sum = 256 * n_layers * valid.sum(dim=[1])[:, None]
        ntokens_wquery = mask.sum(dim=[2]) * n_layers * valid.sum(dim=[1])[:, None]
        ntokens_first = mask.sum(dim=[2]) * n_layers
        scores = scores.sum(dim=[0])
        for k in (5, 10, 20):
            output[f"{prefix}top{k}"] = self.get_topk_score(k, scores, mask, labels, n_layers)
        scores = scores.masked_fill((labels == -100)[:, :, None, None], 0.0)
        scores_wquery = scores.sum(dim=[1, 3])
        output[f"{prefix}nosep"] = scores.masked_fill(~(ids == 1)[:, None], 0).sum(dim=[1, 3]) / ntokens_sum
        output[f"{prefix}first"] = scores[:, 0].sum(dim=[2]) / ntokens_first
        output[f"{prefix}sum"] = scores_wquery / ntokens_sum
        output[f"{prefix}avg"] = scores_wquery / ntokens_wquery
        if mask_query is not None:
            output[f"{prefix}woquery"] = self.get_woquery_score(scores, mask_query, mask, labels, n_layers)
        return output

    def get_topk_score(self, topk, scores, mask, labels, n_layers):   # src/fid.py:205-210
        top = torch.topk(scores, k=topk, dim=-1)[0].sum(dim=[3])
        top = top.masked_fill((labels == -100)[:, :, None], 0.0)
        ntokens_top = n_layers * (~(labels == -100)).sum(dim=[1])[:, None]
        return top.sum(dim=1) / (topk * ntokens_top)

    def get_woquery_score(self, scores, mask_query, mask, labels, n_layers):   # src/fid.py:212-224
        if scores.size(-1) > mask_query.size(-1):
            pad = torch.zeros([mask_query.size(0), scores.size(-1) - mask_query.size(-1)], device=mask_query.device,
                              dtype=torch.bool)
            mask_query = torch.cat([mask_query, pad], dim=-1)
        mq = mask * (~mask_query[:, None])
        woq = scores.masked_fill(~mq[:, None], 0.0)
        ntokens_woquery = 256 * n_layers * (~(labels == -100)).sum(dim=[1])[:, None]
        return woq.sum(dim=[1, 3]) / ntokens_woquery

    def _shift_right(self, input_ids):  # src/modeling_t5.py:789-813
        start, pad = self.config.decoder_start_token_id, self.config.pad_token_id
        shifted = input_ids.new_zeros(input_ids.shape)
        shifted[..., 1:] = input_ids[..., :-1].clone()
        shifted[..., 0] = start
        shifted.masked_fill_(shifted == -100, pad)
        return shifted

    # ---- weights ---------------------------------------------------------------------------
    def _dtype(self):
        d = self.shared.weight.dtype
        return d if d in (torch.float16, torch.bfloat16) else torch.bfloat16

    def _weights(self):
        dt = self._dtype()
        W = self._half.get(self, dt)
        return W, self._half.derived(dt, self._fuse), dt

    @staticmethod
    def _head(W):
        """The LM-head matrix: `lm_head.weight`, or `shared.weight` when the two are tied (named_parameters() lists a tied
        parameter once, under its first name)."""
        return W["lm_head.weight"] if "lm_head.weight" in W else W["shared.weight"]

    @staticmethod
    def _concat_weights(W):
        """The concatenated weights the kernels read, by name: the rows of wi_0 and wi_1 interleaved (wi_0[j], wi_1[j]) for the
        gated-GELU GEMM epilogue ("...DenseReluDense.wi_01"); one [3*H*64, d] q|k|v projection whose single GEMM writes the
        [tokens, q|k|v] buffer the attention reads ("...SelfAttention.qkv"); the cross-attention k|v ("...EncDecAttention.kv").
        Built from W with differentiable ops only."""
        g = {}
        for name in W:
            if name.endswith("DenseReluDense.wi_0.weight"):
                w0, w1 = W[name], W[name.replace("wi_0", "wi_1")]
                g[name.replace("wi_0.weight", "wi_01")] = torch.stack([w0, w1], dim=1).reshape(-1, w0.shape[1])
            elif name.endswith("SelfAttention.q.weight"):
                g[name.replace("q.weight", "qkv")] = torch.cat(
                    [W[name], W[name.replace("q.weight", "k.weight")], W[name.replace("q.weight", "v.weight")]], 0)
            elif name.endswith("EncDecAttention.k.weight"):
                g[name.replace("k.weight", "kv")] = torch.cat([W[name], W[name.replace("k.weight", "v.weight")]], 0)
        return g

    # the projections that read a normalised hidden state, by the suffix of their weight's name in W or _concat_weights
    _NORMED_INPUTS = ("SelfAttention.qkv", "EncDecAttention.q.weight", "DenseReluDense.wi_01", "DenseReluDense.wi.weight")

    @staticmethod
    def _fuse(W):
        """Weights derived once per parameter version: `_concat_weights`, and for the fused norm every projection behind an
        RMSNorm again with the norm weight folded in (W'[n, k] = W[n, k] * ln[k]), named with a "_n" suffix."""
        g = {name: w.contiguous() for name, w in FiD._concat_weights(W).items()}
        for name, w in list(W.items()) + list(g.items()):
            sub = next((s for s in FiD._NORMED_INPUTS if name.endswith(s)), None)
            if sub is not None:
                ln = W[name[: -len(sub)] + "layer_norm.weight"]
                g[name + "_n"] = (w.float() * ln.float()[None, :]).to(w.dtype).contiguous()
        return g

    # ---- the sub-layers of the no-grad forward -------------------------------------------------
    def _norm_in(self, W, G, p, name, x, ss=None, rows=None, **kw):
        """RMSNorm of x with the norm weight of layer prefix p, then the projection p + name (a weight of G or W) on
        ops.linear (kw: its epilogue / out).  ss None: the norm runs as a kernel.  ss given, the norm fused: x is the
        UN-normalised hidden state and ss its rows' sums of squares; the GEMM reads the matrix with the norm weight folded in
        (_fuse) and scales its accumulator rows by rsqrt(ss / d + eps), so the normalised rows are never written or read."""
        eps = self.config.layer_norm_epsilon
        if ss is not None:
            return ops.linear(x, G[p + name + "_n"], row_ss=ss, rs_eps=eps, rows=rows, **kw)
        n = ops.layernorm(x, W[p + "layer_norm.weight"], None, eps, kind=1)
        return ops.linear(n, G[p + name] if p + name in G else W[p + name], rows=rows, **kw)

    def _ff_in(self, W, G, p, x, ss=None, rows=None):
        """The feed-forward's normed input GEMM with its activation in the epilogue: ReLU on wi (T5 v1.0) or the gated GELU
        on the interleaved wi_0 | wi_1 (v1.1)."""
        if self.config.feed_forward_proj == "relu":
            return self._norm_in(W, G, p, "DenseReluDense.wi.weight", x, ss, rows, epilogue=ops.EPI_RELU)
        return self._norm_in(W, G, p, "DenseReluDense.wi_01", x, ss, rows, epilogue=ops.EPI_GATED)

    @staticmethod
    def _residual(x, w, h, ss=None, rows=None):
        """h + x @ w.T in the GEMM's epilogue, then the fp16 overflow clamp the reference applies after every sub-layer
        (src/modeling_t5.py:657-708; no-op in bf16).  ss: receives the sums of squares of the new rows (fused norm)."""
        h = ops.linear(x, w, None, residual=h, epilogue=ops.EPI_RESIDUAL, out_ss=ss, rows=rows)
        return ops.clamp_inf_(h, row_ss=ss, rows=rows)

    def _decoder_block(self, W, G, i, h, self_attn, cross_attn, ss, qkv=None):
        """Decoder block i on the rows h: self_attn(qkv, i) and cross_attn(q, i) return the attention context.  ss: the
        block's four entries of _norm_sums.  qkv: the buffer the q|k|v projection writes (None: a new one)."""
        p = f"decoder.block.{i}.layer."
        qkv = self._norm_in(W, G, p + "0.", "SelfAttention.qkv", h, ss[0], out=qkv)
        h = self._residual(self_attn(qkv, i), W[p + "0.SelfAttention.o.weight"], h, ss[1])
        q = self._norm_in(W, G, p + "1.", "EncDecAttention.q.weight", h, ss[1])
        h = self._residual(cross_attn(q, i), W[p + "1.EncDecAttention.o.weight"], h, ss[2])
        g = self._ff_in(W, G, p + "2.", h, ss[2])
        return self._residual(g, W[p + "2.DenseReluDense.wo.weight"], h, ss[3])

    def _lm_head(self, W, h, dt):
        """Final norm, T5 v1.0's d_model^-0.5 rescale of a tied head (src/modeling_t5.py:1642-1645), LM head."""
        c = self.config
        h = ops.layernorm(h, W["decoder.final_layer_norm.weight"], None, c.layer_norm_epsilon, kind=1)
        if getattr(c, "tie_word_embeddings", False):
            h = (h.float() * (c.d_model ** -0.5)).to(dt)
        return ops.linear(h, self._head(W))

    @torch.no_grad()
    def encode(self, input_ids, attention_mask):
        """FiDStack encoder (src/fid.py:32-78): [B, n*L] -> each passage encoded independently -> [B, n*L, d]."""
        r = self._encode_rows(input_ids, attention_mask, packed=ops._ENC_PACKED)
        if isinstance(r, tuple):                    # packed rows -> the reference's padded layout (zeros at dropped tiles)
            r = ops.expand_packed_tiles(r[0], r[2])
        return r.view(self.encoder.config.bsz, -1, self.config.d_model)

    @torch.no_grad()
    def _encode_rows(self, input_ids, attention_mask, packed):
        """The encoder stack on a [rows, d] matrix.  packed=False (or a shape the packed path does not take): all S * L padded
        positions, returns the final hidden states [S * L, d].  packed=True: the PADDING-COMPACTED encoder - every passage keeps
        its 64-row tiles up to its last live key, packed back to back (ops.segment_tile_scan); the embedding, all projections
        (device-side row count, static launch shapes), the attention (ops.attention_packed) and the norms only see those rows.
        A padded position never influences a live one (its softmax weight is exactly 0; everything else is row-wise) and the
        cross-attention masks it, so logits, loss and generated tokens are those of the padded computation; the dropped rows
        of the returned encoder states read 0 instead of the reference's never-read values.  Returns (rows [S * L, d] of which
        the first *count are valid, keep uint8 [S, L / 64], tile_off int32 [S * L / 64], count int32 [1])."""
        c = self.config
        W, G, dt = self._weights()
        n_ctx = self.encoder.config.n_context
        ids = input_ids.reshape(input_ids.size(0) * n_ctx, -1)
        mask = attention_mask.reshape(attention_mask.size(0) * n_ctx, -1)
        S, L = ids.shape
        _check_passage_length(L)
        d, H = c.d_model, c.num_heads
        add_mask = (1.0 - mask.to(torch.float32)) * -10000.0                      # 4.18 get_extended_attention_mask
        # 64-key blocks made of padding only (every passage is padded to text_maxlength) weigh exactly 0 in the softmax:
        # the attention kernel skips them (ops.key_block_live), once per forward for all layers
        live = ops.key_block_live(add_mask)
        bias = bias_by_delta(W["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], L, L, True,
                             c.relative_attention_num_buckets)
        packed = packed and ops.encoder_packs(live, L)
        rows = None
        if packed:
            keep, tile_off, tile_src, rows = ops.segment_tile_scan(live)
            h = ops.embed_packed_tiles(ids, W["shared.weight"], tile_src)         # embedding gather of the kept tiles

            def attn(qkv):
                return ops.attention_packed(qkv, keep, tile_off, S, H, L, add_mask, bias, scale=1.0)
        else:
            h = W["shared.weight"][ids.reshape(-1)]                              # embedding gather, [S*L, d]

            fwd = ops.encoder_attention(L)

            def attn(qkv):
                return fwd(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=add_mask, bias_delta=bias, scale=1.0,
                           block_live=live)
        qkv = torch.empty((S * L, 3 * H * 64), dtype=dt, device=h.device)
        # fuse_norm: the RMSNorms fused around the GEMMs (_norm_in); only the very first and the final norm run as kernels,
        # 2 x num_layers normalised [tokens, d] tensors are never written or read
        ss = _norm_sums(2 * c.num_layers, S * L, h.device, self.fuse_norm)
        for i in range(c.num_layers):
            p = f"encoder.block.{i}.layer."
            self._norm_in(W, G, p + "0.", "SelfAttention.qkv", h, ss[2 * i], rows, out=qkv)
            h = self._residual(attn(qkv), W[p + "0.SelfAttention.o.weight"], h, ss[2 * i + 1], rows)
            g = self._ff_in(W, G, p + "1.", h, ss[2 * i + 1], rows)
            h = self._residual(g, W[p + "1.DenseReluDense.wo.weight"], h, ss[2 * i + 2], rows)
        h = ops.layernorm(h, W["encoder.final_layer_norm.weight"], None, c.layer_norm_epsilon, kind=1)
        return (h, keep, tile_off, rows) if packed else h

    # ---- decoder ---------------------------------------------------------------------------
    @torch.no_grad()
    def cross_kv(self, enc, out=None, sink=None):
        """K/V projections of the encoder output for every decoder layer ([B*n*L, 2*H*64] each), computed once
        per forward / per generation (the reference recomputes them every decoding step without use_cache).
        `out`: list of pre-allocated buffers (the static cross K|V cache of the decode graph).
        `sink(i, kv)`: instead, hand layer i's projection to `sink` as soon as it is computed; every layer is projected into
        ONE reused scratch buffer (peak memory: one layer), nothing is returned."""
        c = self.config
        W, G, dt = self._weights()
        flat = enc.reshape(-1, c.d_model)
        if flat.dtype != dt:
            flat = flat.to(dt)
        if sink is not None:
            scratch = None
            for i in range(c.num_decoder_layers):
                scratch = ops.linear(flat, G[f"decoder.block.{i}.layer.1.EncDecAttention.kv"], out=scratch)
                sink(i, scratch)
            return None
        return [ops.linear(flat, G[f"decoder.block.{i}.layer.1.EncDecAttention.kv"], out=None if out is None else out[i])
                for i in range(c.num_decoder_layers)]

    @torch.no_grad()
    def decode(self, decoder_input_ids, enc, enc_mask, cross_kv=None, enc_packed=None):
        """Decoder stack + LM head: [B, T] -> logits [B, T, vocab] (src/modeling_t5.py:875-1083,1619-1647).
        enc_packed: the tuple of `_encode_rows(packed=True)` that `enc` was expanded from - the cross K | V projections then
        read the packed rows directly.
        cross_kv: the per-layer `cross_kv` projections of the encoder rows padded (_pad_keys) to _cross_split's key range."""
        c = self.config
        W, G, dt = self._weights()
        B, T = decoder_input_ids.shape
        d, H = c.d_model, c.num_heads
        keys = enc.shape[1]
        split, Lk = _cross_split(keys)
        if cross_kv is None and Lk != keys and ops.cross_attention_streams(T, keys):
            Lk = keys                                         # the stream kernel takes the unpadded range
        if cross_kv is not None and cross_kv[0].shape[0] != B * Lk:
            raise AtlasB200Error(f"decode: cross_kv has {cross_kv[0].shape[0]} rows, the padded key range needs {B * Lk}")
        cross_mask = _cross_mask(enc_mask, B, keys, dt, Lk)
        if Lk != keys and cross_kv is None:
            # no usable split of the key range: every batch element's encoder rows are padded with masked zero rows once,
            # before the K | V projections
            enc = _pad_keys(enc.reshape(B * keys, d), B, keys, Lk).view(B, Lk, d)
            enc_packed = None
        cross_live = ops.key_block_live(cross_mask)           # padded 64-key tiles of the encoder output: skipped, once
        capture = getattr(self, "_capture", False)
        # Only the encoder positions inside a live 64-key tile are ever read by the cross-attention: project K | V for those
        # rows only (compacted, device-side row count: the shapes stay static for the CUDA graph).  At BASELINE configs[3]
        # the 12 K | V projections are 14 % of the step's FLOPs and ~36 % of their rows are padding-only tiles.
        compact = (cross_kv is None and cross_live is not None and not capture and ops._XKV_COMPACT and ops._XATTN_STREAM
                   and T <= 64 and Lk % 64 == 0 and Lk >= 1024)
        xkv = None
        if compact:
            if enc_packed is not None:
                # the encoder already ran on its kept tiles (a superset of the live ones, same tile order): project those rows
                enc_live, keep, tile_off, n_live_rows = enc_packed
                cross_live = keep.view(B, Lk // 64)
            else:
                flat = enc.reshape(-1, d)
                if flat.dtype != dt:
                    flat = flat.to(dt)
                enc_live, tile_off, n_live_rows = ops.compact_live_tiles(flat, cross_live)
            xkv = [ops.linear(enc_live, G[f"decoder.block.{i}.layer.1.EncDecAttention.kv"], rows=n_live_rows)
                   for i in range(c.num_decoder_layers)]
        elif cross_kv is None:
            cross_kv = self.cross_kv(enc)
        h = W["shared.weight"][decoder_input_ids.reshape(-1)]
        bias = bias_by_delta(W["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], T, T, False,
                             c.relative_attention_num_buckets)
        qkv = torch.empty((B * T, 3 * H * 64), dtype=dt, device=h.device)

        def self_attn(qkv, i):
            return ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, B, H, T, T, bias_delta=bias, scale=1.0,
                                 causal_value=-10000.0)

        def cross(q, i):
            if xkv is not None:
                return ops.cross_attention_stream_compact(q, xkv[i], cross_live, tile_off, B, H, T, Lk, cross_mask, scale=1.0)
            r = ops.cross_attention_split(q, 0, cross_kv[i], 0, H * 64, B, H, T, Lk, add_mask=cross_mask, scale=1.0,
                                          split=split, return_lse=capture, tile_live=cross_live)
            if not capture:
                return r
            self._record_xattn(q, cross_kv[i], B, H, T, Lk, r[1], cross_mask, layer=i, keys=keys)
            return r[0]

        # fuse_norm: the RMSNorms fused around the GEMMs like the encoder's; 3 x num_decoder_layers - 1 launches of a
        # ~150-launch dependent chain disappear.  The recording forward keeps the norm kernels.
        ss = _norm_sums(3 * c.num_decoder_layers, B * T, h.device, self.fuse_norm and not capture)
        for i in range(c.num_decoder_layers):
            h = self._decoder_block(W, G, i, h, self_attn, cross, ss[3 * i: 3 * i + 4], qkv)
        return self._lm_head(W, h, dt).view(B, T, -1)

    # ---- training path (autograd through the kernels, grad_ops.py) ---------------------------------------
    def _train_weights(self):
        """16-bit views of the live parameters built with DIFFERENTIABLE casts / concatenations, so that autograd routes
        the kernels' weight gradients back to the reference-named parameters (q / k / v, wi_0 / wi_1 ...)."""
        dt = self._dtype()
        W = {n: (p if p.dtype == dt else p.to(dt)) for n, p in self.named_parameters()}
        return W, self._concat_weights(W), dt

    def _check_trainable(self):
        return None

    def _embed_train(self, W, dt, ids):
        """The token embedding with autograd.  Tied (T5 v1.0): gathered from the parameter itself (cast to `dt` per row), so
        its fp32 scatter-add gradient reaches an fp32 `shared.weight` without a 16-bit rounding and is summed there with
        the LM head's weight gradient in fp32."""
        if "lm_head.weight" in W:
            return grad_ops.embedding(W["shared.weight"], ids)
        return grad_ops.embedding(self.shared.weight, ids, out_dtype=dt)

    def _ff_train(self, W, G, prefix, n):
        """wi -> activation of the feed-forward with autograd (the dropout and wo follow in the caller)."""
        p = prefix + "DenseReluDense."
        if self.config.feed_forward_proj == "relu":
            return grad_ops.linear_relu(n, W[p + "wi.weight"])
        return grad_ops.gated_gelu(grad_ops.linear(n, G[p + "wi_01"]))

    def _dropout_p(self):
        """config.dropout_rate in training mode (nn.Dropout / F.dropout of src/modeling_t5.py:266,286,310,515,561,597,
        964,1059), else 0: masks are generated inside the kernels and re-derived in the backward (csrc/dropout.cuh)."""
        return float(getattr(self.config, "dropout_rate", 0.0) or 0.0) if self.training else 0.0

    def _maybe_ckpt(self, fn, *args):
        if getattr(self, "_grad_ckpt", False):
            from torch.utils.checkpoint import checkpoint

            return checkpoint(fn, *args, use_reentrant=False)
        return fn(*args)

    def _encode_train(self, WG, input_ids, attention_mask):
        """`encode` with autograd (same kernels forward, un-fused norms; backward = grad_ops).  Where the padding-compacted
        encoder takes the shape (ops.encoder_packs, ops._ENC_PACKED), the stack runs on the packed rows like _encode_rows'
        and is expanded to the padded layout at the end: the loss and the gradients are the padded step's up to summation
        order (same dropout masks and draws of dropout keys), the fp16 overflow clamp sees the kept rows only."""
        g = grad_ops
        c = self.config
        W, G, dt = WG
        n_ctx, bsz = self.encoder.config.n_context, self.encoder.config.bsz
        ids = input_ids.reshape(input_ids.size(0) * n_ctx, -1)
        mask = attention_mask.reshape(attention_mask.size(0) * n_ctx, -1)
        S, L = ids.shape
        _check_passage_length(L)
        d, H = c.d_model, c.num_heads
        eps = c.layer_norm_epsilon
        pdrop = self._dropout_p()
        add_mask = (1.0 - mask.to(torch.float32)) * -10000.0
        live = ops.key_block_live(add_mask)
        add_mask._atlas_block_live = live     # read by grad_ops._SelfAttention (all layers share it)
        bias = bias_by_delta(W["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], L, L, True,
                             c.relative_attention_num_buckets)
        packed = ops._ENC_PACKED and ops.encoder_packs(live, L)
        row_tiles = None
        if packed:
            # the tables once per forward; the row count read to the host once (the step is eager and synchronises for the
            # loss anyway), so every GEMM, norm and weight gradient runs unchanged on [rows, d]
            keep, tile_off, tile_src, count = ops.segment_tile_scan(live)
            rows = int(count.item())
            row_tiles = tile_src[: rows // 64]                        # padded tile of every packed tile: dropout masks
            src = (row_tiles.long()[:, None] * 64 + torch.arange(64, device=ids.device)).reshape(-1)
            h = g.dropout(self._embed_train(W, dt, ids.reshape(-1)[src]), pdrop, row_tiles=row_tiles)

            def attention(qkv, bias):
                return g.packed_self_attention(qkv, keep, tile_off, S, H, L, add_mask, bias_delta=bias, scale=1.0,
                                               dropout_p=pdrop)
        else:
            h = g.dropout(self._embed_train(W, dt, ids), pdrop)

            def attention(qkv, bias):
                return g.self_attention(qkv, S, H, L, add_mask=add_mask, bias_delta=bias, scale=1.0, dropout_p=pdrop,
                                        long_segments=True)

        def lin_res(x, w, res):
            # h + dropout(linear(x)) (T5LayerSelfAttention / T5LayerFF); without dropout the add is the GEMM's epilogue;
            # then the fp16 overflow clamp of the block (a no-op for bf16)
            if pdrop:
                return g.clamp_inf(g.dropout(g.linear(x, w), pdrop, residual=res, row_tiles=row_tiles))
            return g.clamp_inf(g.linear(x, w, None, residual=res))

        def block(i, h, bias):
            p = f"encoder.block.{i}.layer.0."
            n = g.layernorm(h, W[p + "layer_norm.weight"], None, eps, kind=1)
            qkv = g.linear(n, G[p + "SelfAttention.qkv"])
            h = lin_res(attention(qkv, bias), W[p + "SelfAttention.o.weight"], h)
            p = f"encoder.block.{i}.layer.1."
            n = g.layernorm(h, W[p + "layer_norm.weight"], None, eps, kind=1)
            return lin_res(g.dropout(self._ff_train(W, G, p, n), pdrop, row_tiles=row_tiles), W[p + "DenseReluDense.wo.weight"],
                           h)

        for i in range(c.num_layers):
            h = self._maybe_ckpt(block, i, h, bias)
        h = g.dropout(g.layernorm(h, W["encoder.final_layer_norm.weight"], None, eps, kind=1), pdrop, row_tiles=row_tiles)
        if packed:
            h = g.expand_packed(h, keep, tile_off)       # zeros at the dropped tiles, which the cross-attention masks
        return h.view(bsz, -1, d)

    def _decode_train(self, WG, decoder_input_ids, enc, enc_mask):
        g = grad_ops
        c = self.config
        W, G, dt = WG
        B, T = decoder_input_ids.shape
        d, H = c.d_model, c.num_heads
        keys = enc.shape[1]
        eps = c.layer_norm_epsilon
        pdrop = self._dropout_p()
        split, Lk = _cross_split(keys, dropout=pdrop > 0)
        flat = enc.reshape(-1, d)
        if flat.dtype != dt:
            flat = flat.to(dt)
        # padded key range (_cross_split): masked zero rows once per forward; the dropout mask of a key depends on its
        # index only, so the real keys keep theirs
        flat = _pad_keys(flat, B, keys, Lk)
        h = g.dropout(self._embed_train(W, dt, decoder_input_ids), pdrop)

        def lin_res(x, w, res):
            if pdrop:
                return g.clamp_inf(g.dropout(g.linear(x, w), pdrop, residual=res))
            return g.clamp_inf(g.linear(x, w, None, residual=res))

        bias = bias_by_delta(W["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], T, T, False,
                             c.relative_attention_num_buckets)
        cross_mask = _cross_mask(enc_mask, B, keys, dt, Lk)
        cross_mask._atlas_block_live = ops.key_block_live(cross_mask)     # padded 64-key tiles: skipped forward and backward

        def block(i, h, bias, flat):
            p = f"decoder.block.{i}.layer.0."
            n = g.layernorm(h, W[p + "layer_norm.weight"], None, eps, kind=1)
            qkv = g.linear(n, G[p + "SelfAttention.qkv"])
            ctx = g.self_attention(qkv, B, H, T, bias_delta=bias, scale=1.0, causal_value=-10000.0, dropout_p=pdrop)
            h = lin_res(ctx, W[p + "SelfAttention.o.weight"], h)
            p = f"decoder.block.{i}.layer.1."
            n = g.layernorm(h, W[p + "layer_norm.weight"], None, eps, kind=1)
            q = g.linear(n, W[p + "EncDecAttention.q.weight"])
            kv = g.linear(flat, G[p + "EncDecAttention.kv"])
            ctx, lse = g.cross_attention(q, kv, B, H, T, Lk, add_mask=cross_mask, scale=1.0, split=split, return_lse=True,
                                         dropout_p=pdrop)
            self._record_xattn(q, kv, B, H, T, Lk, lse, cross_mask, layer=i, keys=keys)
            h = lin_res(ctx, W[p + "EncDecAttention.o.weight"], h)
            p = f"decoder.block.{i}.layer.2."
            n = g.layernorm(h, W[p + "layer_norm.weight"], None, eps, kind=1)
            return lin_res(g.dropout(self._ff_train(W, G, p, n), pdrop), W[p + "DenseReluDense.wo.weight"], h)

        for i in range(c.num_decoder_layers):
            h = self._maybe_ckpt(block, i, h, bias, flat)
        h = g.dropout(g.layernorm(h, W["decoder.final_layer_norm.weight"], None, eps, kind=1), pdrop)
        if getattr(c, "tie_word_embeddings", False):
            h = h * (d ** -0.5)                                      # src/modeling_t5.py:1642-1645
        logits = g.linear(h, self._head(W))
        return logits.view(B, T, -1)

    def _forward_train(self, input_ids, attention_mask, decoder_input_ids, labels, encoder_outputs):
        self._check_trainable()
        WG = self._train_weights()
        if encoder_outputs is not None:
            enc = encoder_outputs[0]
        else:
            enc = self._encode_train(WG, input_ids, attention_mask.to(torch.bool))
        B = enc.shape[0]
        logits = self._decode_train(WG, decoder_input_ids, enc, attention_mask.reshape(B, -1).to(torch.bool))
        loss = None
        pd = self.shared.weight.dtype
        if labels is not None:
            loss = grad_ops.cross_entropy(logits, labels).to(pd)      # CrossEntropyLoss(ignore_index=-100)
        if logits.dtype != pd:
            logits, enc = logits.to(pd), enc.to(pd)
        return FiDOutput(loss, logits, enc)

    # ---- CUDA-graph cache --------------------------------------------------------------------
    def _run(self, tag, fn, inputs):
        """Run `fn(*inputs)` (static shapes, device tensors in / out): replay a captured graph when enabled."""
        if not self.cuda_graphs or getattr(self, "_capture", False):   # recording forwards append to a python list
            return fn(*inputs)
        self._weights()                                      # make sure the 16-bit weight copies exist / are current
        dt = self._dtype()
        # the 16-bit weight buffers are refreshed in place (HalfCache): the graph key only holds their allocation generation
        key = (tag, dt, self.fuse_norm, ops._ENC_PACKED, self._half.sets[dt]["gen"],
               tuple((tuple(t.shape), t.dtype, t.device) for t in inputs))
        runner = self._graphs.get(key)
        if runner is None:
            if len(self._graphs) >= 8:                       # shapes changed often: drop the oldest graph + its pool
                self._graphs.pop(next(iter(self._graphs)))
            runner = _GraphRunner(fn, inputs)
            self._graphs[key] = runner
        out = runner(*inputs)
        # results live in the graph's static buffers: hand out copies
        return out.clone() if torch.is_tensor(out) else tuple(o.clone() for o in out)

    # ---- public forward / generate -----------------------------------------------------------
    def forward(self, input_ids=None, attention_mask=None, decoder_input_ids=None, labels=None, encoder_outputs=None,
                use_cache=False, **unused):
        if decoder_input_ids is None and labels is not None:
            decoder_input_ids = self._shift_right(labels)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # training step (train.py): the same kernels forward, autograd through grad_ops.py backward
            return self._forward_train(input_ids, attention_mask, decoder_input_ids, labels, encoder_outputs)
        if encoder_outputs is not None:
            enc = encoder_outputs[0]
            B = enc.shape[0]
            mask2 = attention_mask.reshape(B, -1)
            logits = self._run("dec", lambda e, m, d: self.decode(d, e, m), (enc, mask2.to(torch.bool), decoder_input_ids))
        else:
            n_ctx, bsz = self.encoder.config.n_context, self.encoder.config.bsz

            def full(ids, mask, dec):
                r = self._encode_rows(ids, mask, packed=ops._ENC_PACKED)
                packed = r if isinstance(r, tuple) else None
                e = (ops.expand_packed_tiles(r[0], r[2]) if packed else r).view(bsz, -1, self.config.d_model)
                return self.decode(dec, e, mask.reshape(e.shape[0], -1), enc_packed=packed), e

            logits, enc = self._run(("full", n_ctx, bsz), full,
                                    (input_ids, attention_mask.to(torch.bool), decoder_input_ids))
        loss = None
        if labels is not None:
            # CrossEntropyLoss(ignore_index=-100), src/modeling_t5.py:1650-1652
            loss = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.size(-1)).float(), labels.reshape(-1),
                                                     ignore_index=-100).to(logits.dtype)
        pd = self.shared.weight.dtype
        if logits.dtype != pd:
            logits, enc = logits.to(pd), enc.to(pd)
        return FiDOutput(loss, logits, enc)

    # ---- greedy generation: KV-cached single-token decode (csrc/decode.cu) ----------------------------------------
    class _DecodeState:
        """Static buffers of one (batch, keys, max_length, dtype) generation shape: per-layer self K|V caches, the cross
        K|V cache, the token / sequence / done / step tensors the step reads and writes on the device, and (optionally)
        the captured CUDA graph of ONE decode step that every step replays (the step index lives in device memory)."""

        def __init__(self, model, B, Lk, Tmax, dt, dev, xkv=None):
            c = model.config
            H, d = c.num_heads, c.d_model
            nl = c.num_decoder_layers
            self.B, self.Lk, self.Tmax = B, Lk, Tmax
            self.self_kv = [torch.zeros((B, Tmax, 2 * H * 64), dtype=dt, device=dev) for _ in range(nl)]
            self.cross_kv, self.cross_scale = FiD._cross_kv_buffers(B * Lk, H, nl, dt, dev, xkv)
            self.cross_mask = torch.zeros((B, Lk), dtype=torch.float32, device=dev)
            self.tok_in = torch.zeros(B, dtype=torch.int64, device=dev)
            self.seq = torch.zeros((B, Tmax), dtype=torch.int64, device=dev)
            self.done = torch.zeros(B, dtype=torch.uint8, device=dev)
            self.t_dev = torch.zeros(1, dtype=torch.int32, device=dev)
            self.logits = None
            self.graph = None
            self.cross_live = None

        def reset(self, start, pad):
            """greedy_search's start: every sequence holds the decoder start token, none is done."""
            self.seq.fill_(pad)
            self.seq[:, 0] = start
            self.tok_in.fill_(start)
            self.done.zero_()
            self.t_dev.zero_()

    @staticmethod
    def _cross_kv_buffers(rows, H, nl, dt, dev, xkv):
        """The cross K|V cache of a decode state: per layer [rows, 2*H*64] in the run's 16-bit dtype (xkv None), or for
        xkv == "fp8" the e4m3 codes uint8 [rows, 2*H*64] plus one fp32 scale per (row, 64-column block) [rows, 2*H]."""
        if xkv is None:
            return [torch.empty((rows, 2 * H * 64), dtype=dt, device=dev) for _ in range(nl)], None
        return ([torch.empty((rows, 2 * H * 64), dtype=torch.uint8, device=dev) for _ in range(nl)],
                [torch.empty((rows, 2 * H), dtype=torch.float32, device=dev) for _ in range(nl)])

    @torch.no_grad()
    def _decode_step_logits(self, st):
        """Decoder stack for ONE new token per sequence (`st.tok_in`, position `st.t_dev`) -> logits [B, vocab].
        Self-attention appends to / reads the per-layer K|V cache; cross-attention streams the cached cross K|V once."""
        c = self.config
        W, G, dt = self._weights()
        H = c.num_heads
        B, Lk = st.B, st.Lk
        nb = getattr(st, "nb", 1)           # beam search: B * nb rows, the nb beams of a batch element consecutive
        h = W["shared.weight"][st.tok_in]                                          # [B * nb, d]

        def self_attn(qkv, i):
            if nb > 1:      # history gathered through the beams' ancestry table: the cache is never reordered
                return ops.decode_self_attention_beam(qkv, st.self_kv[i], st.t_dev, st.anc, H, bias_delta=st.bias, scale=1.0)
            return ops.decode_self_attention(qkv, st.self_kv[i], st.t_dev, H, bias_delta=st.bias, scale=1.0)

        def cross(q, i):
            if st.cross_scale is not None:      # opt-in e4m3 cross K|V cache (cross_kv_dtype="fp8")
                if nb > 1:
                    return ops.decode_cross_attention_beams_e4m3(q, st.cross_kv[i], st.cross_scale[i], B, nb, H, Lk,
                                                                 st.cross_mask, st.chunk, tile_live=st.cross_live)
                return ops.decode_cross_attention_e4m3(q, st.cross_kv[i], st.cross_scale[i], B, H, Lk, add_mask=st.cross_mask,
                                                       scale=1.0, chunk=st.chunk, tile_live=st.cross_live)
            if nb > 1:      # the nb beams share their batch element's cross K | V, streamed once per step
                return ops.decode_cross_attention_beams(q, st.cross_kv[i], B, nb, H, Lk, st.cross_mask, st.chunk,
                                                        tile_live=st.cross_live)
            return ops.decode_cross_attention(q, st.cross_kv[i], B, H, Lk, add_mask=st.cross_mask, scale=1.0,
                                              chunk=st.chunk, tile_live=st.cross_live)

        for i in range(c.num_decoder_layers):       # the step keeps the norm kernels
            h = self._decoder_block(W, G, i, h, self_attn, cross, (None,) * 4)
        return self._lm_head(W, h, dt)

    class _BeamState:
        """Static buffers of one (batch, beams, keys, max_length, dtype) beam-search shape (csrc/beam.cu): the per-layer
        self K|V caches of the R = B * nb beam rows, ONE cross K|V per batch element, the ancestry and token tables, the beam
        scores and the hypothesis slots, all read and written on the device so that one captured graph serves every step."""

        def __init__(self, model, B, nb, Lk, Tmax, dt, dev, xkv=None):
            c = model.config
            H = c.num_heads
            nl = c.num_decoder_layers
            R = B * nb
            self.B, self.nb, self.R, self.Lk, self.Tmax = B, nb, R, Lk, Tmax
            self.self_kv = [torch.zeros((R, Tmax, 2 * H * 64), dtype=dt, device=dev) for _ in range(nl)]
            self.cross_kv, self.cross_scale = FiD._cross_kv_buffers(B * Lk, H, nl, dt, dev, xkv)
            self.cross_mask = torch.zeros((B, Lk), dtype=torch.float32, device=dev)
            self.tok_in = torch.zeros(R, dtype=torch.int64, device=dev)
            self.t_dev = torch.zeros(1, dtype=torch.int32, device=dev)
            self.anc = torch.zeros((2, R, Tmax), dtype=torch.int32, device=dev)
            self.tok = torch.zeros((R, Tmax), dtype=torch.int32, device=dev)
            self.parent = torch.zeros(R, dtype=torch.int32, device=dev)
            self.beam_scores = torch.zeros(R, dtype=torch.float32, device=dev)
            self.done = torch.zeros(B, dtype=torch.uint8, device=dev)
            self.hyp_score = torch.zeros((B, nb), dtype=torch.float64, device=dev)
            self.hyp_len = torch.zeros((B, nb), dtype=torch.int32, device=dev)
            self.hyp_ins = torch.zeros((B, nb), dtype=torch.int32, device=dev)
            self.hyp_tok = torch.zeros((B, nb, Tmax), dtype=torch.int32, device=dev)
            self.hyp_state = torch.zeros((B, 2), dtype=torch.int32, device=dev)
            self.hyp_worst = torch.zeros(B, dtype=torch.float64, device=dev)
            self.cand_score = torch.empty((R, 2 * nb), dtype=torch.float32, device=dev)
            self.cand_tok = torch.empty((R, 2 * nb), dtype=torch.int32, device=dev)
            self.graph = None
            self.cross_live = None

        def reset(self, start, pad):
            """beam_search's start: every row holds the decoder start token, beam 0 scores 0 and the others -1e9."""
            self.anc.copy_(torch.arange(self.R, dtype=torch.int32, device=self.anc.device)[None, :, None].expand_as(self.anc))
            self.tok.fill_(pad)
            self.tok[:, 0] = start
            self.tok_in.fill_(start)
            self.t_dev.zero_()
            self.done.zero_()
            self.beam_scores.fill_(-1e9)
            self.beam_scores.view(self.B, self.nb)[:, 0] = 0.0
            self.hyp_state.zero_()
            self.hyp_worst.fill_(1e9)

        def select_buffers(self):
            """The tensors ops.beam_select reads and writes, in its argument order."""
            return (self.beam_scores, self.tok_in, self.parent, self.done, self.anc, self.tok, self.t_dev, self.hyp_score,
                    self.hyp_len, self.hyp_ins, self.hyp_tok, self.hyp_state, self.hyp_worst)

        def sequences(self, t):
            """The rows' tokens at positions 0..t, gathered through the ancestry of step t -> int64 [R, t + 1]."""
            pos = torch.arange(t + 1, device=self.tok.device)
            return self.tok[self.anc[t & 1, :, : t + 1].long(), pos[None, :]].long()

    def _decode_state(self, B, Lk, Tmax, dt, dev, nb=1, xkv=None):
        key = (B, Lk, Tmax, dt, dev) if nb == 1 else (B, Lk, Tmax, dt, dev, nb)
        if xkv is not None:
            key = key + (xkv,)
        states = self.__dict__.setdefault("_decode_states", {})
        st = states.get(key)
        if st is None:
            if len(states) >= 2:
                states.pop(next(iter(states)))
            st = FiD._DecodeState(self, B, Lk, Tmax, dt, dev, xkv) if nb == 1 else \
                FiD._BeamState(self, B, nb, Lk, Tmax, dt, dev, xkv)
            # keys per block of the cross-attention sweep: ~4 blocks per SM keep every SM streaming
            st.chunk = 256 if Lk >= 2048 else 64
            states[key] = st
        return st

    def _prepare_decode(self, st, enc, attention_mask, W, dt):
        """Per generation: the cross K|V projections, the cross-attention mask and its live 64-key tiles, the self-attention
        bias table - all into the state's fixed buffers (a captured step graph reads them)."""
        c = self.config
        B, Lk = st.B, st.Lk
        if st.cross_scale is None:
            self.cross_kv(enc, out=st.cross_kv)
        else:
            # e4m3 cache: each layer's 16-bit projection (one reused scratch buffer) is quantized into the state's fixed
            # buffers (the captured step graph reads them)
            self.cross_kv(enc, sink=lambda i, kv: ops.quantize_kv_e4m3(kv, out=st.cross_kv[i], scale_out=st.cross_scale[i]))
        st.cross_mask.copy_(_cross_mask(attention_mask, B, Lk, dt))
        live = ops.key_block_live(st.cross_mask)              # padded 64-key tiles: not read by the decode steps
        if live is not None:
            if st.cross_live is None:
                st.cross_live = live                          # fixed buffer: the captured step graph reads it
            else:
                st.cross_live.copy_(live)
        wkey = (self._half.sets[dt]["gen"], self._half.sets[dt]["key"])
        if getattr(st, "wkey", None) != wkey:                                       # weights changed: the bias table is stale
            fresh = bias_by_delta(W["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], st.Tmax,
                                  st.Tmax, False, c.relative_attention_num_buckets)
            if getattr(st, "bias", None) is None:
                st.bias = fresh
            else:
                st.bias.copy_(fresh)            # in place: the captured step graph reads this buffer
            if getattr(st, "wgen", None) != wkey[0]:                                # buffers re-allocated: re-capture
                st.graph, st.wgen = None, wkey[0]
            st.wkey = wkey

    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, max_length=32, min_length=1, num_beams=1,
                 num_return_sequences=1, length_penalty=1.0, forced_bos_token_id=None, prefix_allowed_tokens_fn=None,
                 use_cache=True, cross_kv_dtype=None, **unused):
        """Greedy decoding (what `Atlas.generate` requests with num_beams=1, src/atlas.py:592-619; transformers 4.18
        `greedy_search` with `use_cache`): the encoder and the cross-attention K|V projections run once; every step
        decodes ONE token per sequence against the per-layer self K|V cache and the cached cross K|V (csrc/decode.cu),
        picks the next token on the device and - without a `prefix_allowed_tokens_fn` - is replayed from a single CUDA
        graph with no host synchronisation except an all-done poll every 8 steps.  use_cache=False runs the
        first-generation path (the decoder prefix re-run every step), kept as the parity reference of the tests.
        num_beams > 1: beam search (`_generate_beams`).  min_length=None means no EOS ban (the config's min_length, 0).
        cross_kv_dtype: None (default) keeps the cross K|V cache in the run's 16-bit dtype; "fp8" stores it as e4m3 with one
        fp32 scale per (key, K or V, head) (csrc/kv_fp8.cu): 0.53x the cache bytes, which every step streams once.  LOSSY
        (the decoder attends over the dequantized keys and values): tokens may differ from the 16-bit run."""
        if cross_kv_dtype is not None and cross_kv_dtype != "fp8":
            raise AtlasB200Error(f"cross_kv_dtype={cross_kv_dtype!r} is not supported (None = the run's 16-bit dtype, or \"fp8\")")
        if num_return_sequences != 1:
            raise AtlasB200Error(f"num_return_sequences={num_return_sequences} is not implemented (only 1)")
        if min_length is None:
            min_length = getattr(self.config, "min_length", 0) or 0
        if num_beams is not None and num_beams > 1:
            return self._generate_beams(input_ids, attention_mask, max_length, min_length, int(num_beams),
                                        1.0 if length_penalty is None else float(length_penalty), prefix_allowed_tokens_fn,
                                        unused, cross_kv_dtype)
        if not use_cache:
            if cross_kv_dtype is not None:
                raise AtlasB200Error("cross_kv_dtype='fp8' needs the KV-cached decode (use_cache=True): the use_cache=False "
                                     "path re-runs the decoder prefix on the 16-bit cross K|V")
            return self._generate_prefix_rerun(input_ids, attention_mask, max_length, min_length, prefix_allowed_tokens_fn)
        c = self.config
        enc = self.encode(input_ids, attention_mask)
        B, Lk = enc.shape[0], enc.shape[1]
        W, G, dt = self._weights()
        st = self._decode_state(B, Lk, int(max_length), dt, enc.device, xkv=cross_kv_dtype)
        self._prepare_decode(st, enc, attention_mask, W, dt)
        st.reset(c.decoder_start_token_id, c.pad_token_id)
        n_steps = int(max_length) - 1

        def step():
            logits = self._decode_step_logits(st)
            ops.decode_argmax(logits, st.seq, st.tok_in, st.done, st.t_dev, c.eos_token_id, c.pad_token_id, int(min_length))

        use_graph = self.cuda_graphs and prefix_allowed_tokens_fn is None and n_steps > 0
        if use_graph and (st.graph is None or getattr(st, "min_length", None) != int(min_length)):
            st.graph = _capture(step)[0]
            st.min_length = int(min_length)
            st.reset(c.decoder_start_token_id, c.pad_token_id)
        ran = 0
        for s_i in range(n_steps):
            if use_graph:
                st.graph.replay()
            elif prefix_allowed_tokens_fn is None:
                step()
            else:
                logits = self._decode_step_logits(st).float()
                seq_now = st.seq[:, : s_i + 1]
                allowed = torch.full_like(logits, -float("inf"))
                for b in range(B):
                    allowed[b, prefix_allowed_tokens_fn(b, seq_now[b])] = 0
                logits = (logits + allowed).to(dt)
                ops.decode_argmax(logits, st.seq, st.tok_in, st.done, st.t_dev, c.eos_token_id, c.pad_token_id,
                                  int(min_length))
            ran = s_i + 1
            if (s_i % 8 == 7 or s_i == n_steps - 1) and bool(st.done.all()):      # the only host synchronisation
                break
        seq = st.seq[:, : ran + 1].clone()
        # transformers stops right after the step in which the last sequence finished: drop all-pad trailing columns
        is_eos = seq[:, 1:] == c.eos_token_id
        if bool(is_eos.any(dim=1).all()):
            first = is_eos.float().argmax(dim=1) + 1
            seq = seq[:, : int(first.max()) + 1]
        return seq

    @torch.no_grad()
    def _generate_beams(self, input_ids, attention_mask, max_length, min_length, nb, length_penalty,
                        prefix_allowed_tokens_fn, unused, cross_kv_dtype=None):
        """Beam search: transformers 4.18 `beam_search` with `BeamSearchScorer` (early_stopping=False, one returned
        sequence).  The encoder and the cross K|V projections run once on the B unexpanded rows; each step decodes the
        B * nb beam rows with the KV-cached decoder (self-attention through the ancestry table, the nb beams of a batch
        element sharing its cross K|V), then csrc/beam.cu selects the next beams and updates the hypotheses on the device.
        Without a `prefix_allowed_tokens_fn` the step is replayed from one CUDA graph (all-done poll every 8 steps); with
        one, the steps run eagerly and the function sees every row's sequence rebuilt through the ancestry.  `finalize`
        runs on the host from one copy of the hypotheses and the running beams.  use_cache has no effect here."""
        if nb > ops.MAX_BEAMS:
            raise AtlasB200Error(f"num_beams={nb} exceeds the beam kernels' limit of {ops.MAX_BEAMS}")
        for name in ("do_sample", "early_stopping"):
            if unused.get(name):
                raise AtlasB200Error(f"{name}=True is not implemented with beam search (only early_stopping=False, no sampling)")
        if (unused.get("num_beam_groups") or 1) > 1 or unused.get("diversity_penalty"):
            raise AtlasB200Error("diverse / grouped beam search is not implemented")
        c = self.config
        max_length, min_length = int(max_length), int(min_length)
        V = c.vocab_size
        if V < 2:
            raise AtlasB200Error("beam search needs a vocabulary of at least 2 tokens")
        enc = self.encode(input_ids, attention_mask)
        B, Lk = enc.shape[0], enc.shape[1]
        W, G, dt = self._weights()
        st = self._decode_state(B, Lk, max_length, dt, enc.device, nb=nb, xkv=cross_kv_dtype)
        self._prepare_decode(st, enc, attention_mask, W, dt)
        # 4.18's log_softmax returns the logits' dtype: 16-bit parameters round the log-probs, fp32 ones keep them fp32
        round_lp = self.shared.weight.dtype in (torch.float16, torch.bfloat16)
        eos, pad = c.eos_token_id, c.pad_token_id
        st.reset(c.decoder_start_token_id, pad)
        n_steps = max_length - 1

        def step(mask=None):
            logits = self._decode_step_logits(st)
            ops.beam_topk(logits, st.beam_scores, st.t_dev, 2 * nb, eos, min_length, round_lp, add_mask=mask,
                          cand_score=st.cand_score, cand_tok=st.cand_tok)
            ops.beam_select(st.cand_score, st.cand_tok, nb, V, *st.select_buffers(), eos, pad, length_penalty)

        use_graph = self.cuda_graphs and prefix_allowed_tokens_fn is None and n_steps > 0
        gkey = (min_length, length_penalty, round_lp)
        if use_graph and (st.graph is None or getattr(st, "gkey", None) != gkey):
            st.graph = _capture(step)[0]
            st.gkey = gkey
            st.reset(c.decoder_start_token_id, pad)
        for s_i in range(n_steps):
            if use_graph:
                st.graph.replay()
            elif prefix_allowed_tokens_fn is None:
                step()
            else:
                seqs = st.sequences(s_i)                     # host synchronisation: the callback needs the sequences
                allowed = torch.full((st.R, V), -float("inf"), dtype=torch.float32, device=enc.device)
                for r in range(st.R):
                    allowed[r, prefix_allowed_tokens_fn(r // nb, seqs[r])] = 0
                step(allowed)
            if (s_i % 8 == 7 or s_i == n_steps - 1) and bool(st.done.all()):      # the only host synchronisation
                break
        return self._finalize_beams(st, max_length, length_penalty)

    def _finalize_beams(self, st, max_length, length_penalty):
        """BeamSearchScorer.finalize (4.18) on the host: the running beams of unfinished batch elements join their
        hypotheses, the best (the last of a stable sort by score: among equal scores the last inserted) is returned, padded
        with pad only when the lengths differ and closed by EOS where it is shorter than max_length."""
        c = self.config
        B, nb = st.B, st.nb
        t = int(st.t_dev)
        run = st.sequences(t).cpu().tolist()
        scores = st.beam_scores.cpu().tolist()
        done = st.done.cpu().tolist()
        h_score, h_len, h_ins = st.hyp_score.cpu().tolist(), st.hyp_len.cpu().tolist(), st.hyp_ins.cpu().tolist()
        h_tok, h_state, h_worst = st.hyp_tok.cpu(), st.hyp_state.cpu().tolist(), st.hyp_worst.cpu().tolist()
        best = []
        for b in range(B):
            slots = sorted(range(h_state[b][0]), key=lambda j: h_ins[b][j])            # list order = insertion order
            beams = [(h_score[b][j], h_tok[b, j, : h_len[b][j]].tolist()) for j in slots]
            worst = h_worst[b]
            if not done[b]:
                for k in range(nb):                           # BeamHypotheses.add of the running beam
                    hyp = run[b * nb + k]
                    score = scores[b * nb + k] / (len(hyp) ** length_penalty)
                    if len(beams) < nb or score > worst:
                        beams.append((score, hyp))
                        if len(beams) > nb:
                            order = sorted([(s, i) for i, (s, _) in enumerate(beams)])
                            del beams[order[0][1]]
                            worst = order[1][0]
                        else:
                            worst = min(score, worst)
            best.append(sorted(beams, key=lambda x: x[0]).pop()[1])
        lens = [len(h) for h in best]
        out = torch.full((B, min(max(lens) + 1, max_length)), c.pad_token_id, dtype=torch.int64)
        for b, h in enumerate(best):
            out[b, : len(h)] = torch.tensor(h, dtype=torch.int64)
            if len(h) < max_length:
                out[b, len(h)] = c.eos_token_id
        return out.to(st.tok.device)

    @torch.no_grad()
    def _generate_prefix_rerun(self, input_ids, attention_mask, max_length, min_length, prefix_allowed_tokens_fn):
        """First-generation greedy loop: the encoder and the cross-attention K/V projections run once, every step
        re-runs the whole decoder prefix (no self-attention cache).  Parity reference for the cached path."""
        c = self.config
        enc = self.encode(input_ids, attention_mask)
        B, keys = enc.shape[0], enc.shape[1]
        kv = self.cross_kv(_pad_keys(enc.reshape(B * keys, -1), B, keys, _cross_split(keys)[1]))   # decode's key range
        mask = attention_mask.reshape(B, -1)
        seq = torch.full((B, 1), c.decoder_start_token_id, dtype=torch.long, device=enc.device)
        done = torch.zeros(B, dtype=torch.bool, device=enc.device)
        for step in range(max_length - 1):
            logits = self.decode(seq, enc, mask, cross_kv=kv)[:, -1].float()
            if step + 1 < min_length:
                logits[:, c.eos_token_id] = -float("inf")
            if prefix_allowed_tokens_fn is not None:
                allowed = torch.full_like(logits, -float("inf"))
                for b in range(B):
                    allowed[b, prefix_allowed_tokens_fn(b, seq[b])] = 0
                logits = logits + allowed
            nxt = logits.argmax(dim=-1)
            nxt = torch.where(done, torch.full_like(nxt, c.pad_token_id), nxt)
            seq = torch.cat([seq, nxt[:, None]], dim=1)
            done = done | (nxt == c.eos_token_id)
            if bool(done.all()):
                break
        return seq
