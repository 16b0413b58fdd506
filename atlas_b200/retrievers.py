"""Drop-in for `src.retrievers` (reference src/retrievers.py:16-135): Contriever = BERT encoder + masked
mean pooling, and the dual-encoder wrappers.  Under `torch.no_grad` (index build / refresh, query embedding:
`Atlas.build_index` / `Atlas._retrieve`, src/atlas.py:61-88,90-118) the fused forward runs; with gradients enabled
(retriever training, src/atlas.py:457-465) the same kernels run forward with the hand-written backward kernels behind
torch.autograd (`_encode_train`, grad_ops.py).

Parameter names and shapes are those of the reference's `BertModel` (vendored HF 4.18,
src/modeling_bert.py:190-648,872-1045), so `load_state_dict` of a Contriever checkpoint works:
    embeddings.{word,position,token_type}_embeddings.weight, embeddings.LayerNorm.{weight,bias},
    encoder.layer.N.attention.self.{query,key,value}.{weight,bias}, attention.output.dense / LayerNorm,
    intermediate.dense, output.dense / LayerNorm.
The arithmetic runs in `csrc/`: wgmma GEMMs with fused bias / erf-GELU / residual epilogues, fused attention
reading Q/K/V in place from one [tokens, 2304] projection buffer, the reference's non-standard BertLayerNorm
(uncentred second moment, src/modeling_bert.py:104-114), masked mean pooling that can write straight into
the passage bank rows.  16-bit only on the device: fp32 parameters (the live query encoder without
`--precision bf16`) are cast to fp16 copies that are refreshed when the parameters change.
"""
import copy
import math
from types import SimpleNamespace

import torch
from torch import nn

from . import grad_ops, ops
from ._lib import AtlasB200Error

EMBEDDINGS_DIM: int = 768


class BertConfigLite(SimpleNamespace):
    """The BertConfig fields this path reads (defaults = bert-base-uncased / facebook/contriever)."""

    def __init__(self, **kw):
        d = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12,
                 hidden_act="gelu", pad_token_id=0)
        d.update(kw)
        super().__init__(**d)


def _cfg(config, name, default=None):
    return getattr(config, name, default)


class _LN(nn.Module):
    def __init__(self, h):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(h))
        self.bias = nn.Parameter(torch.zeros(h))


class _Embeddings(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.word_embeddings = nn.Embedding(c.vocab_size, c.hidden_size, padding_idx=_cfg(c, "pad_token_id", 0))
        self.position_embeddings = nn.Embedding(c.max_position_embeddings, c.hidden_size)
        self.token_type_embeddings = nn.Embedding(c.type_vocab_size, c.hidden_size)
        self.LayerNorm = _LN(c.hidden_size)
        self.register_buffer("position_ids", torch.arange(c.max_position_embeddings).expand((1, -1)), persistent=False)


class _SelfAttention(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.query = nn.Linear(c.hidden_size, c.hidden_size)
        self.key = nn.Linear(c.hidden_size, c.hidden_size)
        self.value = nn.Linear(c.hidden_size, c.hidden_size)


class _DenseLN(nn.Module):
    def __init__(self, fin, fout):
        super().__init__()
        self.dense = nn.Linear(fin, fout)
        self.LayerNorm = _LN(fout)


class _Attention(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.self = _SelfAttention(c)
        self.output = _DenseLN(c.hidden_size, c.hidden_size)


class _Intermediate(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.dense = nn.Linear(c.hidden_size, c.intermediate_size)


class _Layer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.attention = _Attention(c)
        self.intermediate = _Intermediate(c)
        self.output = _DenseLN(c.intermediate_size, c.hidden_size)


class _Encoder(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.layer = nn.ModuleList([_Layer(c) for _ in range(c.num_hidden_layers)])


_warned = set()


def _warn_no_dropout(who):
    """Kept for callers of round 1: dropout IS implemented now (grad_ops.dropout / attention dropout_p); nothing to warn."""
    return None


_WEIGHTS_EPOCH = [0]


def _bump_weights_epoch(*_args, **_kw):
    _WEIGHTS_EPOCH[0] += 1


try:    # every optimizer.step() anywhere in the process (AdamWFP32Copy, fairscale OSS ...) marks the 16-bit copies stale:
    # some optimizers write through `param.data`, which does not bump the parameter's version counter
    from torch.optim.optimizer import register_optimizer_step_post_hook as _reg_hook

    _reg_hook(_bump_weights_epoch)
except Exception:       # older torch: version counters + explicit invalidate() only
    pass


class HalfCache:
    """16-bit device copies of a module's parameters, one set per compute dtype (the live query encoder may run
    in bf16 while index refresh embeds passages in fp32-master / fp16 like src/atlas.py:54-59).

    The copies live in FIXED buffers that are refreshed IN PLACE, so CUDA graphs that read them stay valid when the
    weights change (no re-capture per optimizer step).  A refresh happens on the next `get()` after
      * any parameter's autograd version or storage changed (in-place ops, `load_state_dict`, `.to()`),
      * any `optimizer.step()` in the process (global post-step hook: covers optimizers that write through `param.data`),
      * an explicit `invalidate()` (callers that write `param.data` by hand).
    `derived(dtype, build)` caches tensors computed from a set (fused QKV weights ...), refreshed in place with it.
    `gen` changes only when buffers are re-allocated (parameter set / shapes / device changed): the CUDA-graph key."""

    def __init__(self):
        self.sets = {}
        self._dirty = False

    def invalidate(self):
        self._dirty = True

    def get(self, module, dtype):
        params = list(module.named_parameters())
        struct = tuple((n, p.data_ptr(), tuple(p.shape), p.dtype, p.device) for n, p in params)
        key = (tuple(p._version for _, p in params), _WEIGHTS_EPOCH[0])
        ent = self.sets.get(dtype)
        if ent is None or ent["struct"] != struct:
            store = {n: (p.detach() if p.dtype == dtype else p.detach().to(dtype)).contiguous() for n, p in params}
            gen = 0 if ent is None else ent["gen"] + 1
            ent = {"struct": struct, "key": key, "store": store, "derived": None, "derived_stale": False, "gen": gen}
            self.sets[dtype] = ent
            self._dirty = False
        elif (ent["key"] != key or self._dirty) and not torch.cuda.is_current_stream_capturing():
            for n, p in params:
                dst = ent["store"][n]
                if dst.data_ptr() != p.data_ptr():          # a converted copy (an alias of the live tensor needs nothing)
                    dst.copy_(p.detach())
            ent["key"] = key
            ent["derived_stale"] = ent["derived"] is not None
            self._dirty = False
        return ent["store"]

    def derived(self, dtype, build):
        ent = self.sets[dtype]
        if ent["derived"] is None:
            ent["derived"] = build(ent["store"])
        elif ent["derived_stale"] and not torch.cuda.is_current_stream_capturing():
            fresh = build(ent["store"])
            for k, v in fresh.items():
                ent["derived"][k].copy_(v)
            ent["derived_stale"] = False
        return ent["derived"]


class Contriever(nn.Module):
    def __init__(self, config=None, pooling="average", **kwargs):
        super().__init__()
        config = config or BertConfigLite()
        self.config = config
        if not hasattr(config, "pooling"):
            self.config.pooling = pooling
        if config.hidden_size != config.num_attention_heads * 64:
            raise AtlasB200Error("atlas_b200 attention kernels need head_dim 64")
        if _cfg(config, "hidden_act", "gelu") != "gelu":
            raise AtlasB200Error("only the erf GELU of BERT-base / Contriever is implemented")
        self.embeddings = _Embeddings(config)
        self.encoder = _Encoder(config)
        self._half = HalfCache()
        self.apply(self._init_weights)

    def _init_weights(self, m):  # HF BERT init (src/modeling_bert.py:~850), std 0.02
        if isinstance(m, nn.Linear):
            m.weight.data.normal_(mean=0.0, std=0.02)
            if m.bias is not None:
                m.bias.data.zero_()
        elif isinstance(m, nn.Embedding):
            m.weight.data.normal_(mean=0.0, std=0.02)
            if m.padding_idx is not None:
                m.weight.data[m.padding_idx].zero_()

    @classmethod
    def from_pretrained(cls, path, **kw):
        """Local HF-layout directory (config.json + weights), src/model_io.py:45."""
        from ._pretrained import load_pretrained

        return load_pretrained(cls, BertConfigLite, path, **kw)

    def gradient_checkpointing_enable(self):
        """`--use_gradient_checkpoint_retriever` (src/atlas.py:454-455): recompute each BERT layer in the backward."""
        self._grad_ckpt = True

    def gradient_checkpointing_disable(self):
        self._grad_ckpt = False

    def _dtype(self):
        d = self.embeddings.word_embeddings.weight.dtype
        return d if d in (torch.float16, torch.bfloat16) else torch.float16

    def _fuse(self, W):
        """one [2304, 768] projection per layer: q | k | v"""
        f = {}
        for i in range(self.config.num_hidden_layers):
            p = f"encoder.layer.{i}.attention.self."
            f[p + "qkv.weight"] = torch.cat([W[p + "query.weight"], W[p + "key.weight"], W[p + "value.weight"]], 0)
            f[p + "qkv.bias"] = torch.cat([W[p + "query.bias"], W[p + "key.bias"], W[p + "value.bias"]], 0)
        return f

    @torch.no_grad()
    def encode(self, input_ids, attention_mask, token_type_ids=None, dtype=None):
        """last hidden state [B, L, H] in the 16-bit compute dtype (src/modeling_bert.py:929-1045).
        `dtype` overrides the compute dtype (fp16 for passages whatever the live parameters are)."""
        c = self.config
        dt = dtype or self._dtype()
        W = self._half.get(self, dt)
        F = self._half.derived(dt, self._fuse)
        B, L = input_ids.shape
        H, nh = c.hidden_size, c.num_attention_heads
        h = ops.bert_embed_ln(input_ids, token_type_ids, W["embeddings.word_embeddings.weight"],
                              W["embeddings.token_type_embeddings.weight"], W["embeddings.position_embeddings.weight"],
                              W["embeddings.LayerNorm.weight"], W["embeddings.LayerNorm.bias"], c.layer_norm_eps)
        h = h.view(B * L, H)
        # transformers==4.18 get_extended_attention_mask: (1 - mask) * -10000 (src/modeling_bert.py:993)
        add_mask = (1.0 - attention_mask.to(torch.float32)) * -10000.0
        live = ops.key_block_live(add_mask)       # all-padding 64-key blocks (queries are padded to text_maxlength): skipped
        # Padding-compacted encoder (same scheme as FiD._encode_rows): every sequence keeps its 64-row tiles up
        # to its last live key, packed back to back; projections run over the device-side row count, the attention on the
        # packed rows.  Padded positions never influence live ones and every consumer of the result masks them (mean pooling)
        # or reads position 0 (cls pooling): the returned rows of dropped tiles are 0.
        packed = ops._ENC_PACKED and ops._BERT_PACKED and ops.encoder_packs(live, L)
        rows = None
        if packed:
            keep, tile_off, _, rows = ops.segment_tile_scan(live)
            h = ops.compact_live_tiles(h, keep)[0]
        qkv = torch.empty((B * L, 3 * H), dtype=dt, device=h.device)
        for i in range(c.num_hidden_layers):
            p = f"encoder.layer.{i}."
            ops.linear(h, F[p + "attention.self.qkv.weight"], F[p + "attention.self.qkv.bias"], out=qkv, rows=rows)
            if packed:
                ctx = ops.attention_packed(qkv, keep, tile_off, B, nh, L, add_mask, None, scale=1.0 / math.sqrt(64))
            else:
                ctx = ops.attention(qkv, 0, qkv, H, qkv, 2 * H, B, nh, L, L, add_mask=add_mask, scale=1.0 / math.sqrt(64),
                                    block_live=live)
            s1 = ops.linear(ctx, W[p + "attention.output.dense.weight"], W[p + "attention.output.dense.bias"], residual=h,
                            rows=rows)
            h1 = ops.layernorm(s1, W[p + "attention.output.LayerNorm.weight"], W[p + "attention.output.LayerNorm.bias"],
                               c.layer_norm_eps, kind=0)
            inter = ops.linear(h1, W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"],
                               epilogue=ops.EPI_GELU, rows=rows)
            s2 = ops.linear(inter, W[p + "output.dense.weight"], W[p + "output.dense.bias"], residual=h1, rows=rows)
            h = ops.layernorm(s2, W[p + "output.LayerNorm.weight"], W[p + "output.LayerNorm.bias"], c.layer_norm_eps,
                              kind=0)
        if packed:
            h = ops.expand_packed_tiles(h, tile_off)
        return h.view(B, L, H)

    # ---- training path (autograd through the kernels, grad_ops.py) ---------------------------------------
    def _encode_train(self, input_ids, attention_mask, token_type_ids=None):
        """`encode` with autograd: the same GEMM / attention / LayerNorm kernels forward (bias + GELU un-fused so the
        pre-activations are kept), hand-written backward kernels behind torch.autograd (src/modeling_bert.py:929-1045
        under `loss.backward()`).  16-bit views of the parameters are made with differentiable casts / concatenations."""
        g = grad_ops
        c = self.config
        pd = self.embeddings.word_embeddings.weight.dtype
        # fp32 master parameters train through bf16 activations / gradients (fp16 gradients would need loss scaling)
        dt = pd if pd in (torch.float16, torch.bfloat16) else torch.bfloat16
        # nn.Dropout of the reference in training mode (src/modeling_bert.py:246,356,384,463): counter-based masks inside
        # the kernels, re-derived in the backward (csrc/dropout.cuh)
        ph = float(_cfg(c, "hidden_dropout_prob", 0.0) or 0.0) if self.training else 0.0
        pa = float(_cfg(c, "attention_probs_dropout_prob", 0.0) or 0.0) if self.training else 0.0
        W = {n: (p if p.dtype == dt else p.to(dt)) for n, p in self.named_parameters()}
        B, L = input_ids.shape
        H, nh = c.hidden_size, c.num_attention_heads
        pad = self.embeddings.word_embeddings.padding_idx
        x = g.bert_embed_sum(input_ids, token_type_ids, W["embeddings.word_embeddings.weight"],
                             W["embeddings.token_type_embeddings.weight"], W["embeddings.position_embeddings.weight"],
                             -1 if pad is None else int(pad))
        h = g.layernorm(x.view(B * L, H), W["embeddings.LayerNorm.weight"], W["embeddings.LayerNorm.bias"],
                        c.layer_norm_eps, kind=0)
        h = g.dropout(h, ph)
        add_mask = (1.0 - attention_mask.to(torch.float32)) * -10000.0

        def dense_res(x, w, b, res):
            # BertSelfOutput / BertOutput: dense -> dropout -> + input (fused into the GEMM epilogue without dropout)
            if ph:
                return g.dropout(g.linear(x, w, b), ph, residual=res)
            return g.linear(x, w, b, residual=res)

        def layer(i, h):
            p = f"encoder.layer.{i}."
            a = p + "attention.self."
            wqkv = torch.cat([W[a + "query.weight"], W[a + "key.weight"], W[a + "value.weight"]], 0)
            bqkv = torch.cat([W[a + "query.bias"], W[a + "key.bias"], W[a + "value.bias"]], 0)
            qkv = g.linear(h, wqkv, bqkv)
            ctx = g.self_attention(qkv, B, nh, L, add_mask=add_mask, scale=1.0 / math.sqrt(64), dropout_p=pa)
            s1 = dense_res(ctx, W[p + "attention.output.dense.weight"], W[p + "attention.output.dense.bias"], h)
            h1 = g.layernorm(s1, W[p + "attention.output.LayerNorm.weight"], W[p + "attention.output.LayerNorm.bias"],
                             c.layer_norm_eps, kind=0)
            z = g.linear(h1, W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"])
            s2 = dense_res(g.gelu_erf(z), W[p + "output.dense.weight"], W[p + "output.dense.bias"], h1)
            return g.layernorm(s2, W[p + "output.LayerNorm.weight"], W[p + "output.LayerNorm.bias"], c.layer_norm_eps,
                               kind=0)

        for i in range(c.num_hidden_layers):
            if getattr(self, "_grad_ckpt", False):
                from torch.utils.checkpoint import checkpoint

                h = checkpoint(layer, i, h, use_reentrant=False)
            else:
                h = layer(i, h)
        return h.view(B, L, H)

    def forward(self, input_ids=None, attention_mask=None, token_type_ids=None, position_ids=None, head_mask=None,
                inputs_embeds=None, encoder_hidden_states=None, encoder_attention_mask=None, output_attentions=None,
                output_hidden_states=None, normalize=False):
        """src/retrievers.py:22-60.  Returns [B, 768] embeddings in the parameters' dtype."""
        if position_ids is not None or inputs_embeds is not None:
            raise AtlasB200Error("position_ids / inputs_embeds are not used by Atlas and not supported")
        with_grad = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if not with_grad and self.config.pooling == "average" and not normalize:
            emb = self._embed_graphed(input_ids, attention_mask, token_type_ids)
            if emb is not None:
                pd = self.embeddings.word_embeddings.weight.dtype
                return emb if emb.dtype == pd else emb.to(pd)
        if with_grad:   # retriever training (src/atlas.py:457-465): autograd through the kernels
            last_hidden = self._encode_train(input_ids, attention_mask, token_type_ids)
        else:
            last_hidden = self.encode(input_ids, attention_mask, token_type_ids)
        pooling = self.config.pooling
        if pooling == "average":
            emb = (grad_ops.masked_mean_pool if with_grad else ops.masked_mean_pool)(last_hidden, attention_mask)
        elif pooling == "cls":
            emb = last_hidden[:, 0].clone()
        else:
            raise AtlasB200Error(f"pooling={pooling!r} is not implemented (Contriever uses 'average')")
        if normalize:
            emb = torch.nn.functional.normalize(emb.float(), dim=-1).to(emb.dtype)
        pd = self.embeddings.word_embeddings.weight.dtype
        return emb if emb.dtype == pd else emb.to(pd)

    @torch.no_grad()
    def _embed_graphed(self, input_ids, attention_mask, token_type_ids):
        """Small no-grad batches (query embedding: 8 x 384 tokens at BASELINE configs[3]) are launch-bound - ~100 kernel
        launches for well under a millisecond of GPU work - so the whole encode + pooling is replayed from one CUDA graph per
        (shape, dtype, weight-buffer generation), like the reader's forward (fid._GraphRunner).  Larger batches (index refresh)
        keep the eager path: they are GPU-bound and would pin large activation pools.  Returns None when not applicable."""
        import os

        if os.environ.get("ATLAS_B200_CUDA_GRAPH", "1") == "0" or not input_ids.is_cuda:
            return None
        B, L = input_ids.shape
        if B * L > 16384 or torch.cuda.is_current_stream_capturing():
            return None
        from .fid import _GraphRunner

        dt = self._dtype()
        self._half.get(self, dt)                              # the 16-bit weight buffers exist / are current before capture
        self._half.derived(dt, self._fuse)                    # ... and the fused q|k|v copies (refreshed in place, never in a replay)
        gen = self._half.sets[dt]["gen"]
        mask = attention_mask if attention_mask is not None else torch.ones_like(input_ids)
        has_tt = token_type_ids is not None
        key = (B, L, dt, gen, has_tt, input_ids.device, mask.dtype, ops._ENC_PACKED and ops._BERT_PACKED)
        graphs = self.__dict__.setdefault("_graphs", {})
        runner = graphs.get(key)
        if runner is None:
            if len(graphs) >= 4:
                graphs.pop(next(iter(graphs)))

            def fn(ids, m, *tt):
                hidden = self.encode(ids, m, tt[0] if tt else None)
                return ops.masked_mean_pool(hidden, m)

            example = (input_ids, mask) + ((token_type_ids,) if has_tt else ())
            runner = graphs[key] = _GraphRunner(fn, example)
        args = (input_ids, mask) + ((token_type_ids,) if has_tt else ())
        return runner(*args).clone()

    @torch.no_grad()
    def embed_fp16(self, input_ids, attention_mask):
        """Passage embeddings computed with fp16 copies of the weights, whatever the live dtype is: what the
        reference gets from `copy.deepcopy(retriever).half().eval()` (src/atlas.py:54-59)."""
        if self.config.pooling != "average":
            raise AtlasB200Error("embed_fp16: only average pooling is implemented")
        return ops.masked_mean_pool(self.encode(input_ids, attention_mask, dtype=torch.float16), attention_mask)

    @torch.no_grad()
    def embed_into(self, input_ids, attention_mask, bank_rows, dtype=None):
        """Index refresh in place: pooled embeddings written straight into `bank_rows` ([B, 768] slice of
        the passage bank) - replaces `index.embeddings[:, a:b] = embeddings.T` (src/atlas.py:78-79)."""
        last_hidden = self.encode(input_ids, attention_mask, dtype=dtype)
        if last_hidden.dtype != bank_rows.dtype:
            raise AtlasB200Error("embed_into: the retriever copy must have the bank dtype (fp16, src/atlas.py:54-59)")
        ops.masked_mean_pool(last_hidden, attention_mask, out=bank_rows)
        return bank_rows


class BaseRetriever(nn.Module):
    """src/retrievers.py:63-87."""

    def __init__(self, *args, **kwargs):
        super(BaseRetriever, self).__init__()

    def embed_queries(self, *args, **kwargs):
        raise NotImplementedError()

    def embed_passages(self, *args, **kwargs):
        raise NotImplementedError()

    def forward(self, *args, is_passages=False, **kwargs):
        if is_passages:
            return self.embed_passages(*args, **kwargs)
        else:
            return self.embed_queries(*args, **kwargs)

    def gradient_checkpointing_enable(self):
        for m in self.children():
            m.gradient_checkpointing_enable()

    def gradient_checkpointing_disable(self):
        for m in self.children():
            m.gradient_checkpointing_disable()


class DualEncoderRetriever(BaseRetriever):
    """src/retrievers.py:90-105."""

    def __init__(self, opt, contriever):
        super(DualEncoderRetriever, self).__init__()
        self.opt = opt
        self.contriever = contriever

    def _embed(self, *args, **kwargs):
        return self.contriever(*args, **kwargs)

    def embed_queries(self, *args, **kwargs):
        return self._embed(*args, **kwargs)

    def embed_passages(self, *args, **kwargs):
        return self._embed(*args, **kwargs)


class UntiedDualEncoderRetriever(BaseRetriever):
    """src/retrievers.py:108-135."""

    def __init__(self, opt, query_encoder, passage_encoder=None):
        super(UntiedDualEncoderRetriever, self).__init__()
        self.opt = opt
        self.query_contriever = query_encoder
        if passage_encoder is None:
            passage_encoder = copy.deepcopy(query_encoder) if hasattr(query_encoder, "module") else query_encoder
        self.passage_contriever = passage_encoder

    def embed_queries(self, *args, **kwargs):
        return self.query_contriever(*args, **kwargs)

    def embed_passages(self, *args, **kwargs):
        if self.opt.query_side_retriever_training:
            is_train = self.passage_contriever.training
            self.passage_contriever.eval()
            with torch.no_grad():
                passage_emb = self.passage_contriever(*args, **kwargs)
            if is_train:
                self.passage_contriever.train()
        else:
            passage_emb = self.passage_contriever(*args, **kwargs)
        return passage_emb
