"""Autograd wiring of the B200 kernels for the training step (reference: train.py -> `Atlas.forward` ->
`loss.backward()`, src/atlas.py:399-550).  Every Function's forward AND backward run in `lib/libatlas_b200.so`
(ops.py); torch.autograd only chains them and accumulates into the parameters' `.grad`.

What autograd would derive through the reference's modules is implemented by hand:
  Linear           y = x W^T (+ b) (+ residual)      dX = dY W (wgmma GEMM on W^T), dW = dY^T X (wgmma GEMM with both
                                                     operands MN-major: no transposes; split-K, fp32 accumulation over
                                                     the tokens), db = column sums
  Norm             BertLayerNorm / T5 RMSNorm        src/modeling_bert.py:104-114, src/modeling_t5.py:244-253
  Attention        fused attention, saved O only     src/modeling_bert.py:328-366, src/modeling_t5.py:478-524
  CrossAttention   FiD decoder over n*L keys         src/fid.py:298-349
  GatedGelu / Gelu T5DenseGatedGeluDense / BERT FF   src/modeling_t5.py:281-285, src/modeling_bert.py:444
  Relu, LinearRelu T5DenseReluDense (T5 v1.0)        src/modeling_t5.py:256-270; the mask comes from the saved output
  Embedding, BertEmbedSum, MaskedMeanPool, CrossEntropy
Weights arrive as 16-bit tensors that require grad (the caller derives them from the fp32 / bf16 parameters with
differentiable casts / concatenations, so autograd routes dW back to the reference-named parameters).
Dropout (hidden states: `dropout`; attention probabilities: inside the attention kernels) draws counter-based masks
from (seed, offset) keys of torch's CUDA generator and re-derives them in the backward (csrc/dropout.cuh).
"""
import torch

from . import ops
from ._lib import AtlasB200Error


def _need(ctx, i):
    return ctx.needs_input_grad[i]


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, residual):
        y = ops.linear(x, weight, bias, residual=residual)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        ctx.has_res = residual is not None
        ctx.bias_dtype = bias.dtype if bias is not None else None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous()
        dy2 = dy.reshape(-1, dy.shape[-1])
        dx = dw = db = None
        if _need(ctx, 0):
            dx = ops.linear_dgrad(dy2, weight).reshape(x.shape)
        if _need(ctx, 1):
            dw = ops.linear_wgrad(dy2, x.reshape(-1, x.shape[-1]))
        if ctx.has_bias and _need(ctx, 2):
            db = ops.colsum(dy2).to(ctx.bias_dtype)
        dres = dy if (ctx.has_res and _need(ctx, 3)) else None
        return dx, dw, db, dres


def linear(x, weight, bias=None, residual=None):
    """y = x @ weight.T (+ bias) (+ residual), differentiable in x / weight / bias / residual."""
    return _Linear.apply(x, weight, bias, residual)


class _Norm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, kind):
        y = ops.layernorm(x, weight, bias, eps, kind=kind)
        ctx.save_for_backward(x, weight)
        ctx.eps, ctx.kind, ctx.has_bias = eps, kind, bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dx, dw, db = ops.layernorm_bwd(x, dy.contiguous(), weight, ctx.eps, ctx.kind)
        return dx, dw.to(weight.dtype), (db.to(weight.dtype) if ctx.has_bias else None), None, None


def layernorm(x, weight, bias=None, eps=1e-12, kind=0):
    return _Norm.apply(x, weight, bias, eps, kind)


class _SelfAttention(torch.autograd.Function):
    """qkv [B*L, 3*H*64] (q | k | v as written by the fused projection) -> ctx [B*L, H*64]."""

    @staticmethod
    def forward(ctx, qkv, bias_delta, add_mask, B, H, L, scale, causal_value, dropout_p, long_segments):
        ctx.drop = (dropout_p,) + next_dropout_key(qkv.device) if dropout_p else None
        fwd = ops.encoder_attention(L) if long_segments else ops.attention
        out, lse = fwd(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, B, H, L, L, add_mask=add_mask, bias_delta=bias_delta, scale=scale,
                       causal_value=causal_value, return_lse=True, dropout=ctx.drop,
                       block_live=getattr(add_mask, "_atlas_block_live", None))
        ctx.save_for_backward(qkv, out, bias_delta, add_mask, lse)
        ctx.dims = (B, H, L, scale, causal_value)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, out, bias_delta, add_mask, lse = ctx.saved_tensors
        B, H, L, scale, causal_value = ctx.dims
        dqkv = torch.empty_like(qkv)
        dbias = ops.attention_bwd(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, out, dout.contiguous(), dqkv, 0, dqkv, H * 64,
                                  dqkv, 2 * H * 64, B, H, L, L, add_mask=add_mask, bias_delta=bias_delta,
                                  need_dbias=bias_delta is not None and _need(ctx, 1), scale=scale,
                                  causal_value=causal_value, lse=lse, dropout=ctx.drop,
                                  block_live=getattr(add_mask, "_atlas_block_live", None))
        return dqkv, dbias, None, None, None, None, None, None, None, None


def self_attention(qkv, B, H, L, add_mask=None, bias_delta=None, scale=1.0, causal_value=0.0, dropout_p=0.0,
                   long_segments=False):
    """dropout_p: nn.Dropout on the attention probabilities (training), inside the kernels.  long_segments: segments longer
    than ops.ATTENTION_MAX_LK run on ops.attention_long (the FiD encoder's passages; the backward takes any length)."""
    return _SelfAttention.apply(qkv, bias_delta, add_mask, B, H, L, scale, causal_value, float(dropout_p or 0.0),
                                long_segments)


class _PackedSelfAttention(torch.autograd.Function):
    """qkv [rows, 3*H*64] on the packed rows of the padding-compacted encoder (ops.segment_tile_scan) -> ctx [rows, H*64]."""

    @staticmethod
    def forward(ctx, qkv, bias_delta, add_mask, keep, tile_off, S, H, L, scale, dropout_p):
        ctx.drop = (dropout_p,) + next_dropout_key(qkv.device) if dropout_p else None
        out, lse = ops.attention_packed(qkv, keep, tile_off, S, H, L, add_mask, bias_delta, scale=scale, lse=True,
                                        dropout=ctx.drop)
        ctx.save_for_backward(qkv, out, bias_delta, add_mask, keep, tile_off, lse)
        ctx.dims = (S, H, L, scale)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, out, bias_delta, add_mask, keep, tile_off, lse = ctx.saved_tensors
        S, H, L, scale = ctx.dims
        dqkv, dbias = ops.attention_packed_bwd(qkv, out, dout.contiguous(), keep, tile_off, S, H, L, add_mask, bias_delta, lse,
                                               scale=scale, need_dbias=bias_delta is not None and _need(ctx, 1),
                                               dropout=ctx.drop)
        return dqkv, dbias, None, None, None, None, None, None, None, None


def packed_self_attention(qkv, keep, tile_off, S, H, L, add_mask, bias_delta=None, scale=1.0, dropout_p=0.0):
    """`self_attention` of segments of L tokens on their packed rows (keep / tile_off: ops.segment_tile_scan); the same
    dropout masks, draw of the dropout key and gradients on the kept rows as the padded layout's."""
    return _PackedSelfAttention.apply(qkv, bias_delta, add_mask, keep, tile_off, S, H, L, scale, float(dropout_p or 0.0))


class _ExpandPacked(torch.autograd.Function):
    """Packed rows [rows, d] -> the padded layout [n_tiles * 64, d], zeros at the dropped tiles; backward: the gradient rows of
    the kept tiles, packed again (ops.compact_live_tiles over keep, the same tile order)."""

    @staticmethod
    def forward(ctx, x, keep, tile_off):
        ctx.save_for_backward(keep)
        ctx.rows = x.shape[0]
        return ops.expand_packed_tiles(x, tile_off)

    @staticmethod
    def backward(ctx, dy):
        (keep,) = ctx.saved_tensors
        dx, _, _ = ops.compact_live_tiles(dy.contiguous(), keep)
        return dx[: ctx.rows], None, None


def expand_packed(x, keep, tile_off):
    return _ExpandPacked.apply(x, keep, tile_off)


class _CrossAttention(torch.autograd.Function):
    """q [B*T, H*64], kv [B*Lk, 2*H*64] (k | v) -> ctx [B*T, H*64]; forward = split-KV kernel + combine."""

    @staticmethod
    def forward(ctx, q, kv, add_mask, B, H, T, Lk, scale, split, dropout_p):
        ctx.drop = (dropout_p,) + next_dropout_key(q.device) if dropout_p else None
        out, lse = ops.cross_attention_split(q, 0, kv, 0, H * 64, B, H, T, Lk, add_mask=add_mask, scale=scale,
                                             split=split, return_lse=True, dropout=ctx.drop,
                                             tile_live=getattr(add_mask, "_atlas_block_live", None))
        ctx.save_for_backward(q, kv, out, add_mask, lse)
        ctx.dims = (B, H, T, Lk, scale)
        ctx.mark_non_differentiable(lse)
        return out, lse

    @staticmethod
    def backward(ctx, dout, _dlse):
        q, kv, out, add_mask, lse = ctx.saved_tensors
        B, H, T, Lk, scale = ctx.dims
        dq = torch.empty((B * T, H * 64), dtype=q.dtype, device=q.device)
        dkv = torch.empty_like(kv)
        ops.attention_bwd(q, 0, kv, 0, kv, H * 64, out, dout.contiguous(), dq, 0, dkv, 0, dkv, H * 64, B, H, T, Lk,
                          add_mask=add_mask, scale=scale, lse=lse, split_keys=Lk > 1024, dropout=ctx.drop,
                          block_live=getattr(add_mask, "_atlas_block_live", None))
        return dq, dkv, None, None, None, None, None, None, None, None


def cross_attention(q, kv, B, H, T, Lk, add_mask=None, scale=1.0, split=384, return_lse=False, dropout_p=0.0):
    out, lse = _CrossAttention.apply(q, kv, add_mask, B, H, T, Lk, scale, split, float(dropout_p or 0.0))
    return (out, lse) if return_lse else out


def next_dropout_key(device):
    """(seed, offset) for one dropout site, drawn from torch's CUDA generator of `device`: `torch.manual_seed` makes a run
    reproducible and `torch.utils.checkpoint` (which saves / restores the generator state) re-derives the same masks
    when a block is recomputed in the backward.  No device synchronisation."""
    gen = torch.cuda.default_generators[device.index if device.index is not None else torch.cuda.current_device()]
    seed, off = gen.initial_seed(), gen.get_offset()
    gen.set_offset(off + 4)
    return seed & 0xFFFFFFFFFFFFFFFF, off


class _Dropout(torch.autograd.Function):
    """y = (residual +) dropout(x) (nn.Dropout on hidden states, training mode); masks re-derived in the backward."""

    @staticmethod
    def forward(ctx, x, residual, p, row_tiles):
        ctx.key = next_dropout_key(x.device)
        ctx.p = p
        ctx.has_res = residual is not None
        ctx.row_tiles = row_tiles
        return ops.dropout(x, p, ctx.key[0], ctx.key[1], residual=residual, row_tiles=row_tiles)

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        dx = ops.dropout(dy, ctx.p, ctx.key[0], ctx.key[1], row_tiles=ctx.row_tiles) if _need(ctx, 0) else None
        return dx, (dy if (ctx.has_res and _need(ctx, 1)) else None), None, None


def dropout(x, p, residual=None, row_tiles=None):
    """(residual +) dropout(x) with rate p; p == 0 is the identity (plus the residual add).  row_tiles: x holds packed rows
    (ops.dropout), which take the masks of their padded rows."""
    if not p:
        return x if residual is None else x + residual
    return _Dropout.apply(x, residual, float(p), row_tiles)


class _ClampInf(torch.autograd.Function):
    """The reference's fp16 overflow clamp after a T5 sub-layer (src/modeling_t5.py:657-708), device-side decision.
    Backward: identity (the reference's `torch.clamp` zeroes the gradient of the clamped elements; they only exist in a
    step that overflowed fp16, which the reference's training recipe - bf16 - never takes)."""

    @staticmethod
    def forward(ctx, x):
        y = x.clone()            # outputs of the custom Functions upstream may be views: no in-place edit under autograd
        ops.clamp_inf_(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        return dy


def clamp_inf(x):
    return _ClampInf.apply(x) if x.dtype == torch.float16 else x


class _GatedGelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u):
        ctx.save_for_backward(u)
        return ops.gated_gelu(u)

    @staticmethod
    def backward(ctx, dg):
        (u,) = ctx.saved_tensors
        return ops.gated_gelu(u, dg.contiguous())


def gated_gelu(u):
    return _GatedGelu.apply(u)


class _Relu(torch.autograd.Function):
    """Saves the OUTPUT: the reference applies dropout after the ReLU (wi -> relu -> dropout -> wo), so the mask of the
    backward is the pre-dropout activation's.  The forward is the same select kernel with u as its own mask (u > 0 ? u :
    0); the feed-forward of the model uses `linear_relu`, which needs no separate pass."""

    @staticmethod
    def forward(ctx, u):
        g = ops.relu_bwd(u, u)
        ctx.save_for_backward(g)
        return g

    @staticmethod
    def backward(ctx, dg):
        (g,) = ctx.saved_tensors
        return ops.relu_bwd(g, dg)


def relu(u):
    return _Relu.apply(u)


class _LinearRelu(torch.autograd.Function):
    """g = relu(x @ weight.T) with the ReLU in the GEMM epilogue (EPI_RELU): no pre-activation tensor is written; the
    backward masks dG with the saved output, then runs the Linear's dgrad / wgrad on the masked gradient."""

    @staticmethod
    def forward(ctx, x, weight):
        g = ops.linear(x, weight, epilogue=ops.EPI_RELU)
        ctx.save_for_backward(x, weight, g)
        return g

    @staticmethod
    def backward(ctx, dg):
        x, weight, g = ctx.saved_tensors
        du = ops.relu_bwd(g, dg).reshape(-1, g.shape[-1])
        dx = ops.linear_dgrad(du, weight).reshape(x.shape) if _need(ctx, 0) else None
        dw = ops.linear_wgrad(du, x.reshape(-1, x.shape[-1])) if _need(ctx, 1) else None
        return dx, dw


def linear_relu(x, weight):
    """relu(x @ weight.T), differentiable in x and weight (T5DenseReluDense's wi, src/modeling_t5.py:263-264)."""
    return _LinearRelu.apply(x, weight)


class _GeluErf(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        ctx.save_for_backward(z)
        return ops.gelu_erf(z)

    @staticmethod
    def backward(ctx, dy):
        (z,) = ctx.saved_tensors
        return ops.gelu_erf(z, dy.contiguous())


def gelu_erf(z):
    return _GeluErf.apply(z)


class _Embedding(torch.autograd.Function):
    """rows = table[ids] (cast to out_dtype); backward = fp32 scatter-add of the row gradients (csrc/backward.cu),
    `padding_idx` rows dropped, returned in the table's dtype."""

    @staticmethod
    def forward(ctx, table, ids, padding_idx, out_dtype):
        ctx.save_for_backward(ids)
        ctx.shape, ctx.dtype, ctx.padding_idx = table.shape, table.dtype, padding_idx
        rows = table[ids.reshape(-1)]
        return rows if out_dtype is None else rows.to(out_dtype)

    @staticmethod
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        dt = ops.scatter_add_rows(dy.contiguous(), ctx.shape[0], index=ids, skip_index=ctx.padding_idx)
        return dt.to(ctx.dtype), None, None, None


def embedding(table, ids, padding_idx=-1, out_dtype=None):
    """[n, H] rows of a 16-bit table, or of an fp32 one cast to out_dtype (the gather itself is a torch index: plumbing)."""
    return _Embedding.apply(table, ids, padding_idx, out_dtype)


class _BertEmbedSum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input_ids, token_type_ids, word, type_, pos, pad_id):
        ctx.save_for_backward(input_ids, token_type_ids)
        ctx.meta = (word.shape, type_.shape, pos.shape, word.dtype, pad_id)
        return ops.bert_embed_sum(input_ids, token_type_ids, word, type_, pos)

    @staticmethod
    def backward(ctx, dy):
        input_ids, tts = ctx.saved_tensors
        ws, ts, ps, dt, pad_id = ctx.meta
        B, L = input_ids.shape
        d2 = dy.contiguous().reshape(B * L, -1)
        dword = ops.scatter_add_rows(d2, ws[0], index=input_ids, skip_index=pad_id).to(dt)
        if tts is None:
            tts = torch.zeros_like(input_ids)
        dtype_ = ops.scatter_add_rows(d2, ts[0], index=tts).to(dt)
        dpos = ops.scatter_add_rows(d2, ps[0], modulo=L).to(dt)
        return None, None, dword, dtype_, dpos, None


def bert_embed_sum(input_ids, token_type_ids, word, type_, pos, pad_id=-1):
    return _BertEmbedSum.apply(input_ids, token_type_ids, word, type_, pos, pad_id)


class _MaskedMeanPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask):
        ctx.save_for_backward(mask)
        ctx.shape = x.shape
        return ops.masked_mean_pool(x, mask)

    @staticmethod
    def backward(ctx, demb):
        (mask,) = ctx.saved_tensors
        _, L, H = ctx.shape
        return ops.masked_mean_pool_bwd(demb.contiguous(), mask, L, H), None


def masked_mean_pool(x, mask):
    return _MaskedMeanPool.apply(x, mask)


class _CrossEntropy(torch.autograd.Function):
    """mean over the rows with label != -100 of (logsumexp(logits) - logits[label]), fp32 scalar."""

    @staticmethod
    def forward(ctx, logits, labels):
        lse, rows = ops.cross_entropy_fwd(logits, labels)
        n_valid = (labels.reshape(-1) != -100).sum().to(torch.float32)
        ctx.save_for_backward(logits, labels, lse, n_valid)
        return rows.sum() / n_valid

    @staticmethod
    def backward(ctx, g):
        logits, labels, lse, n_valid = ctx.saved_tensors
        return ops.cross_entropy_bwd(logits, labels, lse, g.to(torch.float32) / n_valid), None


def cross_entropy(logits, labels):
    if logits.dtype not in (torch.float16, torch.bfloat16):
        raise AtlasB200Error("cross_entropy: 16-bit logits expected")
    return _CrossEntropy.apply(logits, labels)
