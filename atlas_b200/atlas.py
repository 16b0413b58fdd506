"""Drop-in for `src.atlas.Atlas` (reference src/atlas.py:42-647): the retrieve-then-read step that
`train.py` / `evaluate.py` drive, on top of the B200 index, Contriever and FiD of this package.

Same constructor, method names, argument meaning and return types as the reference class:
`build_index`, `retrieve` / `_retrieve` / `retrieve_with_rerank`, `tokenize` / `retriever_tokenize` /
`reader_tokenize` / `tokenize_passages`, `forward -> (reader_loss, retriever_loss)`, the four gold-score
modes, `kldivloss`, `logprob`, `compute_reader_loss_and_logits`, `generate`.  What is different underneath:

  * `build_index` (src/atlas.py:61-88) writes the pooled fp16 embeddings of every batch straight into the
    bank rows the scan kernel reads (`Contriever.embed_into`) - no `deepcopy().half()` of the retriever per
    call (16-bit weight copies are cached and refreshed when the parameters change), no `[B,768]` temporary,
    no transposed strided write;
  * `_retrieve` embeds the queries with the B200 Contriever kernels and runs the fused scan + top-k
    (`DistributedIndex.search_knn`); the passage dicts come from the node-shared store;
  * the reader passes run on the wgmma FiD kernels (`atlas_b200.fid.FiD`).

Tokenisation, string formatting and the loss arithmetic on `[bsz, n_context]` tensors stay on the host / in
plain torch exactly as the reference does them: they are not on the measured path.
"""
import math
import time
from typing import List, Optional

import numpy as np
import torch
from torch import nn

from . import dist_utils, token_cache
from ._lib import AtlasB200Error
from .index import DistributedFAISSIndex
from .retrievers import EMBEDDINGS_DIM

IGNORE_INDEX: int = -100
BERT_MAX_SEQ_LENGTH: int = 512


def _device():
    if not torch.cuda.is_available():
        raise AtlasB200Error("atlas_b200.Atlas needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _to_cuda(tok_dict):
    """Token dict -> current CUDA device (src/atlas.py:646-647)."""
    if tok_dict is None:
        return None
    dev = _device()
    return {k: v.to(dev, non_blocking=True) for k, v in tok_dict.items()}


def encode_passages(batch, tokenizer, max_length):
    """[bsz][n_i] strings -> {input_ids, attention_mask} of shape [bsz, n, max_length]; short examples are
    padded with "" passages (src/atlas.py:26-39)."""
    bsz = len(batch)
    n = max(len(example) for example in batch)
    flat = []
    for example in batch:
        flat.extend(example)
        flat.extend([""] * (n - len(example)))
    tokens = tokenizer(flat, padding="max_length", max_length=max_length, return_tensors="pt", truncation=True)
    return {k: v.view(bsz, n, -1) for k, v in tokens.items()}


def select_crossattention_scores(scores, mode):
    """Pick the aggregate named after the `eval` / `std` prefix of gold_score_mode (src/atlas.py:639-643)."""
    for prefix in ("eval", "std"):
        if prefix in mode:
            key = mode[len(prefix):]
            if key not in scores and key.startswith("norm") and "norms" + key[4:] in scores:
                # `--gold_score_mode evalnormsum` (= the paper's `adist`, the only eval* choice of src/options.py:244) asks for
                # "normsum", but `aggregate_value(..., prefix="norms")` names the aggregate "normssum" (src/fid.py:162,198):
                # the reference raises KeyError here.  The intended aggregate is served instead.
                key = "norms" + key[4:]
            return scores[key]
    return None


def _unwrap(module):
    return module.module if hasattr(module, "module") else module


class Atlas(nn.Module):
    def __init__(self, opt, reader, retriever, reader_tokenizer, retriever_tokenizer):
        super().__init__()
        self.reader = reader
        self.retriever = retriever
        self.reader_tokenizer = reader_tokenizer
        self.retriever_tokenizer = retriever_tokenizer
        self.opt = opt
        self.READER_ALL_TOKENS = list(self.reader_tokenizer.vocab.values())
        self._token_cache, self._token_cache_key = None, None     # retriever-side passage tokens, kept across refreshes
        self._reader_cache = None                                 # reader-side passage-part tokens (opt.cache_reader_tokens)
        self._token_bank = None                                   # device-resident reader token bank (set_token_bank)

    # ------------------------------------------------------------------------------------------
    # passage side of the retriever: index build / refresh
    # ------------------------------------------------------------------------------------------
    def _passage_tower(self):
        """The Contriever that embeds passages (tied or untied dual encoder, src/retrievers.py:90-135)."""
        r = _unwrap(self.retriever)
        for name in ("passage_contriever", "contriever"):
            if hasattr(r, name):
                return _unwrap(getattr(r, name))
        return r

    def _get_fp16_retriever_copy(self):
        """The reference deep-copies the retriever to fp16 for every build / rerank (src/atlas.py:54-59).  The
        B200 Contriever keeps cached fp16 weight copies itself, so this returns a light view whose call embeds
        passages in fp16 without touching the live (fp32 / bf16) parameters."""
        tower = self._passage_tower()
        if not hasattr(tower, "embed_into"):
            raise AtlasB200Error("atlas_b200.Atlas needs an atlas_b200.retrievers Contriever as passage encoder")

        def embed(input_ids=None, attention_mask=None, is_passages=True, **unused):
            return tower.embed_fp16(input_ids, attention_mask)

        return embed

    @torch.no_grad()
    def build_index(self, index, passages, gpu_embedder_batch_size, logger=None):
        """(Re)embed the local passage shard into the bank IN PLACE (src/atlas.py:61-88).  No communication:
        every rank rewrites its own rows; one barrier at the end like the reference.
        An index with host-resident rows (`is_in_gpu = False`, DistributedFAISSIndex) gets every batch embedded into one
        of two device staging buffers and copied to its rows asynchronously; it is then marked stale and retrained."""
        tower = self._passage_tower()
        bank = getattr(index, "_bank", None)
        if bank is None or not hasattr(tower, "embed_into"):
            raise AtlasB200Error("build_index needs atlas_b200.index.DistributedIndex.init_embeddings() first and "
                                 "an atlas_b200 Contriever passage encoder")
        fmt = self.opt.retriever_format
        max_len = min(self.opt.text_maxlength, gpu_embedder_batch_size)
        total = 0
        n_batch = math.ceil(len(passages) / gpu_embedder_batch_size)
        # token cache (atlas_b200/token_cache.py): the first build tokenises like the reference and records the ids; later
        # refreshes of the SAME passage shard slice identical batches out of the record instead of re-tokenising
        use_cache = bool(getattr(self.opt, "cache_retriever_tokens", True)) and len(passages) > 0 and token_cache.fits(
            len(passages), max_len, int(getattr(self.opt, "token_cache_max_bytes", 8 << 30)))
        key = token_cache.cache_key(passages, max_len, fmt)
        cache = self._token_cache if (use_cache and self._token_cache_key == key and self._token_cache is not None
                                      and self._token_cache.complete) else None
        record = None
        host = not getattr(index, "is_in_gpu", True)
        stage = [torch.empty((gpu_embedder_batch_size, EMBEDDINGS_DIM), dtype=torch.float16, device=_device())
                 for _ in range(2)] if host else None
        if use_cache and cache is None:
            record = token_cache.RetrieverTokenCache(len(passages), max_len, device=getattr(self.opt, "token_cache_device", "cpu"))
        for i in range(n_batch):
            a, b = i * gpu_embedder_batch_size, min(len(passages), (i + 1) * gpu_embedder_batch_size)
            if cache is not None:
                ids, mask = cache.batch(a, b, device=_device())
                enc = {"input_ids": ids, "attention_mask": mask}
            else:
                chunk = passages[a:b]
                enc = self.retriever_tokenizer([fmt.format(**p) for p in chunk], padding="longest", return_tensors="pt",
                                               max_length=max_len, truncation=True)
                if record is not None:
                    record.append(enc["input_ids"], enc["attention_mask"])
                enc = _to_cuda(enc)
            rows = stage[i & 1][:b - a] if host else bank[total:total + (b - a)]
            tower.embed_into(enc["input_ids"], enc["attention_mask"], rows, dtype=torch.float16)
            if host:    # stream-ordered: the staging buffer is rewritten two batches later, after this copy
                bank[total:total + (b - a)].copy_(rows, non_blocking=True)
            total += b - a
            if logger is not None and i % 500 == 0 and i > 0:
                logger.info(f"Number of passages encoded: {total}")
        if record is not None and record.complete:
            self._token_cache, self._token_cache_key = record, key
        if host:
            torch.cuda.current_stream().synchronize()
            index.mark_stale()
        dist_utils.barrier()
        if logger is not None:
            logger.info(f"{total} passages encoded on process: {dist_utils.get_rank()}")
        if not index.is_index_trained():
            index.train_index()

    # ------------------------------------------------------------------------------------------
    # retrieval
    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _retrieve(self, index, topk, query, query_ids_retriever, query_mask_retriever, batch_metadata=None,
                  filtering_fun=None, iter_stats={}):
        """Query embedding + distributed exact search (src/atlas.py:90-118).  Collective: ranks with an empty
        batch still call `search_knn` (with 0 query rows)."""
        self.retriever.eval()
        if len(query) > 0:
            query_emb = self.retriever(query_ids_retriever, query_mask_retriever, is_passages=False)
        else:
            query_emb = torch.empty((0, EMBEDDINGS_DIM), device=_device())
        if self.training:
            self.retriever.train()
        t0 = time.time()
        cap = getattr(self.opt, "per_gpu_batch_size", None)
        if cap and getattr(index, "max_queries_per_rank", 0) is None and len(query) <= cap:
            # every rank runs the same options: the per-GPU batch size bounds the queries of any rank, which lets the
            # distributed search skip its size exchange (index.py: `max_queries_per_rank`)
            index.max_queries_per_rank = int(cap)
        refine = getattr(self.opt, "faiss_refine_factor", None)
        if refine is not None and hasattr(index, "refine_factor"):
            # --index_mode faiss: re-rank refine * topk PQ candidates per rank by exact score (the flat index is exact)
            index.refine_factor = int(refine)
        if isinstance(index, DistributedFAISSIndex):
            # --index_mode faiss: score each query against its best faiss_nprobe inverted lists only (None: every list)
            index.nprobe = getattr(self.opt, "faiss_nprobe", None)
        if filtering_fun is not None:
            passages, scores = index.search_knn(query_emb, topk * self.opt.filtering_overretrieve_ratio)
            passages, scores = filtering_fun(batch_metadata, passages, scores, topk, training=self.training)
        else:
            passages, scores = index.search_knn(query_emb, topk)
        iter_stats["runtime/search"] = (time.time() - t0, 1)
        return passages, scores, query_emb

    @torch.no_grad()
    def retrieve_with_rerank(self, index, topk, query, query_ids_retriever, query_mask_retriever, batch_metadata=None,
                             filtering_fun=None, iter_stats={}):
        """Retrieve `n_to_rerank_with_retrieve_with_rerank` candidates from the (possibly stale) index, re-embed
        them with the CURRENT passage encoder in fp16 and keep the top-k by fresh score (src/atlas.py:120-176)."""
        bsz = len(query)
        n_cand = self.opt.n_to_rerank_with_retrieve_with_rerank
        passages, _, query_emb = self._retrieve(index, n_cand, query, query_ids_retriever, query_mask_retriever,
                                                batch_metadata, filtering_fun, iter_stats)
        embed = self._get_fp16_retriever_copy()
        fmt = self.opt.retriever_format
        strings = [fmt.format(**p) for ps in passages for p in ps]
        step = max(1, min(len(strings), self.opt.per_gpu_embedder_batch_size))
        passage_emb = query_emb.new_zeros(len(strings), query_emb.shape[-1])
        for b in range(0, len(strings), step):
            enc = self.retriever_tokenizer(strings[b:b + step], padding="longest", return_tensors="pt",
                                           max_length=min(self.opt.text_maxlength, BERT_MAX_SEQ_LENGTH),
                                           truncation=True)
            passage_emb[b:b + step] = embed(**_to_cuda(enc), is_passages=True).to(query_emb)
        fresh = torch.einsum("id, ijd->ij", [query_emb, passage_emb.view(bsz, n_cand, -1)])
        top_scores, top_inds = torch.topk(fresh, topk, dim=1)
        top_inds = top_inds.tolist()
        out_passages = [[passages[i][j] for j in top_inds[i]] for i in range(bsz)]
        return out_passages, top_scores.tolist()

    @torch.no_grad()
    def retrieve(self, *args, **kwargs):
        fn = self.retrieve_with_rerank if self.opt.retrieve_with_rerank else self._retrieve
        return fn(*args, **kwargs)[:2]

    # ------------------------------------------------------------------------------------------
    # tokenisation (host; same tokenizer calls as the reference)
    # ------------------------------------------------------------------------------------------
    def append_query(self, query, passages):
        return [self.opt.encoder_format.format(query=query, **p) for p in passages]

    def retriever_tokenize(self, query):
        """src/atlas.py:187-199: queries padded to min(text_maxlength, 512)."""
        if not self.retriever_tokenizer:
            return None
        enc = self.retriever_tokenizer(query, max_length=min(self.opt.text_maxlength, BERT_MAX_SEQ_LENGTH),
                                       padding="max_length", truncation=True, return_tensors="pt")
        return _to_cuda(enc)

    def _prompt_mask(self, prompts):
        return self.reader_tokenizer(prompts, max_length=self.opt.target_maxlength, padding="max_length",
                                     truncation=True, return_tensors="pt", add_special_tokens=False)["attention_mask"]

    def reader_tokenize(self, query, target, target_tokens):
        """Targets -> (labels with pads = -100, decoder_input_ids = shift_right) on the device
        (src/atlas.py:201-246); with a decoder prompt the prompt positions are masked out of the labels."""
        prompts = None
        if target_tokens is None:
            if self.opt.decoder_prompt_format is not None:
                prompts = [self.opt.decoder_prompt_format.format_map({"query": q}) for q in query]
                target = [p + t for p, t in zip(prompts, target)]
            if self.opt.decoder_format is not None:
                target = [self.opt.decoder_format.format(target=t) for t in target]
            target = [t if t.endswith("</s>") else t + "</s>" for t in target]
            target_tokens = self.reader_tokenizer(target, max_length=self.opt.target_maxlength, padding="max_length",
                                                  truncation=True, return_tensors="pt", add_special_tokens=False)
        ids = target_tokens["input_ids"]
        decoder_input_ids = self.reader._shift_right(ids)
        labels = ids.masked_fill(~target_tokens["attention_mask"].bool(), IGNORE_INDEX)
        if self.opt.decoder_prompt_format is not None:
            if prompts is None:
                prompts = [self.opt.decoder_prompt_format.format_map({"query": q}) for q in query]
            pm = self._prompt_mask(prompts)
            pad = torch.zeros((pm.size(0), ids.size(-1) - pm.size(-1)), dtype=pm.dtype)
            labels = labels.masked_fill(torch.cat([pm, pad], dim=1).bool(), IGNORE_INDEX)
        dev = _device()
        return labels.to(dev), decoder_input_ids.to(dev)

    def tokenize(self, query, target, target_tokens):
        if query is None and target is None:
            return None, None, None
        assert (target_tokens is None or self.opt.decoder_prompt_format is None
                ), "decoder_prompt_format not compatible with target tokenized in iterator"
        query_enc = self.retriever_tokenize(query) if not self.opt.use_file_passages else None
        labels, decoder_input_ids = self.reader_tokenize(query, target, target_tokens)
        return query_enc, labels, decoder_input_ids

    def reader_passage_tokens(self, query, passages):
        """Reader tokens of "query + passage", [bsz, n, text_maxlength] ids + mask on the device (the first half of
        `tokenize_passages`, src/atlas.py:261-270).  With a device token bank attached (`set_token_bank`) the rows are
        assembled on the GPU from the passage ids; otherwise the reference's host tokenisation runs."""
        reader_tok = None
        bank = getattr(self, "_token_bank", None)
        if bank is not None and getattr(self.opt, "device_token_bank", True):
            n = max(len(ps) for ps in passages)
            gids = torch.tensor([[int(p["id"]) for p in ps] + [-1] * (n - len(ps)) for ps in passages], dtype=torch.int64)
            q_ids, q_lens = bank.query_tokens(self.reader_tokenizer, query, _device())
            reader_tok = bank.splice(gids.to(_device(), non_blocking=True), self.opt.text_maxlength, q_ids, q_lens)
        if reader_tok is None and getattr(self.opt, "cache_reader_tokens", False):
            # opt-in: passage parts tokenised once per passage id, spliced behind the query part (token_cache.py)
            rc = self._reader_cache
            if rc is None or rc.max_length != self.opt.text_maxlength:
                rc = self._reader_cache = token_cache.ReaderTokenCache(self.reader_tokenizer, self.opt.encoder_format,
                                                                       self.opt.text_maxlength)
            if rc.usable:
                reader_tok = _to_cuda(rc.encode(query, passages))
        if reader_tok is None:
            reader_text = [self.append_query(q, ps) for q, ps in zip(query, passages)]
            reader_tok = _to_cuda(encode_passages(reader_text, self.reader_tokenizer, self.opt.text_maxlength))
        return reader_tok

    def tokenize_passages(self, query, passages):
        """Reader tokens of "query + passage" ([bsz, n, text_maxlength]) and retriever tokens of the passages
        ([bsz, n, min(text_maxlength, 512)]) (src/atlas.py:261-280)."""
        if len(query) == 0:
            return None, None
        retriever_tok = None
        if self.retriever_tokenizer:
            fmt = self.opt.retriever_format
            retriever_text = [[fmt.format(**p) for p in ps] for ps in passages]
            retriever_tok = _to_cuda(encode_passages(retriever_text, self.retriever_tokenizer,
                                                     min(self.opt.text_maxlength, BERT_MAX_SEQ_LENGTH)))
        return self.reader_passage_tokens(query, passages), retriever_tok

    def set_token_bank(self, bank):
        """Attach a `token_bank.DeviceTokenBank` (reader-side passage tokens on the GPU, keyed by the passages' integer
        "id"): `tokenize_passages` then assembles the reader input on the device instead of tokenising
        bsz x n_context strings per step (src/atlas.py:261-280).  None detaches it."""
        self._token_bank = bank

    # ------------------------------------------------------------------------------------------
    # gold scores for retriever distillation
    # ------------------------------------------------------------------------------------------
    def _reader_per_passage(self, reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz, n_ctx,
                            with_decoder_inputs=True):
        """One reader pass in which every (query, passage) pair is its own example (`n_context = 1`,
        `bsz = bsz * n_ctx`): the shape both ppmean and emdr scoring use (src/atlas.py:282-296,379-396)."""
        cfg.n_context = 1
        cfg.bsz = bsz * n_ctx
        rep_labels = torch.repeat_interleave(labels, n_ctx, dim=0)
        kw = {}
        if with_decoder_inputs:
            kw["decoder_input_ids"] = torch.repeat_interleave(decoder_input_ids, n_ctx, dim=0)
        out = self.reader(input_ids=reader_ids.reshape(bsz * n_ctx, -1), attention_mask=reader_mask.reshape(bsz * n_ctx, -1),
                          labels=rep_labels, use_cache=False, **kw)
        return out, rep_labels

    def perplexity_score(self, reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz):
        """ppmean (default gold_score_mode): minus the mean token cross-entropy of the target given each passage
        alone -> [bsz, n] (src/atlas.py:282-308)."""
        with torch.no_grad():
            self.reader.eval()
            n_ctx = reader_ids.size(1)
            out, rep_labels = self._reader_per_passage(reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz, n_ctx)
            logits = out.logits
            token_loss = nn.functional.cross_entropy(logits.view(-1, logits.size(-1)), rep_labels.flatten(),
                                                     reduction="none")
            n_tok = (rep_labels.view(bsz, n_ctx, -1) > -1).sum(dim=-1)
            return -token_loss.view(bsz, n_ctx, -1).sum(dim=-1) / n_tok

    def eval_score(self, reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz, mask_query):
        """Cross-attention based gold scores (src/atlas.py:310-340); needs the reader's score capture."""
        self.reader.eval()
        self.reader.reset_score_storage()
        cfg.bsz = reader_ids.size(0)
        cfg.n_context = reader_ids.size(1)
        ids2 = reader_ids.view(reader_ids.size(0), -1)
        mask2 = reader_mask.view(reader_mask.size(0), -1)
        with torch.no_grad():
            self.reader(input_ids=ids2, attention_mask=mask2, decoder_input_ids=decoder_input_ids, labels=labels,
                        use_cache=False)
            agg = self.reader.get_crossattention_scores(cfg.n_context, mask2, labels=labels, ids=reader_ids,
                                                        mode=self.opt.gold_score_mode, mask_query=mask_query)
            gold = select_crossattention_scores(agg, self.opt.gold_score_mode)
        if self.training:
            self.reader.train()
        return gold

    def loop_score(self, reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz):
        """Leave-one-out: encode once, then one decoder pass per passage with that passage masked out; score =
        mean token loss without it -> [bsz, n] (src/atlas.py:342-376)."""
        with torch.no_grad():
            n_ctx, doc_len = reader_ids.size(1), reader_ids.size(-1)
            self.reader.eval()
            cfg.bsz, cfg.n_context = bsz, n_ctx
            full = self.reader(input_ids=reader_ids.view(bsz, -1), attention_mask=reader_mask.view(bsz, -1),
                               decoder_input_ids=decoder_input_ids, labels=labels, use_cache=False)
            enc = full.encoder_last_hidden_state
            n_tok = (labels > -1).sum(-1)
            cols = []
            for drop in range(n_ctx):
                m = reader_mask.clone()
                m[:, drop] = False
                out = self.reader(encoder_outputs=[enc], attention_mask=m.view(bsz, n_ctx * doc_len),
                                  decoder_input_ids=decoder_input_ids, labels=labels, use_cache=False)
                tl = nn.functional.cross_entropy(out.logits.view(-1, out.logits.size(-1)), labels.view(-1),
                                                 reduction="none")
                cols.append(tl.view(bsz, labels.shape[-1]).sum(dim=-1) / n_tok)
            return torch.stack(cols, dim=1)

    @torch.no_grad()
    def emdr_score(self, reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz):
        """EMDR2: per-passage reader logits [bsz * n, T, vocab] (src/atlas.py:378-397)."""
        self.reader.eval()
        out, _ = self._reader_per_passage(reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz,
                                          self.opt.retriever_n_context, with_decoder_inputs=False)
        return out.logits

    # ------------------------------------------------------------------------------------------
    # the step
    # ------------------------------------------------------------------------------------------
    def forward(self, index, query, target, target_tokens=None, passages=None, batch_metadata=None, filtering_fun=None,
                use_cache=False, train_retriever=False, iter_stats={}):
        """Retrieve -> read -> losses (src/atlas.py:399-550).  Returns (reader_loss, retriever_loss or None) and
        fills `iter_stats[key] = (value, weight)`."""
        t_start = time.time()
        bsz = len(query)
        opt = self.opt
        query_mask_reader = self.reader_tokenizer.batch_encode_plus(
            query, max_length=opt.text_maxlength, padding="longest", truncation=True, return_tensors="pt",
            add_special_tokens=False)["attention_mask"].bool().to(_device())
        query_enc, labels, decoder_input_ids = self.tokenize(query, target, target_tokens)

        if not opt.use_file_passages:
            t0 = time.time()
            passages, _ = self.retrieve(index, opt.retriever_n_context, query, query_enc["input_ids"],
                                        query_enc["attention_mask"], batch_metadata=batch_metadata,
                                        filtering_fun=filtering_fun, iter_stats=iter_stats)
            iter_stats["runtime/retrieve"] = (time.time() - t0, 1)

        reader_tokens, retriever_tokens = self.tokenize_passages(query, passages)
        reader_ids = reader_tokens["input_ids"]
        reader_mask = reader_tokens["attention_mask"].bool()
        n_ctx_train = min(opt.n_context, reader_ids.size(1))
        cfg = self.reader.encoder.config
        mode = opt.gold_score_mode

        retriever_loss, gold_score, retriever_score, query_emb = None, None, None, None
        if train_retriever:
            if opt.use_gradient_checkpoint_retriever:
                self.retriever.gradient_checkpointing_enable()
            query_emb = self.retriever(**query_enc, is_passages=False)
            if "std" in mode:
                retriever_tokens = {k: v[:, :n_ctx_train] for k, v in retriever_tokens.items()}
            flat = {k: v.reshape(-1, v.size(-1)) for k, v in retriever_tokens.items()}
            passage_emb = self.retriever(**flat, is_passages=True).to(query_emb)
            retriever_score = torch.einsum("id, ijd->ij", [query_emb, passage_emb.view(bsz, -1, passage_emb.size(-1))])
            if opt.use_gradient_checkpoint_retriever:
                self.retriever.gradient_checkpointing_disable()
            if "eval" in mode:
                gold_score = self.eval_score(reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz, query_mask_reader)
            elif "loop" in mode:
                gold_score = self.loop_score(reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz)
            elif "ppmean" in mode:
                gold_score = self.perplexity_score(reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz)
            elif "emdr" in mode:
                gold_score = self.emdr_score(reader_ids, reader_mask, decoder_input_ids, labels, cfg, bsz)
            self.reader.reset_score_storage()
            if self.training:
                self.reader.train()

        cfg.bsz, cfg.n_context = reader_ids.size(0), n_ctx_train
        ids_train = reader_ids[:, :n_ctx_train].contiguous().view(bsz, -1)
        mask_train = reader_mask[:, :n_ctx_train].contiguous().view(bsz, -1)
        if opt.use_gradient_checkpoint_reader:
            self.reader.gradient_checkpointing_enable()
        reader_output = self.reader(input_ids=ids_train, attention_mask=mask_train, decoder_input_ids=decoder_input_ids,
                                    labels=labels, use_cache=False)
        reader_loss = reader_output[0]
        if opt.use_gradient_checkpoint_reader:
            self.reader.gradient_checkpointing_disable()

        if train_retriever:
            xattn = None
            if opt.compute_crossattention_stats or "std" in mode:
                xattn = self.reader.get_crossattention_scores(n_ctx_train, mask_train, ids=ids_train,
                                                              mask_query=query_mask_reader, labels=labels, mode="all")
            if "std" in mode:
                gold_score = select_crossattention_scores(xattn, mode).detach()
            retriever_score = retriever_score / np.sqrt(query_emb.size(-1))
            if opt.compute_crossattention_stats:
                with torch.no_grad():
                    for key, val in xattn.items():
                        corr = torch.corrcoef(torch.stack([gold_score.view(-1), val.view(-1)]))[0, 1].item()
                        iter_stats[f"corr/{key}"] = (0.0 if np.isnan(corr) else corr, len(query))
            if gold_score is not None:
                gold_score, retriever_score = gold_score.float(), retriever_score.float()
                if mode == "emdr":
                    retriever_loss = self.logprob(retriever_score, gold_score, labels)
                else:
                    retriever_loss = self.kldivloss(retriever_score, gold_score)

        self.reader.reset_score_storage()
        iter_stats["loss/reader_loss"] = (reader_loss.item(), len(query))
        if retriever_loss is not None:
            iter_stats["loss/retriever_loss"] = (retriever_loss.item(), len(query))
        iter_stats["runtime/forward"] = (time.time() - t_start, 1)
        return reader_loss, retriever_loss

    def kldivloss(self, score, gold_score):
        """KL(softmax(gold / tau_g) || softmax(score / tau_s)) with KLDivLoss's default element-mean reduction
        (src/atlas.py:552-555)."""
        target = torch.softmax(gold_score / self.opt.temperature_gold, dim=-1)
        logp = torch.nn.functional.log_softmax(score / self.opt.temperature_score, dim=-1)
        return torch.nn.KLDivLoss()(logp, target)

    def logprob(self, score, gold_score, labels):
        """EMDR2 objective: -mean_t log sum_j p_reader(y_t | passage j) p_retriever(j) (src/atlas.py:557-575)."""
        n = self.opt.retriever_n_context
        with torch.no_grad():
            rep = torch.repeat_interleave(labels, n, dim=0)
            rep[rep == IGNORE_INDEX] = 0
            valid = labels >= 0
            glp = torch.nn.functional.log_softmax(gold_score / self.opt.temperature_gold, dim=-1)
            glp = torch.gather(glp, dim=-1, index=rep[..., None]).view(glp.size(0), -1)
            glp = glp.view(score.size(0), score.size(1), -1)
        log_score = torch.nn.functional.log_softmax(score / self.opt.temperature_score, dim=-1)
        marg = torch.logsumexp(glp + log_score[..., None], dim=1)
        return -1 * torch.sum(marg * valid) / torch.sum(valid)

    @torch.no_grad()
    def compute_reader_loss_and_logits(self, tokens, decoder_input_ids, labels):
        """src/atlas.py:577-590."""
        ids, mask = tokens["input_ids"], tokens["attention_mask"]
        cfg = self.reader.encoder.config
        cfg.bsz = ids.size(0)
        cfg.n_context = min(self.opt.n_context, ids.size(1))
        dev = _device()
        out = self.reader(input_ids=ids.to(dev).view(ids.size(0), -1), attention_mask=mask.to(dev).view(mask.size(0), -1),
                          decoder_input_ids=decoder_input_ids.to(dev), labels=labels.to(dev), use_cache=False)
        return out[0].cpu().item(), out[1]

    @torch.no_grad()
    def generate(self, tokens, query, choices=None):
        """src/atlas.py:592-619."""
        cfg = self.reader.encoder.config
        cfg.bsz = tokens["input_ids"].size(0)
        cfg.n_context = min(self.opt.n_context, tokens["input_ids"].size(1))
        dev = _device()
        flat = {k: v.view(v.size(0), -1).to(dev) for k, v in tokens.items()}
        allowed_fn = None
        if self.opt.decoder_prompt_format is not None:
            prefixes = [self.opt.decoder_prompt_format.format_map({"query": q}) for q in query]
            allowed_fn = self.get_prefix_allowed_tokens_fn(prefixes)
        return self.reader.generate(input_ids=flat["input_ids"], attention_mask=flat["attention_mask"],
                                    num_return_sequences=1, max_length=self.opt.generation_max_length,
                                    min_length=self.opt.generation_min_length,
                                    num_beams=self.opt.generation_num_beams,
                                    length_penalty=self.opt.generation_length_penalty, forced_bos_token_id=None,
                                    prefix_allowed_tokens_fn=allowed_fn,
                                    cross_kv_dtype=getattr(self.opt, "generation_cross_kv_dtype", None))

    def get_prefix_allowed_tokens_fn(self, prefix_str: Optional[List[str]] = None):
        """Force the decoder prompt: while the generated prefix is shorter than the prompt only the next prompt
        token is allowed, afterwards the whole vocabulary (src/atlas.py:621-636)."""
        if not prefix_str:
            return None
        prompt_ids = self.reader_tokenizer.batch_encode_plus(prefix_str, add_special_tokens=False)["input_ids"]

        def allowed(batch_id: int, input_ids: torch.Tensor):
            pos = input_ids.shape[-1]
            if pos > len(prompt_ids[batch_id]):
                return self.READER_ALL_TOKENS
            return prompt_ids[batch_id][pos - 1]

        return allowed
