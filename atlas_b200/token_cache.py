"""Retriever-side passage token cache for index refresh.

`Atlas.build_index` (src/atlas.py:61-88) formats and tokenises EVERY local passage again on every index refresh
(`fstr.format(**p)` + a tokenizer call per 512-passage batch, src/atlas.py:69-76): 4 Mi tokenizer calls' worth of host
work per refresh per GPU at BASELINE configs[2], while the GPU embeds a batch in milliseconds.  Passages do not change
between refreshes - only the retriever's weights do - so the token ids are computed once and kept as one int32 matrix
`ids [N, Lmax]` + `lens [N]` (pinned host memory by default, or on the device); a refresh then slices batches out of
it.  The batches are IDENTICAL to what the tokenizer call of the reference produces (`padding="longest"`: a batch is cut
at its longest passage; `truncation=True, max_length`), which `tests/test_token_cache.py` checks tensor for tensor.
"""
import torch


class RetrieverTokenCache:
    def __init__(self, n, max_len, pad_id=0, device="cpu"):
        self.n, self.max_len, self.pad_id = int(n), int(max_len), int(pad_id)
        self.device = torch.device(device)
        pin = self.device.type == "cpu" and torch.cuda.is_available()
        self.ids = torch.full((self.n, self.max_len), self.pad_id, dtype=torch.int32, device=self.device,
                              pin_memory=pin)
        self.lens = torch.zeros(self.n, dtype=torch.int32, device=self.device, pin_memory=pin)
        self.filled = 0

    def nbytes(self):
        return self.ids.numel() * 4 + self.lens.numel() * 4

    def append(self, input_ids, attention_mask):
        """Store one tokenised batch (`padding="longest"` output of the tokenizer, any device)."""
        b, l = input_ids.shape
        if self.filled + b > self.n or l > self.max_len:
            raise ValueError(f"token cache overflow: batch {tuple(input_ids.shape)} into [{self.n}, {self.max_len}] at {self.filled}")
        rows = slice(self.filled, self.filled + b)
        self.ids[rows, :l] = input_ids.to(self.device, torch.int32)
        self.lens[rows] = attention_mask.sum(dim=1).to(self.device, torch.int32)
        # the cache assumes right padding (what BERT / T5 tokenizers do): the mask must be a prefix of ones
        if not bool((attention_mask.long().cumprod(dim=1).sum(dim=1) == attention_mask.long().sum(dim=1)).all()):
            raise ValueError("token cache needs right-padded batches")
        self.filled += b

    @property
    def complete(self):
        return self.filled == self.n

    def batch(self, start, stop, device=None):
        """(input_ids int64 [b, L], attention_mask int64 [b, L]) of passages [start, stop), padded to the longest
        passage of the batch - the tensors `tokenizer(texts, padding="longest", truncation=True, max_length=...)` returns."""
        lens = self.lens[start:stop]
        longest = int(lens.max()) if stop > start else 0
        ids = self.ids[start:stop, :longest]
        if device is not None:
            ids, lens = ids.to(device, non_blocking=True), lens.to(device, non_blocking=True)
        mask = (torch.arange(longest, device=ids.device)[None, :] < lens[:, None]).to(torch.int64)
        return ids.to(torch.int64), mask


def cache_key(passages, max_len, fmt):
    """Identity of a passage shard for cache reuse: the list object, its length, its first / last passage ids, the format
    and the truncation length."""
    def pid(p):
        return p.get("id") if isinstance(p, dict) else None

    ends = (pid(passages[0]), pid(passages[-1])) if len(passages) else (None, None)
    return (id(passages), len(passages), ends, int(max_len), fmt)


def fits(n, max_len, max_bytes):
    """Whether an [n, max_len] int32 record stays under the configured budget (default 8 GiB of pinned host memory:
    4 Mi passages x 384 tokens = 6.4 GB)."""
    return n * max_len * 4 + n * 4 <= max_bytes


# ----------------------------------------------------------------------------------------------------------------------
# reader side: "query + passage" token rows spliced from cached passage tokens
# ----------------------------------------------------------------------------------------------------------------------
PASSAGE_FIELDS = ("{title}", "{text}", "{id}", "{section}")


def split_encoder_format(fmt):
    """`encoder_format` (default "{query} title: {title} context: {text}", src/options.py) -> (query part, passage part)
    when every passage field comes after the query and the cut falls on white space; None otherwise (no caching)."""
    cuts = [fmt.find(f) for f in PASSAGE_FIELDS if f in fmt]
    if not cuts:
        return None
    pos = min(cuts)
    head, tail = fmt[:pos], fmt[pos:]
    if "{query}" in tail or any(f in head for f in PASSAGE_FIELDS):
        return None
    if pos > 0 and not head[-1].isspace():
        return None
    return head, tail


class ReaderTokenCache:
    """Token ids of the passage part of the reader input, computed once per passage id (`Atlas.tokenize_passages`,
    src/atlas.py:261-280, re-tokenises bsz x n_context strings of ~text_maxlength tokens every step; the passage part is
    the same every time a passage is retrieved).  A step tokenises only the bsz query parts and splices:
        row = (query ids + passage ids)[: max_length - 1] + [eos], padded to max_length
    which equals tokenising the concatenated string for tokenizers that split on white space (exact for the word-level
    tokenizer of the tests; SentencePiece pieces at a white-space cut agree except for normaliser corner cases, hence
    opt-in: `opt.cache_reader_tokens`).  Bounded: at most `max_entries` passages (oldest dropped first)."""

    def __init__(self, tokenizer, encoder_format, max_length, max_entries=1 << 22):
        self.tok = tokenizer
        self.max_length = int(max_length)
        self.parts = split_encoder_format(encoder_format)
        self.max_entries = int(max_entries)
        self.store = {}
        self.hits = self.misses = 0
        eos = getattr(tokenizer, "eos_token_id", None)
        self.eos = 1 if eos is None else int(eos)
        pad = getattr(tokenizer, "pad_token_id", None)
        self.pad = 0 if pad is None else int(pad)

    @property
    def usable(self):
        return self.parts is not None

    def _ids(self, text):
        return list(self.tok(text, add_special_tokens=False)["input_ids"])

    def passage_ids(self, passage):
        key = passage.get("id") if isinstance(passage, dict) else None
        if key is not None and key in self.store:
            self.hits += 1
            return self.store[key]
        self.misses += 1
        ids = self._ids(self.parts[1].format(**passage))[: self.max_length]
        if key is not None:
            if len(self.store) >= self.max_entries:
                self.store.pop(next(iter(self.store)))
            self.store[key] = ids
        return ids

    def encode(self, queries, passages):
        """-> {input_ids, attention_mask} int64 [bsz, n, max_length], what `encode_passages` returns for
        `[[encoder_format.format(query=q, **p) for p in ps] for q, ps in zip(queries, passages)]`."""
        bsz = len(queries)
        n = max(len(ps) for ps in passages)
        L = self.max_length
        ids = torch.full((bsz, n, L), self.pad, dtype=torch.int64)
        mask = torch.zeros((bsz, n, L), dtype=torch.int64)
        for b, (q, ps) in enumerate(zip(queries, passages)):
            q_ids = self._ids(self.parts[0].format(query=q))
            for j in range(n):
                if j < len(ps):
                    row = (q_ids + self.passage_ids(ps[j]))[: L - 1] + [self.eos]
                else:
                    row = [self.eos]                       # the "" padding passage: EOS only (src/atlas.py:26-39)
                ids[b, j, : len(row)] = torch.tensor(row, dtype=torch.int64)
                mask[b, j, : len(row)] = 1
        return {"input_ids": ids, "attention_mask": mask}
