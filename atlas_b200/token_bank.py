"""Device-resident reader token bank.

`Atlas.tokenize_passages` (src/atlas.py:261-280) formats and tokenises bsz x n_context "query + passage" strings of
~text_maxlength tokens on the host EVERY step and copies [bsz, n, L] int64 ids + mask to the device; at
BASELINE configs[3] (8 x 40 x 384) that host work is of the order of the whole GPU step.  The passage part of a row is
the same every time a passage is retrieved, so it is tokenised ONCE per passage into an int32 matrix on the GPU
(`ids [N, Lp]`, `lens [N]`, keyed by global passage id); a step tokenises only the bsz query parts and one kernel
(`atlas_b200_splice_tokens`, csrc/elementwise.cu) assembles
    row = (query ids ++ passage ids)[: L - 1] ++ [eos], padded            (+ the attention mask)
on the device.  This equals tokenising the concatenated string for tokenizers that split on white space (exact for the
word-level tokenizer of the tests; SentencePiece agrees at a white-space cut except for normaliser corner cases), hence
opt-in: `opt.device_token_bank = True` (INTEGRATION.md).

The bank is REPLICATED on every rank (retrieved passages come from any shard): 4 Mi passages x 256 tokens x 4 B =
4.3 GB of the 180 GB; rows are addressed by global passage id.
"""
import ctypes

import torch

from ._lib import AtlasB200Error, check, current_stream_ptr, lib, require_cuda
from .token_cache import split_encoder_format


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class DeviceTokenBank:
    def __init__(self, ids, lens, eos_id=1, pad_id=0, parts=None):
        require_cuda(ids, "token bank ids")
        if ids.dtype != torch.int32 or lens.dtype != torch.int32 or ids.dim() != 2 or lens.shape[0] != ids.shape[0]:
            raise AtlasB200Error("DeviceTokenBank: ids int32 [N, Lp] and lens int32 [N] expected")
        self.ids, self.lens = ids.contiguous(), lens.contiguous()
        self.eos_id, self.pad_id = int(eos_id), int(pad_id)
        self.parts = parts          # (query part, passage part) of encoder_format, None = raw rows

    @property
    def rows(self):
        return self.ids.shape[0]

    def nbytes(self):
        return self.ids.numel() * 4 + self.lens.numel() * 4

    @classmethod
    def build(cls, passages_by_gid, tokenizer, encoder_format, max_passage_tokens, device, batch=4096):
        """Tokenise the passage part of `encoder_format` for every passage ONCE.  `passages_by_gid`: sequence indexed by
        global passage id (every rank passes the whole corpus; the bank is replicated)."""
        parts = split_encoder_format(encoder_format)
        if parts is None:
            raise AtlasB200Error(f"encoder_format {encoder_format!r} cannot be split into a query and a passage part at "
                                 "white space: the device token bank is not usable with it")
        n = len(passages_by_gid)
        ids = torch.full((n, max_passage_tokens), 0, dtype=torch.int32)
        lens = torch.zeros(n, dtype=torch.int32)
        for a in range(0, n, batch):
            b = min(n, a + batch)
            texts = [parts[1].format(**passages_by_gid[i]) for i in range(a, b)]
            enc = tokenizer(texts, add_special_tokens=False)["input_ids"]
            for i, row in enumerate(enc):
                row = row[:max_passage_tokens]
                ids[a + i, : len(row)] = torch.tensor(row, dtype=torch.int32)
                lens[a + i] = len(row)
        eos = getattr(tokenizer, "eos_token_id", None)
        pad = getattr(tokenizer, "pad_token_id", None)
        return cls(ids.to(device), lens.to(device), 1 if eos is None else eos, 0 if pad is None else pad, parts)

    def query_tokens(self, tokenizer, queries, device):
        """Token ids of the query part of every row (host tokenisation of bsz short strings) -> (ids int64 [B, Lq], lens)."""
        head = self.parts[0] if self.parts is not None else "{query}"
        enc = tokenizer([head.format(query=q) for q in queries], add_special_tokens=False)["input_ids"]
        width = max(1, max((len(r) for r in enc), default=1))
        ids = torch.zeros((len(enc), width), dtype=torch.int64)
        lens = torch.zeros(len(enc), dtype=torch.int32)
        for i, r in enumerate(enc):
            ids[i, : len(r)] = torch.tensor(r, dtype=torch.int64)
            lens[i] = len(r)
        return ids.to(device, non_blocking=True), lens.to(device, non_blocking=True)

    @torch.no_grad()
    def splice(self, gids, text_maxlength, query_ids=None, query_lens=None):
        """gids int64 [B, n] global passage ids on the device (< 0 = padding passage) -> {input_ids int64 [B, n, L],
        attention_mask bool [B, n, L]} on the device: what `encode_passages(..., reader_tokenizer, text_maxlength)` returns
        (src/atlas.py:26-39,270-280), without leaving the GPU."""
        require_cuda(gids, "gids")
        B, n = gids.shape
        L = int(text_maxlength)
        g = gids.to(torch.int64).contiguous()
        out_ids = torch.empty((B, n, L), dtype=torch.int64, device=gids.device)
        out_mask = torch.empty((B, n, L), dtype=torch.bool, device=gids.device)
        q = query_ids.contiguous() if query_ids is not None else None
        ql = query_lens.to(torch.int32).contiguous() if query_lens is not None else None
        check(lib().atlas_b200_splice_tokens(_ptr(self.ids), _ptr(self.lens), self.ids.stride(0), self.rows, _ptr(g), _ptr(q),
                                             _ptr(ql), q.stride(0) if q is not None else 0, B, n, L, self.eos_id,
                                             self.pad_id, _ptr(out_ids), _ptr(out_mask), current_stream_ptr()))
        return {"input_ids": out_ids, "attention_mask": out_mask}
