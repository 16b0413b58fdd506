"""numpy restatement of transformers 4.18 `beam_search` (the version the reference pins) for `FiD.generate(num_beams > 1)`:
the logits processors after the log-softmax (MinLength, PrefixConstrained), the fp32 beam scores, the top-2nb over
[nb * V] per batch element, `BeamSearchScorer.process`, `BeamHypotheses` (add / is_done with early_stopping=False) and
`finalize` with one returned sequence.

The step logits come from a callback (or are fed step by step), so the same oracle checks the selection kernels on synthetic
logits and whole generations on the logits the GPU computed for its beams.  Modes:
  mode="fp64"            log-probs and beam scores in fp64 (the exact-arithmetic restatement);
  mode="fp16" / "bf16"   log-probs rounded to that 16-bit type (4.18's log_softmax returns the logits' dtype when the
                         parameters are 16-bit), beam scores and their sums in fp32, as 4.18 computes them;
  mode="fp32"            log-probs rounded to fp32, fp32 sums (4.18 with fp32 parameters);
  step(logprobs=...)     processed log-probs supplied directly (summed in the mode's precision), for checking the
                         selection logic alone.

Order of candidates (torch.topk leaves ties undefined; the kernels define it): the larger score first, NaN above every number,
among equal scores (or NaNs) the lower flat index beam * V + token.

Every step records a margin: the smallest gap that decided something - between consecutive ranks of the top 2nb + 1
candidates, between a new hypothesis and the worst kept one, and between the worst hypothesis and the is_done bound (in
sum-of-log-prob units) - together with the log-prob magnitude of the candidates at that gap, so a caller can tell decisions
that a one-ulp change of a 16-bit log-prob could flip."""
import numpy as np


def round_to(x, mode):
    """float64 array -> float64 array of the nearest `mode` values (round to nearest even)."""
    x = np.asarray(x, dtype=np.float64)
    if mode == "fp16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).astype(np.float64)
    if mode == "bf16":
        f = x.astype(np.float32)
        u = f.view(np.uint32).astype(np.uint64)
        r = (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32)
        out = r.view(np.float32).astype(np.float64)
        return np.where(np.isnan(x), x, out)
    if mode == "fp32":
        return x.astype(np.float32).astype(np.float64)
    if mode in ("fp64", None):
        return x
    raise ValueError(f"unknown mode {mode!r}")


def ulp16(x, mode):
    """Spacing of the 16-bit type at |x| (its subnormal spacing below the normal range)."""
    mant, emin = (7, -126) if mode == "bf16" else (10, -14)
    a = np.maximum(np.abs(np.asarray(x, dtype=np.float64)), 2.0 ** emin)
    return np.exp2(np.floor(np.log2(a)) - mant)


def log_softmax(logits):
    """float64 log_softmax per row; a row of -inf (or with a NaN) gives NaN everywhere, as torch does."""
    x = np.asarray(logits, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        m = x.max(axis=-1, keepdims=True)
        z = x - m
        return z - np.log(np.exp(z).sum(axis=-1, keepdims=True))


def rank_order(scores):
    """Indices of a 1-D score array in candidate order: NaN first, then descending, ties by the lower index."""
    s = np.asarray(scores, dtype=np.float64)
    nan = np.isnan(s)
    neg = np.where(nan, 0.0, -s)
    return np.lexsort((np.arange(s.size), neg, ~nan))


def length_norm(length, length_penalty):
    return length ** length_penalty                 # Python's int ** float, as 4.18 computes it


class Hypotheses:
    """BeamHypotheses (4.18): at most nb (score, tokens) in list order; worst_score starts at 1e9."""

    def __init__(self, nb, length_penalty):
        self.nb, self.length_penalty = nb, length_penalty
        self.beams = []
        self.worst = 1e9

    def __len__(self):
        return len(self.beams)

    def add(self, tokens, sum_logprobs):
        """Returns the margin of the decision when the list was full (|score - worst| times the normaliser), else None."""
        denom = length_norm(len(tokens), self.length_penalty)
        score = sum_logprobs / denom
        margin = abs(score - self.worst) * denom if len(self.beams) >= self.nb else None
        if len(self.beams) < self.nb or score > self.worst:
            self.beams.append((score, list(tokens)))
            if len(self.beams) > self.nb:
                order = sorted([(s, i) for i, (s, _) in enumerate(self.beams)])
                del self.beams[order[0][1]]
                self.worst = order[1][0]
            else:
                self.worst = min(score, self.worst)
        return margin

    def is_done(self, best_sum_logprobs, cur_len):
        if len(self.beams) < self.nb:
            return False, None
        denom = length_norm(cur_len, self.length_penalty)
        bound = best_sum_logprobs / denom
        return self.worst >= bound, abs(self.worst - bound) * denom


class BeamSearch:
    """One beam search over B batch elements and nb beams: feed `step` the [B * nb, V] logits of the current beams
    (row b * nb + k) until `finished`, then `finalize`."""

    def __init__(self, B, nb, V, max_length, min_length=None, length_penalty=1.0, mode="fp64", eos=1, pad=0, start=0,
                 prefix_fn=None):
        self.B, self.nb, self.V = B, nb, V
        self.max_length = int(max_length)
        self.min_length = 0 if min_length is None else int(min_length)   # the config's min_length (0): no EOS ban
        self.length_penalty = float(length_penalty)
        self.mode = mode
        self.eos, self.pad = eos, pad
        self.prefix_fn = prefix_fn
        self.score_dtype = np.float64 if mode == "fp64" else np.float32
        self.beam_scores = np.full(B * nb, -1e9, dtype=self.score_dtype)
        self.beam_scores[::nb] = 0.0
        self.seqs = [[start] for _ in range(B * nb)]
        self.cur_len = 1
        self.hyps = [Hypotheses(nb, self.length_penalty) for _ in range(B)]
        self.done = [False] * B
        self.history = []

    @property
    def finished(self):
        return all(self.done) or self.cur_len >= self.max_length

    def sequences(self):
        return [list(s) for s in self.seqs]

    def processed_logprobs(self, logits):
        """log_softmax (+ the 16-bit rounding of the mode), then MinLength and PrefixConstrained -> float64 [R, V]."""
        lp = round_to(log_softmax(logits), self.mode)
        if self.cur_len < self.min_length:
            lp[:, self.eos] = -np.inf
        if self.prefix_fn is not None:
            mask = np.full(lp.shape, -np.inf)
            for r in range(self.B * self.nb):
                mask[r, self.prefix_fn(r // self.nb, list(self.seqs[r]))] = 0.0
            lp = lp + mask
        return lp

    def step(self, logits=None, logprobs=None):
        """One beam_search iteration.  Returns a dict: tokens, parents (global rows) and scores of the new beams [R], the
        step's margin and the log-prob magnitude at it."""
        B, nb, V = self.B, self.nb, self.V
        R = B * nb
        lp = self.processed_logprobs(logits) if logprobs is None else np.asarray(logprobs, dtype=np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            scores = lp.astype(self.score_dtype) + self.beam_scores[:, None]
        tokens = np.full(R, self.pad, dtype=np.int64)
        parents = np.arange(R, dtype=np.int64)
        new_scores = np.zeros(R, dtype=self.score_dtype)
        margin, lp_scale = np.inf, 0.0

        def note(gap, scale):
            nonlocal margin, lp_scale
            if gap is not None and not np.isnan(gap) and gap < margin:
                margin, lp_scale = gap, scale

        for b in range(B):
            if self.done[b]:
                continue                                # pad, score 0, rows kept in place
            flat = scores[b * nb:(b + 1) * nb].reshape(-1)
            flat_lp = lp[b * nb:(b + 1) * nb].reshape(-1)
            order = rank_order(flat)[: 2 * nb + 1]
            with np.errstate(invalid="ignore"):
                for i in range(min(2 * nb, order.size - 1)):
                    note(float(flat[order[i]]) - float(flat[order[i + 1]]),
                         max(abs(float(flat_lp[order[i]])), abs(float(flat_lp[order[i + 1]]))))
            top = order[: 2 * nb]
            filled = 0
            for rank, f in enumerate(top):
                beam, tok = divmod(int(f), V)
                row = b * nb + beam
                if tok == self.eos:
                    if rank >= nb:
                        continue
                    note(self.hyps[b].add(self.seqs[row], float(flat[f])), abs(float(flat_lp[f])))
                else:
                    k = b * nb + filled
                    tokens[k], parents[k], new_scores[k] = tok, row, flat[f]
                    filled += 1
                if filled == nb:
                    break
            assert filled == nb, "fewer than nb non-EOS candidates"
            fin, gap = self.hyps[b].is_done(float(flat[top[0]]), self.cur_len)
            note(gap, abs(float(flat_lp[top[0]])))
            self.done[b] = self.done[b] or fin
        self.seqs = [self.seqs[int(parents[r])] + [int(tokens[r])] for r in range(R)]
        self.beam_scores = new_scores
        self.cur_len += 1
        rec = dict(tokens=tokens, parents=parents, scores=new_scores.copy(), margin=margin, lp_scale=lp_scale,
                   done=list(self.done))
        self.history.append(rec)
        return rec

    def finalize(self):
        """BeamSearchScorer.finalize -> int64 [B, min(max len + 1, max_length)]: the best hypothesis per batch element (the
        last of a stable sort by score), pad fill only when the lengths differ, EOS at position len when len < max_length."""
        best = []
        for b in range(self.B):
            h = self.hyps[b]
            if not self.done[b]:
                for k in range(self.nb):
                    r = b * self.nb + k
                    h.add(self.seqs[r], float(self.beam_scores[r]))
            best.append(sorted(h.beams, key=lambda x: x[0]).pop()[1])
        lens = [len(s) for s in best]
        width = min(max(lens) + 1, self.max_length)
        out = np.full((self.B, width), self.pad if min(lens) != max(lens) else -1, dtype=np.int64)
        for b, s in enumerate(best):
            out[b, : len(s)] = s
            if len(s) < self.max_length:
                out[b, len(s)] = self.eos
        assert (out >= 0).all()
        return out


def beam_search(step_logits, B, nb, V, max_length, min_length=None, length_penalty=1.0, mode="fp64", eos=1, pad=0,
                start=0, prefix_fn=None):
    """Drive a whole search: step_logits(sequences) -> [B * nb, V] logits of those beams.  Returns (output, BeamSearch)."""
    s = BeamSearch(B, nb, V, max_length, min_length, length_penalty, mode, eos, pad, start, prefix_fn)
    while not s.finished:
        s.step(step_logits(s.sequences()))
    return s.finalize(), s
