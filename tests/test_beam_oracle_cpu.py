"""CPU: the numpy restatement of transformers 4.18 beam search (oracle/beam_oracle.py) on hand-written cases whose answers are
worked out by hand in the comments.  Log-probs are dyadic so every fp32 sum is exact.  EOS = 1, pad = 0, start = 0; the
beam scores are fp32 as in 4.18 (mode "fp32") unless a case says otherwise."""
import numpy as np
import pytest

import beam_oracle as bo

EOS, PAD = 1, 0
LOW = -30.0     # a log-prob that never ranks


def _search(B, nb, V, max_length=8, mode="fp32", **kw):
    return bo.BeamSearch(B, nb, V, max_length, mode=mode, eos=EOS, pad=PAD, start=0, **kw)


def test_rank_order_nan_first_ties_by_index():
    s = np.array([1.0, np.nan, 2.0, 1.0, -np.inf, np.nan, 2.0])
    assert bo.rank_order(s).tolist() == [1, 5, 2, 6, 0, 3, 4]


def test_eos_below_nb_becomes_hypothesis_eos_at_nb_or_later_is_skipped():
    s = _search(1, 2, 4, length_penalty=1.0)
    s.beam_scores[:] = [0.0, -1.0]
    lp = np.array([[LOW, -0.5, -1.0, LOW],       # row 0: EOS -0.5 (rank 0), token 2 -1.0 (rank 1)
                   [LOW, -0.25, LOW, -0.75]])    # row 1: EOS -1.25 (rank 2: skipped), token 3 -1.75 (rank 3)
    rec = s.step(logprobs=lp)
    assert rec["tokens"].tolist() == [2, 3] and rec["parents"].tolist() == [0, 1]
    assert rec["scores"].tolist() == [-1.0, -1.75]
    assert s.hyps[0].beams == [(-0.5, [0])]      # the parent's tokens without the EOS, -0.5 / 1 ** 1


def test_hypothesis_overflow_deletes_the_earliest_of_equal_lowest_scores():
    h = bo.Hypotheses(2, 1.0)
    h.add([0, 5], -2.0)                          # -1
    h.add([0, 6], -2.0)                          # -1, full, worst -1
    h.add([0, 7, 8], -3.0)                       # -1: not above worst, rejected
    assert [t for _, t in h.beams] == [[0, 5], [0, 6]] and h.worst == -1.0
    h.add([0, 9], -1.0)                          # -0.5: the first of the two -1 goes (lower list index)
    assert h.beams == [(-1.0, [0, 6]), (-0.5, [0, 9])] and h.worst == -1.0


def test_finalize_equal_scores_last_inserted_wins():
    s = _search(1, 2, 4, max_length=6)
    s.hyps[0].add([0, 4], -1.0)
    s.hyps[0].add([0, 3], -1.0)                  # same score -0.5, inserted last
    s.done[0] = True
    assert s.finalize().tolist() == [[0, 3, EOS]]


@pytest.mark.parametrize("lp,tie_best,above_best", [(0.0, -4.0, -3.9), (0.5, -8.0, -7.9), (1.0, -16.0, -15.0),
                                                    (2.0, -64.0, -63.0)])
def test_is_done_under_length_penalty(lp, tie_best, above_best):
    # one kept hypothesis of 4 tokens and sum -4: worst = -4 / 4 ** lp = -4, -2, -1, -0.25; at cur_len 16 the bound is
    # best / 16 ** lp, equal to worst for tie_best (done: worst >= bound) and above it for above_best (not done)
    h = bo.Hypotheses(1, lp)
    assert h.is_done(tie_best, 16)[0] is False   # not full yet
    h.add([0, 2, 3, 4], -4.0)
    assert h.worst == -4.0 / 4 ** lp
    assert h.is_done(tie_best, 16)[0] is True
    assert h.is_done(above_best, 16)[0] is False


def test_batch_elements_finish_at_different_steps():
    s = _search(2, 2, 4, max_length=5)
    other = np.array([[-3.0, -3.0, -1.0, -2.0]] * 2)     # batch element 1: EOS never among the first nb
    # step 1 (cur_len 1), b0: EOS -0.5 rank 0 -> hypothesis -0.5; tokens 2 (-1) and 3 (-2) become the beams
    s.step(logprobs=np.vstack([[LOW, -0.5, -1.0, -2.0], [LOW] * 4, other]))
    # step 2 (cur_len 2), b0: row 0 EOS -1.5 (rank 0) -> hypothesis -0.75: full, worst -0.75 >= best -1.5 / 2 -> done;
    # the beams are row 1's token 2 (-2.25) and row 0's token 0 (-31: equal to row 0's token 2, lower index)
    rec = s.step(logprobs=np.vstack([[LOW, -0.5, LOW, LOW], [LOW, LOW, -0.25, LOW], other]))
    assert s.done == [True, False] and rec["tokens"][:2].tolist() == [2, 0] and rec["parents"][:2].tolist() == [1, 0]
    rec = s.step(logprobs=np.vstack([np.zeros((2, 4)), other]))
    assert rec["tokens"][:2].tolist() == [PAD, PAD] and rec["scores"][:2].tolist() == [0.0, 0.0]
    s.step(logprobs=np.vstack([np.zeros((2, 4)), other]))
    assert s.finished and s.cur_len == 5
    out = s.finalize()
    # b0: best hypothesis [0] (-0.5) + EOS, padded because the lengths differ; b1: a running beam of max_length tokens
    assert out.shape == (2, 5)
    assert out[0].tolist() == [0, EOS, PAD, PAD, PAD]
    assert out[1].tolist() == [0, 2, 2, 2, 2]


def test_finalize_lengths_pad_and_eos():
    s = _search(2, 1, 4, max_length=3)
    s.hyps[0].add([0, 2], -1.0)
    s.hyps[1].add([0, 3], -1.0)
    s.done = [True, True]
    assert s.finalize().tolist() == [[0, 2, EOS], [0, 3, EOS]]        # equal lengths: no pad fill, EOS appended
    s = _search(2, 1, 4, max_length=3)
    s.hyps[0].add([0, 2], -1.0)
    s.hyps[1].add([0, 3, 3], -1.0)
    s.done = [True, True]
    assert s.finalize().tolist() == [[0, 2, EOS], [0, 3, 3]]          # len 3 == max_length: no EOS


@pytest.mark.parametrize("min_length,banned", [(3, [True, True, False]), (None, [False, False, False]),
                                               (0, [False, False, False])])
def test_min_length_bans_eos(min_length, banned):
    s = _search(1, 2, 3, max_length=6, min_length=min_length)
    logits = np.array([[0.5, 2.0, 1.0], [0.5, 2.0, 1.0]])
    for step in range(3):
        lp = s.processed_logprobs(logits)
        assert bool(np.isneginf(lp[:, EOS]).all()) == banned[step], step
        s.step(logits)


def test_prefix_mask_added_after_log_softmax():
    s = _search(1, 2, 4, mode="fp64", prefix_fn=lambda b, sent: [2, 3])
    logits = np.array([[1.0, 0.0, 2.0, -1.0]] * 2)
    lp = s.processed_logprobs(logits)
    ref = bo.log_softmax(logits)
    assert np.isneginf(lp[:, :2]).all()
    assert np.array_equal(lp[:, 2:], ref[:, 2:])       # not renormalised over the allowed tokens
    assert np.all(lp[:, 2] < 0)


def test_vocab_smaller_than_two_beams_picks_from_the_minus_1e9_beam():
    s = _search(1, 2, 2, max_length=4)
    # all 4 candidates are the top 4: row 0 EOS (hypothesis), row 0 token 0, row 1 EOS (rank 2, skipped), row 1 token 0
    rec = s.step(logprobs=np.array([[-1.5, -0.5], [-1.5, -0.5]]))
    assert rec["parents"].tolist() == [0, 1] and rec["tokens"].tolist() == [0, 0]
    assert rec["scores"][1] == np.float32(-1e9 - 1.5) and len(s.hyps[0]) == 1


def test_stop_at_max_length_without_eos():
    out, s = bo.beam_search(lambda seqs: np.log(np.array([[4.0, 1e-4, 2.0, 1.0]] * 2)), 1, 2, 4, max_length=3,
                            eos=EOS, pad=PAD)
    assert s.cur_len == 3 and not s.done[0]
    assert all(len(h) == 3 for _, h in s.hyps[0].beams)   # finalize kept the two running beams, no EOS hypothesis
    assert out.tolist() == [[0, 0, 0]]                   # the best running beam; len == max_length: no EOS


def test_rounding_modes():
    x = np.array([1.0 + 2.0 ** -9, 1.0 + 3 * 2.0 ** -11, -np.inf, np.nan])
    assert bo.round_to(x, "bf16")[:2].tolist() == [1.0, 1.0]
    assert bo.round_to(x, "fp16")[:2].tolist() == [1.0 + 2.0 ** -9, 1.0 + 2.0 ** -9]
    assert bo.round_to(np.array([1.0 + 2.0 ** -30]), "fp32").tolist() == [1.0]
    assert np.isneginf(bo.round_to(x, "bf16")[2]) and np.isnan(bo.round_to(x, "fp16")[3])
