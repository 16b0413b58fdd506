"""The key segments of FiD's split-KV decoder cross-attention (`fid._cross_split`): every key range a split existed for keeps
that split unpadded, and every other range gets a padded plan the split-KV kernel and its dropout masks take."""
import pytest

from atlas_b200._lib import AtlasB200Error
from atlas_b200.fid import _cross_split

N_CONTEXT = list(range(1, 101))
LENGTHS = list(range(64, 513, 4)) + [100, 150, 200, 250, 300, 500]


def _divisor_split(Lk, dropout):
    """The divisor rule alone, with its two refusals (what `_cross_split` returned before padded plans existed)."""
    split = None
    if dropout:
        split = next((s for s in range(min(512, Lk) // 32 * 32, 63, -32) if Lk % s == 0), None)
    split = split or next((s for s in range(min(384, Lk), 63, -1) if Lk % s == 0), None) or \
        next(s for s in range(min(512, Lk), 0, -1) if Lk % s == 0)
    if split < 64 and Lk > 512:
        raise AtlasB200Error("no divisor in [64, 512]")
    if dropout and split % 32 != 0 and split != Lk:
        raise AtlasB200Error("dropout needs a multiple of 32")
    return split


def _check_padded(Lk, split, Lk_pad):
    assert split % 64 == 0 and 64 <= split <= 512, (Lk, split)
    assert Lk_pad % split == 0 and Lk <= Lk_pad, (Lk, split, Lk_pad)
    assert Lk_pad - Lk < (64 if Lk <= 512 else 384), (Lk, Lk_pad)
    assert Lk_pad == split or split <= 384, (Lk, split, Lk_pad)
    # never more dead keys than 384-key segments would leave
    assert Lk_pad <= -(-Lk // 384) * 384 or Lk <= 512


@pytest.mark.parametrize("dropout", [False, True])
def test_existing_splits_kept_and_the_rest_padded(dropout):
    """Every n_context x text_maxlength of the grid, and every key range up to 4096."""
    kept = padded = 0
    for Lk in sorted({n * L for n in N_CONTEXT for L in LENGTHS} | set(range(1, 4097))):
        try:
            want = _divisor_split(Lk, dropout)
        except AtlasB200Error:
            want = None
        split, Lk_pad = _cross_split(Lk, dropout=dropout)
        if want is not None:
            assert (split, Lk_pad) == (want, Lk), (Lk, dropout)
            kept += 1
        else:
            _check_padded(Lk, split, Lk_pad)
            padded += 1
    assert kept > 0 and padded > 0


def test_issue_shapes():
    # the reference's training defaults: --text_maxlength 200 --dropout 0.1
    for n in (2, 3, 5, 10, 25, 30, 50):
        with pytest.raises(AtlasB200Error):
            _divisor_split(n * 200, True)
        split, Lk_pad = _cross_split(n * 200, dropout=True)
        _check_padded(n * 200, split, Lk_pad)
    assert _cross_split(6000, dropout=True) == (384, 6144)
    assert _cross_split(6000) == (375, 6000)                # evaluation keeps its divisor
    assert _cross_split(600, dropout=True) == (320, 640)
    assert _cross_split(400, dropout=True) == (448, 448)    # one segment up to 512 keys
    # no divisor in [64, 512] at all (1031 is prime), with and without dropout
    with pytest.raises(AtlasB200Error):
        _divisor_split(1031, False)
    assert _cross_split(1031) == _cross_split(1031, dropout=True) == (384, 1152)
    # the bench configuration (40 x 384) keeps its regular split
    assert _cross_split(40 * 384) == (384, 40 * 384)


def test_forced_padding():
    for Lk in (64, 100, 512, 600, 6000, 6400, 40 * 384):
        split, Lk_pad = _cross_split(Lk, force_pad=True)
        _check_padded(Lk, split, Lk_pad)
    assert _cross_split(6000, force_pad=True) == (384, 6144)
