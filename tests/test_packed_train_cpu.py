"""CPU: argument checks of the packed-encoder entry points (include/atlas_b200.h "Padding-compacted FiD encoder") and the rule
that selects the padding-compacted encoder.  Rejected calls return ATLAS_B200_EINVAL during argument validation, before any
CUDA call."""
import ctypes

import pytest
import torch

EINVAL = 1


def _buf():
    buf = (ctypes.c_float * 4096)()
    return buf, ctypes.cast(buf, ctypes.c_void_p)      # non-null stand-in for every device pointer


@pytest.mark.parametrize("L", [640, 100])
def test_attention_packed_rejects_segment_length(L):
    from atlas_b200 import _lib

    lib = _lib.lib()
    _keep, p = _buf()
    H = 4
    rc = lib.atlas_b200_attention_packed(p, 3 * H * 64, 0, H * 64, 2 * H * 64, p, H * 64, p, None, p, p, 2, H, L, 1.0, p, 0.1,
                                         1, 0, 1, None)
    assert rc == EINVAL, rc
    assert b"attention_packed" in lib.atlas_b200_last_error()
    rc = lib.atlas_b200_attention_packed_bwd(p, 3 * H * 64, p, H * 64, p, H * 64, p, 3 * H * 64, p, None, None, p, p, p, p, 2,
                                             H, L, 1.0, 0.1, 1, 0, 1, None)
    assert rc == EINVAL, rc
    assert b"attention_packed_bwd" in lib.atlas_b200_last_error()


def test_attention_packed_bwd_requires_lse():
    from atlas_b200 import _lib

    lib = _lib.lib()
    _keep, p = _buf()
    H, L = 4, 512
    rc = lib.atlas_b200_attention_packed_bwd(p, 3 * H * 64, p, H * 64, p, H * 64, p, 3 * H * 64, p, None, None, None, p, p, p,
                                             2, H, L, 1.0, 0.0, 0, 0, 1, None)
    assert rc == EINVAL, rc
    assert b"lse" in lib.atlas_b200_last_error()


def test_dropout_row_tiles_need_whole_tiles():
    from atlas_b200 import _lib

    lib = _lib.lib()
    _keep, p = _buf()
    rc = lib.atlas_b200_dropout(p, 64, None, 0, p, 64, 100, 64, 0.1, 1, 0, p, 1, None)
    assert rc == EINVAL, rc
    assert b"row_tiles" in lib.atlas_b200_last_error()


def test_encoder_packs_selection():
    from atlas_b200 import ops

    live = torch.ones(2, 9, dtype=torch.uint8)
    for L in (64, 384, 448, 512, 576):
        assert ops.encoder_packs(live, L), L
    for L in (200, 640):
        assert not ops.encoder_packs(live, L), L
    assert not ops.encoder_packs(None, 512)
    assert ops.encoder_attention(640) is ops.attention_long
