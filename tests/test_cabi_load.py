"""CPU: the C-ABI shared library loads without a GPU driver and exports every symbol that
include/atlas_b200.h declares.  No compute calls."""
import ctypes
import os
import re

from conftest import ROOT


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "atlas_b200.h")).read()
    return sorted(set(re.findall(r"\b(atlas_b200_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_header_symbols():
    from atlas_b200 import _lib

    assert os.path.exists(_lib.LIB_PATH), "build the library first: python -c 'import __graft_entry__ as g; g.build()'"
    L = ctypes.CDLL(_lib.LIB_PATH)
    declared = _declared_symbols()
    assert len(declared) >= 8
    for sym in declared:
        assert hasattr(L, sym), f"{sym} declared in include/atlas_b200.h but not exported"
    assert set(_lib.EXPORTED_SYMBOLS) == set(declared)


def test_workspace_size_is_pure_host():
    from atlas_b200 import _lib

    L = _lib.lib()
    small = L.atlas_b200_mips_workspace_bytes(10000, 64, 40)
    big = L.atlas_b200_mips_workspace_bytes(4 << 20, 256, 40)
    assert 0 < small < big < (1 << 31)
    assert L.atlas_b200_version().startswith(b"atlas_b200")


def test_no_cpu_fallback():
    import pytest
    import torch

    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    bank = torch.zeros(64, 768, dtype=torch.float16)
    with pytest.raises(AtlasB200Error):
        ops.mips_topk(bank, torch.zeros(1, 768), 4)


def test_argtypes_match_header_prototypes():
    """Every prototype in include/atlas_b200.h has as many parameters as the ctypes argtypes of `_lib.lib()`: with a wrong
    count ctypes passes the arguments shifted, which shows only on a GPU run, as garbage pointers."""
    from atlas_b200 import _lib

    L = _lib.lib()
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "atlas_b200.h")).read(), flags=re.S)
    protos = re.findall(r"(atlas_b200_\w+)\s*\(([^)]*)\)\s*;", text)
    assert {name for name, _ in protos} == set(_lib.EXPORTED_SYMBOLS)
    for name, params in protos:
        n = 0 if params.strip() in ("", "void") else len(params.split(","))
        argtypes = getattr(L, name).argtypes or []
        assert len(argtypes) == n, f"{name}: {n} parameters in the header, {len(argtypes)} argtypes"


def test_attention_bwd_rejects_missing_lse():
    """atlas_b200_attention_bwd_train without the forward's log-sum-exp (lse = NULL) is rejected during argument
    validation, before any CUDA call: the backward reads the log-sum-exp the forward wrote and has no path that
    recomputes it."""
    from atlas_b200 import _lib

    L = _lib.lib()
    B, H, Lq, Lk, ld = 2, 4, 64, 64, 3 * 4 * 64
    buf = (ctypes.c_float * (B * H * Lq))()
    p = ctypes.cast(buf, ctypes.c_void_p)     # non-null stand-in for q, k, v, out, dout, dq, dk, dv and dsum
    rc = L.atlas_b200_attention_bwd_train(p, ld, 0, p, ld, 64 * H, p, ld, 128 * H, p, 64 * H, p, 64 * H, p, ld, 0, p, ld,
                                          64 * H, p, ld, 128 * H, None, None, None, None, p, None, B, H, Lq, Lk,
                                          0.125, 0.0, 0.0, 0, 0, None, 1, None)
    assert rc == 1, rc                                             # ATLAS_B200_EINVAL
    assert b"log-sum-exp" in L.atlas_b200_last_error() and b"lse" in L.atlas_b200_last_error()
