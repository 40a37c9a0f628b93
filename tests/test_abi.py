"""CPU: the C-ABI shared library loads and exports every symbol include/gnnrag_b200.h declares; argument
validation fails with status codes (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

from gnn_rag_b200 import _build, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "gnnrag_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = set(re.findall(r"\b(gr_[a-z0-9_]+)\s*\(", text))
    names.discard("gr_pad4")          # static inline helper
    return sorted(names)


def test_library_builds_and_loads():
    _build.build()
    lib = _lib.load()
    assert lib.gr_abi_version() == 1


def test_every_declared_symbol_is_exported_and_bound():
    lib = ctypes.CDLL(_build.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 15
    for name in syms:
        assert hasattr(lib, name), "missing export: " + name
        assert name in _lib.SIGNATURES, "no ctypes signature for " + name
    assert sorted(_lib.SIGNATURES) == syms


def declared_arities():
    """name -> number of parameters of every prototype in the header."""
    text = open(os.path.join(ROOT, "include", "gnnrag_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(gr_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", text, flags=re.S):
        params = m.group(2).strip()
        out[m.group(1)] = 0 if params in ("", "void") else params.count(",") + 1
    return out


def test_ctypes_signatures_have_the_header_arity():
    """A drifted binding (argument added on one side only) would scramble the stack silently."""
    ar = declared_arities()
    for name, (_res, argtypes) in _lib.SIGNATURES.items():
        assert name in ar, name
        assert len(argtypes) == ar[name], "%s: header has %d parameters, ctypes binding %d" % (
            name, ar[name], len(argtypes))


def test_new_entry_points_validate_arguments():
    lib = _lib.load()
    assert lib.gr_aggregate_dual_abs_supported(2000, 200, 208, 6107) == 1
    assert lib.gr_aggregate_dual_abs_supported(2000, 64, 64, 100) == 0        # other shapes: generic kernel
    assert lib.gr_aggregate_dual_abs_supported(32, 200, 208, 100) == 0        # N < one tile
    assert lib.gr_lstm_max_hidden() == 256
    assert lib.gr_lstm_forward(None, None, None, None, 1, 1, 8, None) == -1
    assert lib.gr_pad_table256(None, 0, 1, 8, None, None) == -1
    assert lib.gr_kl_loss_pred(None, None, None, None, None, 1, 1, None) == -1
    assert lib.gr_frontier_rows(None, None, None, None, None, 1, None, None, None) == -1
    # fused layer kernel: size helpers are pure host arithmetic, null pointers are refused before any CUDA call
    assert lib.gr_fused_layer_workspace_bytes(200, 208, 2, 200) >= 2 * 200 * 7 * 5 * 32 * 2
    assert lib.gr_fused_ell_bytes(64, 2000, 512000) > 2 * (2 * 512000 + 4 * 128000) * 8
    assert lib.gr_fused_ell_bytes(0, 2000, 10) == 0
    assert lib.gr_fused_ell_build(None, None, None, None, None, None, None, None, 1, 128, 0, None, 0, None) == -1
    assert lib.gr_fused_layer(None, None, None, None, None, None, None, None, None, None, None, None, None, None, 208,
                              208, None, 1000, None, None, 0, None, None, 0, None, None, 1, 128, 200, 2, 200, 0, 0,
                              None, 0, None, 0, None) == -1
    assert lib.gr_aggregate_backward(None, None, None, None, None, None, None, None, 0, 0, 0, None, None, None, 1, 1, 8,
                                     1, 0, None) == -1


def test_argument_validation_returns_status_codes():
    lib = _lib.load()
    rc = lib.gr_linear(None, 4, None, 4, None, None, 0, 0, None, 4, 4, 4, 4, 0, None)
    assert rc == -1 and b"null pointer" in lib.gr_last_error()
    rc = lib.gr_csr_build(None, None, None, 3, 0, 10, 5, None, None, None, None, None, None, None, None,
                          None, None, None, 0, None)
    assert rc == -1 and b"idx_bytes" in lib.gr_last_error()
    rc = lib.gr_set_option(b"no_such_option", 1)
    assert rc == -1
    assert lib.gr_set_option(b"agg_tma", 0) == 0
    assert lib.gr_set_option(b"linear_tc", 0) == -1 and b"unknown option" in lib.gr_last_error()   # never read: removed
    assert lib.gr_csr_build_workspace_bytes(1000, 100) > 0
    assert lib.gr_rank_workspace_bytes(4, 100) == 4 * 100 * 8
    with pytest.raises(_lib.GrError):
        _lib.check(-1)


def test_models_refuse_cpu():
    import gnn_rag_b200 as G
    from gnn_rag_b200 import synthetic as S
    args = S.model_args("ReaRev", entity_dim=16, word_dim=8)
    m = G.ReaRev(args, 100, 10, 20)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(S.make_batch(0, 2, 10, 20, 100, 10, 20))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(S.make_batch(0, 2, 10, 20, 100, 10, 20), training=True)
