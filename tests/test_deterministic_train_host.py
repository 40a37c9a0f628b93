"""Host checks of the deterministic backward entry points (include/gnnrag_b200.h, *_det): they refuse null pointers,
out-of-range widths and short workspaces with a status code and a message before touching the device, and their
workspace-size helpers grow with the shapes they describe."""
import ctypes

import pytest

from gnn_rag_b200 import _lib

GR_ERR_INVALID_ARG = -1
GR_ERR_WORKSPACE = -3


@pytest.fixture(scope="module")
def L():
    return _lib.load()


def _err(L):
    return (L.gr_last_error() or b"").decode()


P = ctypes.c_void_p(16)       # never dereferenced: every call below is refused before any launch
NUL = None


def _agg(L, D=64, I=2, ptr=P, ws_bytes=1 << 30, F=100):
    return L.gr_aggregate_backward_det(ptr, P, P, P, NUL, P, P, P, P, I * D, 0, D, P, P, P, 2, 10, D, I, F,
                                       P, P, P, P, P, 5, P, ws_bytes, NUL)


def _type(L, D=64, ptr=P, ws_bytes=1 << 30, F=100):
    return L.gr_type_layer_backward_det(P, NUL, ptr, P, P, P, NUL, P, P, P, P, D, P, D, P, D, 5, D, F, P, ws_bytes,
                                        NUL)


def _graft(L, D=64, ptr=P, ws_bytes=1 << 30, p=0.0):
    return L.gr_graft_aggregate_backward_det(P, P, P, P, P, P, P, D, P, D, NUL, p, P, D, P, P, D, P, D, 2, 10, D,
                                             ptr, P, P, P, P, 5, 100, P, ws_bytes, NUL)


def _attn(L, D=64, Q=4, ptr=P, ws_bytes=1 << 30):
    return L.gr_graft_attention_backward_det(P, P, Q, P, D, 5, P, 2, 30, D, P, P, P, D, ptr, P, P, ws_bytes, NUL)


@pytest.mark.parametrize("call,name", [(_agg, "gr_aggregate_backward_det"), (_type, "gr_type_layer_backward_det"),
                                       (_graft, "gr_graft_aggregate_backward_det"),
                                       (_attn, "gr_graft_attention_backward_det")])
def test_null_pointers_are_refused(L, call, name):
    assert call(L, ptr=NUL) == GR_ERR_INVALID_ARG
    assert name in _err(L) and "null" in _err(L)


def test_widths_outside_the_kernels_are_refused(L):
    for D, I in ((0, 1), (257, 1), (64, 0), (64, 5)):
        assert _agg(L, D=D, I=I) == GR_ERR_INVALID_ARG
        assert "D <= 256" in _err(L)
    for D in (0, 513):
        assert _type(L, D=D) == GR_ERR_INVALID_ARG and "D <= 512" in _err(L)
        assert _graft(L, D=D) == GR_ERR_INVALID_ARG and "D <= 512" in _err(L)
        assert _attn(L, D=D) == GR_ERR_INVALID_ARG and "D <= 512" in _err(L)
    assert _attn(L, Q=0) == GR_ERR_INVALID_ARG and "Q > 0" in _err(L)
    assert _graft(L, p=1.0) == GR_ERR_INVALID_ARG and "dropout" in _err(L)


def test_short_workspaces_are_refused(L):
    assert _agg(L, ws_bytes=16) == GR_ERR_WORKSPACE and "workspace too small" in _err(L)
    assert _type(L, ws_bytes=16) == GR_ERR_WORKSPACE and "workspace too small" in _err(L)
    assert _graft(L, ws_bytes=16) == GR_ERR_WORKSPACE and "workspace too small" in _err(L)
    assert _attn(L, ws_bytes=16) == GR_ERR_WORKSPACE and "workspace too small" in _err(L)


def test_row_of_refuses_bad_arguments(L):
    assert L.gr_csr_row_of(NUL, 10, P, NUL) == GR_ERR_INVALID_ARG and "null" in _err(L)
    assert L.gr_csr_row_of(P, 0, P, NUL) == GR_ERR_INVALID_ARG


def test_workspace_helpers():
    L = _lib.load()
    # aggregation: per-fact scalars q plus the larger of the dx (windows of 32 rows x I*D) and dP (windows of 64
    # facts x D) partials -- never a per-fact x D buffer
    a = L.gr_aggregate_backward_det_workspace_bytes(64, 2000, 200, 2, 384000)
    assert a >= 384000 * 4 + 2 * (64 * 2000 // 32) * 2 * 200 * 4
    assert a < 384000 * 200 * 4 // 8
    assert L.gr_aggregate_backward_det_workspace_bytes(1, 1, 1, 1, 0) > 0
    assert L.gr_aggregate_backward_det_workspace_bytes(0, 1, 1, 1, 0) == 0
    assert L.gr_aggregate_backward_det_workspace_bytes(200, 10, 64, 2, 200) > \
        L.gr_aggregate_backward_det_workspace_bytes(200, 10, 64, 1, 200)
    t = L.gr_type_layer_backward_det_workspace_bytes(64000, 100)
    assert 2 * 1000 * 100 * 4 <= t < 2 * 1000 * 100 * 4 + 512
    assert L.gr_type_layer_backward_det_workspace_bytes(-1, 100) == 0
    assert L.gr_graft_aggregate_backward_det_workspace_bytes(6400, 512) == 2 * 100 * 512 * 4
    w = L.gr_graft_attention_backward_det_workspace_bytes(4, 300, 7, 64)
    assert w >= 4 * 300 * 7 * 4 + 2 * ((4 * 300 + 63) // 64) * 64 * 4
    assert L.gr_graft_attention_backward_det_workspace_bytes(4, 300, 0, 64) == 0
