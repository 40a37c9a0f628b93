"""Host checks of the bf16 node-tensor entry points (include/gnnrag_b200.h, *_ex with GR_IO_BF16): unknown io bits,
null pointers and widths outside the kernels are refused with a status code and a message before touching the device;
the workspace-size helpers serve both modes; the ops wrappers accept exactly fp32 and bf16 node-sized tensors."""
import ctypes

import pytest
import torch

from gnn_rag_b200 import _lib, ops

GR_ERR_INVALID_ARG = -1
GR_IO_BF16 = 1
P = ctypes.c_void_p(16)       # never dereferenced: every call below is refused before any launch
NUL = None


@pytest.fixture(scope="module")
def L():
    return _lib.load()


def _err(L):
    return (L.gr_last_error() or b"").decode()


def _agg(L, io, D=64, I=2, ptr=P):
    return L.gr_aggregate_ex(ptr, P, P, NUL, P, P, P, P, I * D, 0, D, NUL, 2, 10, D, I, 100, io, NUL)


def _agg_bwd(L, io, D=64, I=2, ptr=P):
    return L.gr_aggregate_backward_ex(ptr, P, P, NUL, P, P, P, P, I * D, 0, D, P, P, P, 2, 10, D, I, 100, io, NUL)


def _agg_bwd_det(L, io, D=64, I=2, ptr=P):
    return L.gr_aggregate_backward_det_ex(ptr, P, P, P, NUL, P, P, P, P, I * D, 0, D, P, P, P, 2, 10, D, I, 100,
                                          P, P, P, P, P, 5, P, 1 << 30, io, NUL)


def _type(L, io, D=64, ptr=P):
    return L.gr_type_layer_ex(ptr, P, NUL, P, P, NUL, P, P, D, NUL, NUL, 0, 2, 10, D, 100, io, NUL)


def _type_bwd(L, io, D=64, ptr=P):
    return L.gr_type_layer_backward_ex(ptr, P, NUL, P, P, NUL, P, D, P, D, P, D, 2, 10, D, 100, io, NUL)


def _type_bwd_det(L, io, D=64, ptr=P):
    return L.gr_type_layer_backward_det_ex(P, NUL, ptr, P, P, P, NUL, P, P, P, P, D, P, D, P, D, 5, D, 100, P, 1 << 30,
                                           io, NUL)


def _graft_fwd(L, io, D=64, ptr=P):
    return L.gr_graft_aggregate_train_ex(ptr, P, P, P, P, P, P, D, P, D, NUL, 0.0, P, D, 2, 10, D, io, NUL)


def _graft_bwd(L, io, D=64, ptr=P):
    return L.gr_graft_aggregate_backward_ex(ptr, P, P, P, P, P, P, D, P, D, NUL, 0.0, P, D, P, P, D, P, D, 2, 10, D,
                                            io, NUL)


def _graft_bwd_det(L, io, D=64, ptr=P):
    return L.gr_graft_aggregate_backward_det_ex(ptr, P, P, P, P, P, P, D, P, D, NUL, 0.0, P, D, P, P, D, P, D, 2, 10,
                                                D, P, P, P, P, P, 5, 100, P, 1 << 30, io, NUL)


CALLS = [_agg, _agg_bwd, _agg_bwd_det, _type, _type_bwd, _type_bwd_det, _graft_fwd, _graft_bwd, _graft_bwd_det]


@pytest.mark.parametrize("call", CALLS, ids=lambda c: c.__name__)
def test_unknown_io_bits_are_refused(L, call):
    for io in (2, 0x80000000, GR_IO_BF16 | 4):
        assert call(L, io) == GR_ERR_INVALID_ARG
        assert "io flags" in _err(L)


@pytest.mark.parametrize("call", CALLS, ids=lambda c: c.__name__)
@pytest.mark.parametrize("io", [0, GR_IO_BF16])
def test_null_pointers_are_refused_in_both_modes(L, call, io):
    assert call(L, io, ptr=NUL) == GR_ERR_INVALID_ARG
    assert "null" in _err(L)


@pytest.mark.parametrize("io", [0, GR_IO_BF16])
def test_widths_outside_the_kernels_are_refused_in_both_modes(L, io):
    for D, I in ((0, 1), (257, 1), (64, 0), (64, 5)):
        for call in (_agg_bwd, _agg_bwd_det):
            assert call(L, io, D=D, I=I) == GR_ERR_INVALID_ARG and "D <= 256" in _err(L)
    assert _agg(L, io, D=0) == GR_ERR_INVALID_ARG
    for D in (0, 513):
        for call in (_type_bwd, _type_bwd_det, _graft_fwd, _graft_bwd, _graft_bwd_det):
            assert call(L, io, D=D) == GR_ERR_INVALID_ARG and "D <= 512" in _err(L), call.__name__
    assert _type(L, io, D=0) == GR_ERR_INVALID_ARG


def test_workspace_helpers_serve_both_modes():
    """The workspace-size helpers take no io word: the workspace holds fp32 partial sums in both modes, so one size
    serves both, and the _ex entry points take the same workspace arguments as their fp32 counterparts."""
    for name in ("gr_aggregate_backward_det", "gr_type_layer_backward_det", "gr_graft_aggregate_backward_det"):
        assert ctypes.c_uint32 not in _lib.SIGNATURES[name + "_workspace_bytes"][1]
        base, ex = _lib.SIGNATURES[name][1], _lib.SIGNATURES[name + "_ex"][1]
        assert ex[:-1] == base[:-1] + [ctypes.c_uint32] and ex[-1] == base[-1]


@pytest.fixture
def host_node_io(monkeypatch):
    """ops._node_io with the CUDA-residency check lifted, so its dtype rules can be checked on CPU tensors."""
    monkeypatch.setattr(ops, "_cuda", lambda t, dtype=None, name="tensor": t)
    return ops._node_io


def test_node_tensor_dtypes(host_node_io):
    f32, bf = torch.zeros(2, 3), torch.zeros(2, 3, dtype=torch.bfloat16)
    assert host_node_io(out=f32) == 0
    assert host_node_io(out=bf) == ops.IO_BF16 == GR_IO_BF16
    assert host_node_io(head_tab=bf, grad_sum=bf, grad_head=None) == GR_IO_BF16
    for bad in (torch.float16, torch.float64, torch.int32):
        with pytest.raises(RuntimeError, match="must be torch.float32 or torch.bfloat16"):
            host_node_io(grad_out=torch.zeros(2, 3, dtype=bad))
    with pytest.raises(RuntimeError, match="share one dtype"):
        host_node_io(grad_out=bf, out=f32)


def test_node_tensors_must_be_on_cuda():
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops._node_io(out=torch.zeros(2, 3, dtype=torch.bfloat16))
