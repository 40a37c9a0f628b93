"""CPU: the argument checks of the row-selected fp32 output of the wgmma GEMM (gr_linear_tc_planes_rows, c_rows), which
come before any CUDA call (the pointers are placeholders), and the refusals of its Python wrapper and of the
ReaRev layer's last-layer flag."""
import ctypes

import pytest

from gnn_rag_b200 import _lib, modules

PTR = ctypes.c_void_p(0x1000)
INVALID, WORKSPACE = -1, -3


def _rows_call(C, c_rows, C_hi=None, ws_bytes=16, fn="gr_linear_tc_planes_rows"):
    lib = _lib.load()
    args = [PTR, PTR, 2048, PTR, 2048, None, C, 256, C_hi, C_hi, 256 if C_hi else 0, None, None, 256, 200, 1040, 200,
            208, 0, PTR, ws_bytes]
    if fn == "gr_linear_tc_planes_rows":
        args.append(c_rows)
    rc = getattr(lib, fn)(*args, None)
    return rc, lib.gr_last_error().decode()


def test_rows_without_fp32_output_are_refused():
    rc, err = _rows_call(None, PTR, C_hi=PTR)
    assert rc == INVALID and "gr_linear_tc_planes_rows" in err and "c_rows selects rows of C" in err, (rc, err)


def test_null_rows_is_the_plain_entry_point():
    # with c_rows NULL (or a C to select from) the checks that remain are the ones of gr_linear_tc_planes: here the
    # 16-byte workspace, refused under the entry point's own name
    for c_rows in (None, PTR):
        rc, err = _rows_call(PTR, c_rows)
        assert rc == WORKSPACE and err.startswith("gr_linear_tc_planes_rows:"), (c_rows, rc, err)
    rc, err = _rows_call(PTR, None, fn="gr_linear_tc_planes")
    assert rc == WORKSPACE and err.startswith("gr_linear_tc_planes:"), (rc, err)
    rc, err = _rows_call(None, None)
    assert rc == INVALID and "no output requested" in err, (rc, err)


def test_rows_prototype_is_the_plain_one_with_c_rows_before_the_stream():
    sig = _lib.SIGNATURES
    plain, rows = sig["gr_linear_tc_planes"], sig["gr_linear_tc_planes_rows"]
    assert rows[0] == plain[0]
    assert rows[1] == plain[1][:-1] + [ctypes.c_void_p] + plain[1][-1:]


def test_a_last_layer_keeps_the_full_fp32_h():
    layer = modules.ReasonGNNLayer.__new__(modules.ReasonGNNLayer)
    for kw in (dict(need_h=False), dict(need_h=True, h_rows=object())):
        with pytest.raises(AssertionError, match="last layer keeps the full fp32 h"):
            modules.ReasonGNNLayer.forward(layer, None, None, next_layer=False, **kw)
