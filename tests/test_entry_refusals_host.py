"""CPU: every training entry point refuses bad arguments with a fixed (status, gr_last_error()) pair, whichever of
its fp32, `_ex`, `_det` and `_det_ex` forms is called.  Every call below is refused before any CUDA call, so the
pointers are placeholders that are never dereferenced."""
import os
import re

import pytest

from gnn_rag_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTR = 0x1000          # a non-null device pointer: never dereferenced, every call is refused first
INVALID, WORKSPACE = -1, -3


def _param_names():
    text = open(os.path.join(ROOT, "include", "gnnrag_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return {m.group(1): [p.split()[-1].lstrip("*") for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(gr_\w+)\s*\(([^;{}()]*)\)\s*;", text)}


PARAMS = _param_names()


def call(name, args):
    """Call entry point `name` with arguments by parameter name; a parameter not in `args` is a pointer."""
    lib = _lib.load()
    rc = getattr(lib, name)(*[args.get(p, PTR) for p in PARAMS[name]])
    return rc, lib.gr_last_error().decode()


# ---- per op: good arguments, the entry points, and the refusals ------------------------------------------------------
# An entry is (entry point, the forms it takes ("fp32", "ex", "det", ...), the name its argument checks report, the
# name its workspace check reports).  A case is (forms it applies to, argument overrides, status, message after "<name>: ").

AGG = dict(w=None, possible=None, out_row_stride=16, out_col0=0, seg_stride=8, B=2, N=3, D=8, I=2, F=4, io=0,
           stream=None)
AGG_ENTRIES = [("gr_aggregate", {"fp32"}, "gr_aggregate_ex", None),
               ("gr_aggregate_ex", {"ex"}, "gr_aggregate_ex", None)]
AGG_CASES = [
    ({"fp32", "ex"}, dict(rowptr=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(out=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(src=None), INVALID, "null edge arrays"),
    ({"fp32", "ex"}, dict(B=0), INVALID, "B, N, D, I must be positive"),
    ({"fp32", "ex"}, dict(N=0), INVALID, "B, N, D, I must be positive"),
    ({"fp32", "ex"}, dict(D=0), INVALID, "B, N, D, I must be positive"),
    ({"fp32", "ex"}, dict(I=0), INVALID, "B, N, D, I must be positive"),
    ({"ex"}, dict(io=2), INVALID, "unknown io flags"),
]

AGG_BWD = dict(w=None, grad_row_stride=16, grad_col0=0, seg_stride=8, B=2, N=3, D=8, I=2, F=4, R1=3, io=0,
               stream=None)
AGG_BWD_ENTRIES = [
    ("gr_aggregate_backward", {"fp32"}, "gr_aggregate_backward_ex", None),
    ("gr_aggregate_backward_ex", {"ex"}, "gr_aggregate_backward_ex", None),
    ("gr_aggregate_backward_det", {"fp32", "det"}, "gr_aggregate_backward_det_ex", "gr_aggregate_backward_det"),
    ("gr_aggregate_backward_det_ex", {"ex", "det"}, "gr_aggregate_backward_det_ex", "gr_aggregate_backward_det"),
]
_SIZES = "need 0 < D <= 256 and 0 < I <= 4"
_STRIDE = "grad_out row stride / segment stride smaller than the rows it must hold"
AGG_BWD_CASES = [
    ({"fp32", "ex"}, dict(rowptr=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(grad_prior=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(rel=None), INVALID, "null edge arrays"),
    ({"fp32", "ex"}, dict(B=0), INVALID, _SIZES),
    ({"fp32", "ex"}, dict(N=0), INVALID, _SIZES),
    ({"fp32", "ex"}, dict(D=0), INVALID, _SIZES),
    ({"fp32", "ex"}, dict(D=257, seg_stride=257, grad_row_stride=514), INVALID, _SIZES),
    ({"fp32", "ex"}, dict(I=0), INVALID, _SIZES),
    ({"fp32", "ex"}, dict(I=5, grad_row_stride=40), INVALID, _SIZES),
    ({"fp32", "ex"}, dict(seg_stride=7, grad_row_stride=15), INVALID, _STRIDE),
    ({"fp32", "ex"}, dict(grad_row_stride=15), INVALID, _STRIDE),
    ({"fp32", "ex"}, dict(grad_col0=1), INVALID, _STRIDE),
    ({"ex"}, dict(io=2), INVALID, "unknown io flags"),
    ({"det"}, dict(rix_ptr=None), INVALID, "null pointer"),
    ({"det"}, dict(row_of=None), INVALID, "null edge arrays"),
    ({"det"}, dict(F=-1), INVALID, _SIZES),
    ({"det"}, dict(R1=0), INVALID, _SIZES),
    ({"det"}, dict(workspace_bytes="short"), WORKSPACE, None),
    ({"det"}, dict(workspace=None), WORKSPACE, None),
]

TYPE = dict(w_t=None, w_h=None, out_row_stride=8, out_hi=None, out_lo=None, ld_planes=0, B=2, N=3, D=8, F=4, io=0,
            stream=None)
TYPE_ENTRIES = [("gr_type_layer", {"fp32"}, "gr_type_layer_ex", None),
                ("gr_type_layer_ex", {"ex"}, "gr_type_layer_ex", None)]
TYPE_CASES = [
    ({"fp32", "ex"}, dict(rowptr_h=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(out=None), INVALID, "no output requested"),
    ({"fp32", "ex"}, dict(rel_t=None), INVALID, "null edge arrays"),
    ({"fp32", "ex"}, dict(B=0), INVALID, "B, N, D must be positive"),
    ({"fp32", "ex"}, dict(N=0), INVALID, "B, N, D must be positive"),
    ({"fp32", "ex"}, dict(D=0), INVALID, "B, N, D must be positive"),
    ({"ex"}, dict(io=2), INVALID, "unknown io flags"),
]

TYPE_BWD = dict(w_t=None, w_h=None, ld_grad=8, ld_out=8, ld_gtable=8, B=2, N=3, D=8, F=4, R1=3, io=0, stream=None)
TYPE_BWD_ENTRIES = [
    ("gr_type_layer_backward", {"fp32", "atomic"}, "gr_type_layer_backward_ex", None),
    ("gr_type_layer_backward_ex", {"ex", "atomic"}, "gr_type_layer_backward_ex", None),
    ("gr_type_layer_backward_det", {"fp32", "det"}, "gr_type_layer_backward_det_ex", "gr_type_layer_backward_det"),
    ("gr_type_layer_backward_det_ex", {"ex", "det"}, "gr_type_layer_backward_det_ex", "gr_type_layer_backward_det"),
]
_TSIZES = "bad sizes (need 0 < D <= 512)"
TYPE_BWD_CASES = [
    ({"fp32", "ex"}, dict(grad_out=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(grad_table=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(rel_h=None), INVALID, "null edge arrays"),
    ({"fp32", "ex"}, dict(D=0), INVALID, _TSIZES),
    ({"fp32", "ex"}, dict(D=513, ld_grad=513, ld_out=513, ld_gtable=513), INVALID, _TSIZES),
    ({"fp32", "ex"}, dict(F=-1), INVALID, _TSIZES),
    ({"fp32", "ex"}, dict(ld_grad=7), INVALID, "leading dimension smaller than D"),
    ({"fp32", "ex"}, dict(ld_out=7), INVALID, "leading dimension smaller than D"),
    ({"fp32", "ex"}, dict(ld_gtable=7), INVALID, "leading dimension smaller than D"),
    ({"ex"}, dict(io=2), INVALID, "unknown io flags"),
    ({"atomic"}, dict(B=0), INVALID, _TSIZES),        # the atomic forms take B, N and row pointers, the others R1
    ({"atomic"}, dict(N=0), INVALID, _TSIZES),
    ({"atomic"}, dict(rowptr_t=None), INVALID, "null pointer"),
    ({"det"}, dict(R1=0), INVALID, _TSIZES),
    ({"det"}, dict(rix_ptr_h=None), INVALID, "null pointer"),
    ({"det"}, dict(row_of_t=None), INVALID, "null edge arrays"),
    ({"det"}, dict(workspace_bytes="short"), WORKSPACE, None),
    ({"det"}, dict(workspace=None), WORKSPACE, None),
]

GNET_AGG = dict(ld_self=8, ld_head=8, ld_sum=8, ld_grad=8, ld_gself=8, ld_ghead=8, seed=None, p=0.0, B=2, N=3,
                D=8, R1=3, F=4, io=0, stream=None)
GNET_AGG_ENTRIES = [
    ("gr_graft_aggregate_train", {"fp32", "fwd"}, "gr_graft_aggregate_train_ex", None),
    ("gr_graft_aggregate_train_ex", {"ex", "fwd"}, "gr_graft_aggregate_train_ex", None),
    ("gr_graft_aggregate_backward", {"fp32"}, "gr_graft_aggregate_backward_ex", None),
    ("gr_graft_aggregate_backward_ex", {"ex"}, "gr_graft_aggregate_backward_ex", None),
    ("gr_graft_aggregate_backward_det", {"fp32", "det"}, "gr_graft_aggregate_backward_det_ex",
     "gr_graft_aggregate_backward_det"),
    ("gr_graft_aggregate_backward_det_ex", {"ex", "det"}, "gr_graft_aggregate_backward_det_ex",
     "gr_graft_aggregate_backward_det"),
]
_GSIZES = "bad sizes (need 0 < D <= 512)"
_LD = "leading dimension smaller than D"
GNET_AGG_CASES = [
    ({"fp32", "ex"}, dict(self_tab=None), INVALID, "null pointer"),
    ({"fwd"}, dict(rowptr_t=None), INVALID, "null pointer"),
    ({"fp32", "ex"}, dict(B=0), INVALID, _GSIZES),
    ({"fp32", "ex"}, dict(N=0), INVALID, _GSIZES),
    ({"fp32", "ex"}, dict(D=0), INVALID, _GSIZES),
    ({"fp32", "ex"}, dict(D=513, ld_self=513, ld_head=513), INVALID, _GSIZES),
    ({"fp32", "ex"}, dict(ld_self=7), INVALID, _LD),
    ({"fp32", "ex"}, dict(ld_head=7), INVALID, _LD),
    ({"fp32", "ex"}, dict(p=1.0), INVALID, "@dropout probability outside [0, 1)"),
    ({"fp32", "ex"}, dict(p=-0.25), INVALID, "@dropout probability outside [0, 1)"),
    ({"fp32", "ex"}, dict(p=0.5), INVALID, "@null seed with p > 0"),
    ({"ex"}, dict(io=2), INVALID, "unknown io flags"),
    ({"fwd"}, dict(sum_out=None), INVALID, "null pointer"),
    ({"fwd"}, dict(ld_sum=7), INVALID, _LD),
    ({"det"}, dict(F=-1), INVALID, _GSIZES),
    ({"det"}, dict(R1=0), INVALID, _GSIZES),
    ({"det"}, dict(rix_fact=None), INVALID, "null pointer"),
    ({"det"}, dict(tails=None), INVALID, "null pointer"),
    ({"det"}, dict(workspace_bytes="short"), WORKSPACE, None),
    ({"det"}, dict(workspace=None), WORKSPACE, None),
]
# the backward forms: gradient outputs and their leading dimensions
GNET_AGG_BWD_CASES = [
    (dict(rowptr_h=None), INVALID, "null pointer"),
    (dict(grad_head=None), INVALID, "null pointer"),
    (dict(grad_s=None), INVALID, "null pointer"),
    (dict(ld_grad=7), INVALID, _LD),
    (dict(ld_ghead=7), INVALID, _LD),
]

ATTN = dict(Q=3, ldr=8, R1=3, B=2, max_fact=5, D=8, ld_grel=8, stream=None)
ATTN_ENTRIES = [
    ("gr_graft_attention_backward", {"fp32"}, "gr_graft_attention_backward", None),
    ("gr_graft_attention_backward_det", {"fp32", "det"}, "gr_graft_attention_backward_det",
     "gr_graft_attention_backward_det"),
]
_ASIZES = "bad sizes (need 0 < D <= 512, 0 < B <= 65535, Q > 0)"
_DSIZES = "bad sizes (need 0 < D <= 512, Q > 0)"
ATTN_CASES = [
    ({"fp32"}, dict(qh=None), INVALID, "null pointer"),
    ({"fp32"}, dict(grad_rel=None), INVALID, "null pointer"),
]
for _bad in (dict(B=0), dict(D=0), dict(D=513, ldr=513, ld_grel=513), dict(Q=0), dict(max_fact=-1), dict(R1=0),
             dict(ldr=7), dict(ld_grel=7)):
    ATTN_CASES.append(({"fp32"}, _bad, INVALID, None))     # message differs between the two forms
ATTN_CASES += [
    ({"det"}, dict(rix_ptr=None), INVALID, "null pointer"),
    ({"det"}, dict(rix_slot=None), INVALID, "null pointer"),
    ({"det"}, dict(B=1 << 16, max_fact=1 << 15), INVALID, "B*max_fact exceeds int32"),
    ({"det"}, dict(workspace_bytes="short"), WORKSPACE, None),
    ({"det"}, dict(workspace=None), WORKSPACE, None),
]


def _workspace_need(name, a):
    lib = _lib.load()
    if name.startswith("gr_aggregate_backward_det"):
        return lib.gr_aggregate_backward_det_workspace_bytes(a["B"], a["N"], a["D"], a["I"], a["F"])
    if name.startswith("gr_type_layer_backward_det"):
        return lib.gr_type_layer_backward_det_workspace_bytes(a["F"], a["D"])
    if name.startswith("gr_graft_aggregate_backward_det"):
        return lib.gr_graft_aggregate_backward_det_workspace_bytes(a["F"], a["D"])
    return lib.gr_graft_attention_backward_det_workspace_bytes(a["B"], a["max_fact"], a["Q"], a["D"])


def _cases():
    groups = [(AGG, AGG_ENTRIES, AGG_CASES), (AGG_BWD, AGG_BWD_ENTRIES, AGG_BWD_CASES),
              (TYPE, TYPE_ENTRIES, TYPE_CASES), (TYPE_BWD, TYPE_BWD_ENTRIES, TYPE_BWD_CASES),
              (GNET_AGG, GNET_AGG_ENTRIES, GNET_AGG_CASES), (ATTN, ATTN_ENTRIES, ATTN_CASES)]
    for good, entries, cases in groups:
        for name, forms, arg_name, ws_name in entries:
            mine = [(o, rc, m) for f, o, rc, m in cases if f & forms]
            if name.startswith("gr_graft_aggregate_backward"):
                mine += GNET_AGG_BWD_CASES
            for over, rc, msg in mine:
                if name.startswith("gr_graft_attention_backward") and msg is None and rc == INVALID:
                    msg = _DSIZES if "det" in forms else _ASIZES
                yield pytest.param(name, good, over, rc, msg, arg_name, ws_name,
                                   id="%s-%s" % (name, "-".join("%s=%s" % kv for kv in over.items())))


@pytest.mark.parametrize("name,good,over,rc,msg,arg_name,ws_name", list(_cases()))
def test_entry_point_refuses(name, good, over, rc, msg, arg_name, ws_name):
    args = {p: v for p, v in good.items() if p in PARAMS[name]}
    need = _workspace_need(name, args) if "workspace_bytes" in PARAMS[name] else 0
    args["workspace_bytes"] = need
    assert set(over) <= set(PARAMS[name]), "a refusal case must override parameters of the entry point it calls"
    args.update(over)
    if args.get("workspace_bytes") == "short":
        args["workspace_bytes"] = need - 1
    if rc == WORKSPACE:
        expected = "%s: workspace too small (%d < %d)" % (ws_name, args["workspace_bytes"], need)
    elif msg.startswith("@"):            # dropout arguments are checked in a helper that reports its own name
        expected = "drop_args: invalid argument: " + msg[1:]
    else:
        expected = "%s: invalid argument: %s" % (arg_name, msg)
    assert need > 0 or "workspace_bytes" not in PARAMS[name]
    assert call(name, args) == (rc, expected)
