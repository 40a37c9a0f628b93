"""CPU: every training entry point refuses bad arguments with a fixed (status, gr_last_error()) pair, whichever of
its fp32, `_ex`, `_det` and `_det_ex` forms is called, and admits exactly the shapes the matching rule of ops
admits.  Every call below is refused before any CUDA call, so the
pointers are placeholders that are never dereferenced."""
import ctypes
import os
import re

import pytest

from gnn_rag_b200 import _lib, ops

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


# ---- gr_aggregate_dual_abs: the hi-only output needs a persistent kernel ---------------------------------------------
# Only the persistent kernels (agg_abs_ws 1 and 2; 3 falls back to 2) have a form that writes the hi plane alone; the
# one-CTA-per-tile kernel (no tile counter, or agg_abs_ws 0) always stores the lo plane.  An admitted call is refused
# later in the same entry point by a misaligned padded table, before any CUDA call.

DUAL_ABS = dict(w_t=None, w_h=None, table_rows=3, out_lo=None, ld_planes=2 * 2 * 208, out_col0=0, seg_pitch=208,
                B=2, N=64, D=200, I=2, F=4, stream=None)
_DUAL_ABS_ERR = "gr_aggregate_dual_abs: invalid argument: "
_HI_ONLY = "hi-only output (bf16 activation storage) needs a persistent kernel (a tile counter and agg_abs_ws != 0)"


@pytest.mark.parametrize("mode,counter,refused", [(0, True, True), (1, True, False), (2, True, False),
                                                  (3, True, False), (2, False, True)])
def test_aggregate_dual_abs_hi_only_needs_a_persistent_kernel(mode, counter, refused):
    args = dict(DUAL_ABS, pn_fwd=PTR + 8, tile_counter=PTR if counter else None)
    ops.set_option("agg_abs_ws", mode)
    try:
        got = call("gr_aggregate_dual_abs", args)
    finally:
        ops.set_option("agg_abs_ws", 2)
    want = _HI_ONLY if refused else "misaligned planes / padded tables"
    assert got == (INVALID, _DUAL_ABS_ERR + want)
    args["out_lo"] = PTR                                  # both planes: every mode and the counter-less kernel admit it
    assert call("gr_aggregate_dual_abs", args) == (INVALID, _DUAL_ABS_ERR + "misaligned planes / padded tables")


# ---- the shape rules of ops against the entry points that enforce them ----------------------------------------------
# For each bound of a rule: the largest shape it admits and the first it refuses.  The entry point must refuse the
# second with its shape message.  It refuses the first as well, but later, by a check it runs after the shape check
# (a null output, a stride, a workspace), so that no call reaches CUDA.

UNSUPPORTED = -4


def _host_ptrs(n):
    """The host array of n weight pointers that the question-side entry points read before their shape check."""
    return (ctypes.c_void_p * n)(*[PTR] * n)


def _agg_bwd(D, I):
    # grad_col0 = 1 puts the last segment one column past the row: the stride check comes after the shape check
    args = dict(AGG_BWD, D=D, I=I, seg_stride=max(D, 1), grad_row_stride=I * D, grad_col0=1)
    err = "gr_aggregate_backward_ex: invalid argument: "
    return "gr_aggregate_backward", args, (INVALID, err + _STRIDE), (INVALID, err + _SIZES)


def _type_bwd(D):
    args = dict(TYPE_BWD, D=D, ld_grad=D, ld_out=D, ld_gtable=D, grad_table=None)
    err = "gr_type_layer_backward_ex: invalid argument: "
    return "gr_type_layer_backward", args, (INVALID, err + "null pointer"), (INVALID, err + _TSIZES)


def _instructions(Q, D, I):
    args = dict(pad_id=0, Wq_host=_host_ptrs(I), bq_host=_host_ptrs(I), out=None, attn_out=None, B=2, Q=Q, D=D, I=I,
                stream=None)
    err = "gr_instructions: invalid argument: "
    refused = "bad shape (num_ins <= 8)" if I > 8 else "question length x entity_dim too large for shared memory"
    return "gr_instructions", args, (INVALID, err + "null pointer"), (INVALID, err + refused)


def _query_reform(D, I):
    args = dict(ldh=D, Wr_host=_host_ptrs(I), Wg_host=_host_ptrs(I), ins_out=None, seed_out=None, B=2, N=3, D=D, I=I,
                stream=None)
    err = "gr_query_reform: invalid argument: "
    refused = "bad shape (D <= 1024, num_ins <= 8)" if D > 1024 or I > 8 else \
        "num_ins x entity_dim too large for shared memory"
    return "gr_query_reform", args, (INVALID, err + "null pointer"), (INVALID, err + refused)


def _linear_tc(N, K):
    M = 16
    args = dict(lda=K, ldw=K, bias=None, ldc=N, M=M, N=N, K=K, flags=0, workspace_bytes=0, stream=None)
    need = _lib.load().gr_linear_tc_workspace_bytes(M, N, K)
    return ("gr_linear_tc", args, (WORKSPACE, "gr_linear_tc: workspace too small (0 < %d)" % need),
            (UNSUPPORTED, "gr_linear_tc: unsupported shape M=%d N=%d K=%d (need 8 <= N <= 256, K >= 8)" % (M, N, K)))


# (ops rule, entry point case, largest admitted shape, first refused shape)
RULE_BOUNDS = [
    ("aggregate_backward_ok", _agg_bwd, (256, 4), (257, 4)),
    ("aggregate_backward_ok", _agg_bwd, (1, 4), (0, 4)),
    ("aggregate_backward_ok", _agg_bwd, (256, 4), (256, 5)),
    ("aggregate_backward_ok", _agg_bwd, (256, 1), (256, 0)),
    ("fact_train_ok", _type_bwd, (512,), (513,)),
    ("instructions_ok", _instructions, (20, 50, 8), (20, 50, 9)),
    ("instructions_ok", _instructions, (244, 200, 2), (245, 200, 2)),      # (Q D + 9 D + 2 Q) floats <= 200 KB
    ("query_reform_ok", _query_reform, (1024, 1), (1025, 1)),
    ("query_reform_ok", _query_reform, (8, 8), (8, 9)),
    ("query_reform_ok", _query_reform, (768, 3), (769, 3)),              # 16 D floats <= 48 KB
    ("tc_linear_ok", _linear_tc, (8, 8), (7, 8)),
    ("tc_linear_ok", _linear_tc, (256, 8), (257, 8)),
    ("tc_linear_ok", _linear_tc, (8, 8), (8, 7)),
]


@pytest.mark.parametrize("rule,case,admitted,refused", RULE_BOUNDS,
                         ids=["%s-%s" % (r[0], "x".join(map(str, r[3]))) for r in RULE_BOUNDS])
def test_ops_shape_rule_is_the_entry_points(rule, case, admitted, refused):
    ok = getattr(ops, rule)
    name, args, past_shape_check, _ = case(*admitted)
    assert ok(*admitted) and call(name, args) == past_shape_check
    name, args, _, shape_refusal = case(*refused)
    assert not ok(*refused) and call(name, args) == shape_refusal
