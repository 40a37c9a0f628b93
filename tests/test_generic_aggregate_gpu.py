"""GPU: the generic aggregation kernel (csrc/aggregate.cu, ``agg_kernel``) against float64 in every instantiation its
launcher picks, on the case table of tests/agg_cases.py.

Each case is one set of logical inputs; its runs call ``ops.aggregate`` / ``ops.aggregate_dual`` with different output
layouts, alignments and options, which select different instantiations (VEC, CH, NI, DT / SEGP, bulk-TMA staging, fp32,
bf16 or split-bf16 planes output).  Every run is held to:

* accuracy: a message element sums n edges (n the row's in-degree in that direction) into two fp32 chains A, S and
  forms A - S, with c = w*(w*p): within (2n + 8) u of ``fp64_ref.aggregate_abs`` (u = 2^-24); where the float64 value
  is exactly 0 the output is exactly 0;
* bit identity: all instantiations run the same per-edge FMA chain in CSR order and the same epilogue (``ffma2`` is
  fmaf per lane), so every fp32 output equals the two single-direction calls bit for bit, the planes are
  hi = bf16_rn(y), lo = bf16_rn(y - hi) of it and a bf16 output is bf16_rn(y);
* writes: nothing outside the I (or 2I) segments changes; plane columns D .. Dw - 1 are zero (Dw = min(round16(D),
  max(pitch, D))) and columns Dw .. pitch - 1 keep their sentinel; ``possible`` is written for every row.
"""
import copy

import numpy as np
import pytest
import torch

from gnn_rag_b200 import ops

import agg_cases as C
import fp64_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64
SENT = -7.25           # fp32 sentinel
PSENT = 3.0            # bf16 sentinel


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t if dtype is None else t.to(dtype)


def _off_by_one(t):
    """The same values starting one element past the allocation's (256-byte aligned) start."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=DEV)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def _segments(case, run):
    """(direction, instruction, first column) of every output segment of a run."""
    s = run.seg(case.D)
    if run.kind in C.SINGLE_KINDS:
        d = 1 if run.kind == "inv" else 0
        return [(d, j, run.col0 + j * s) for j in range(case.I)]
    return [(d, j, run.col0 + (2 * j + d) * s) for j in range(case.I) for d in (0, 1)]


def _call(case, run, g, x):
    """Run one call; returns (fp32 out or None, bf16 out or None, planes or None, possible or None, plan of the
    pointers actually passed)."""
    D, I, Nt = case.D, case.I, case.Nt
    W = run.width(D, I)
    tf, ti = x["tf"], x["ti"]
    if run.table_off:
        tf, ti = _off_by_one(tf), _off_by_one(ti)
    if run.csr_off:
        g = copy.copy(g)
        for name in ("src_t", "rel_t", "src_h", "rel_h"):
            setattr(g, name, _off_by_one(getattr(g, name)))
    out = bf = planes = possible = None
    s = run.seg(D)
    ops.set_option("agg_tma", run.tma)
    try:
        if run.kind in C.SINGLE_KINDS:
            d = "inv" if run.kind == "inv" else "fwd"
            tab, ww = (ti, x["w_h"]) if d == "inv" else (tf, x["w_t"])
            if run.kind == "bf16":
                bf = torch.full((Nt, W), PSENT, dtype=torch.bfloat16, device=DEV)
            else:
                out = torch.full((Nt, W), SENT, device=DEV)
            if run.kind == "possible":
                possible = torch.full((Nt,), -1.0, device=DEV)
            o = out if out is not None else bf
            rp, src, rel, _f = g.csr(d)
            pl = C.plan(D, I, 1, out=out.data_ptr() if out is not None else None,
                        out_bf=bf.data_ptr() if bf is not None else None, out_row_stride=o.stride(0),
                        out_col0=run.col0, seg_stride_j=s, ins=x["ins"].data_ptr(), tables=(tab.data_ptr(),),
                        srcs=(src.data_ptr(),), rels=(rel.data_ptr(),), agg_tma=run.tma)
            ops.aggregate(g, d, x["prior"], tab, x["ins"], out=o, out_col0=run.col0, seg_stride=s, w=ww,
                          possible=possible)
        else:
            if run.kind in ("dual", "both"):
                out = torch.full((Nt, W), SENT, device=DEV)
            if run.kind in ("planes", "both"):
                planes = tuple(torch.full((Nt, W), PSENT, dtype=torch.bfloat16, device=DEV) for _ in range(2))
            pl = C.plan(D, I, 2, out=out.data_ptr() if out is not None else None,
                        out_hi=planes[0].data_ptr() if planes else None,
                        out_lo=planes[1].data_ptr() if planes else None,
                        out_row_stride=out.stride(0) if out is not None else 0, out_col0=run.col0,
                        seg_stride_j=2 * s, seg_stride_dir=s, ld_planes=planes[0].stride(0) if planes else 0,
                        ins=x["ins"].data_ptr(), tables=(tf.data_ptr(), ti.data_ptr()),
                        srcs=(g.src_t.data_ptr(), g.src_h.data_ptr()), rels=(g.rel_t.data_ptr(), g.rel_h.data_ptr()),
                        agg_tma=run.tma)
            ops.aggregate_dual(g, x["prior"], tf, ti, x["ins"], out, run.col0, x["w_t"], x["w_h"], planes=planes,
                               seg_pitch=s)
    finally:
        ops.set_option("agg_tma", 0)
    return out, bf, planes, possible, pl


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


@pytest.mark.parametrize("case", C.CASES, ids=lambda c: c.name)
def test_generic_aggregate_vs_fp64(case):
    D, I, B, N, Nt = case.D, case.I, case.B, case.N, case.Nt
    xi = C.make_inputs(case)
    h, r, t = xi["heads"], xi["rels"], xi["tails"]
    facts = tuple(_t(a) for a in (h, r, t))
    g = ops.csr_build(*facts, B, N, case.R1)
    g.check_status()
    x = dict(tf=_t(xi["table_fwd"]), ti=_t(xi["table_inv"]), ins=_t(xi["ins"]), prior=_t(xi["prior"]),
             w_t=None, w_h=None)
    w64 = None
    if xi["w"] is not None:
        wd = _t(xi["w"])
        x["w_t"], x["w_h"] = ops.gather_f32(wd, g.fact_t), ops.gather_f32(wd, g.fact_h)
        w64 = wd.to(F64)
    ins64, prior64 = x["ins"].to(F64), x["prior"].to(F64)
    want, bound = [], []
    for d, (tab, dst) in enumerate(((x["tf"], t), (x["ti"], h))):
        direction = ("fwd", "inv")[d]
        want.append(R.aggregate(tab.to(F64), ins64, prior64, *facts, w64, direction).view(Nt, I, D))
        scale = R.aggregate_abs(tab.to(F64), ins64, prior64, *facts, w64, direction).view(Nt, I, D)
        n = _t(np.bincount(dst, minlength=Nt), F64).view(Nt, 1, 1)
        bound.append((2 * n + 8) * U * scale)
    for d in (0, 1):
        assert (want[d] == 0).any() and (want[d] != 0).any()
    if case.hub:                                  # the edge at slice position 1024 is far outside the bound
        for d, (src_of, dst, tab) in enumerate(((h, t, x["tf"]), (t, h, x["ti"]))):
            f = C.csr_order(dst, Nt)[C.csr_rowptr(dst, Nt)[0] + C.EDGE_CAP]
            row, src = int(dst[f]), int(src_of[f])
            planted = C.BIG ** 2 * prior64.view(-1)[src] * torch.relu(tab[int(r[f])].to(F64) * ins64[row // N])
            nz = bound[d][row] > 0
            ratio = (planted[nz] / bound[d][row][nz]).max().item()
            print("planted/bound %s dir %d: %.3g" % (case.name, d, ratio))
            assert ratio > 100

    # the two singles at the default layout: the bits every other run must reproduce
    y = [ops.aggregate(g, dname, x["prior"], tab, x["ins"], w=ww).view(Nt, I, D)
         for dname, tab, ww in (("fwd", x["tf"], x["w_t"]), ("inv", x["ti"], x["w_h"]))]
    worst = 0.0
    for d in (0, 1):
        err = (y[d].to(F64) - want[d]).abs()
        assert (err <= bound[d]).all(), (d, (err / bound[d]).nan_to_num(posinf=1e30).max().item())
        assert (y[d][want[d] == 0] == 0).all()
        nz = bound[d] > 0
        worst = max(worst, (err[nz] / bound[d][nz]).max().item())
    print("max err/bound %s: %.3g" % (case.name, worst))
    hi_want = [v.to(torch.bfloat16) for v in y]
    lo_want = [(v - hv.float()).to(torch.bfloat16) for v, hv in zip(y, hi_want)]
    poss_want = R.possible(prior64, facts, w64, Nt)[0]

    for run in case.runs:
        out, bf, planes, possible, pl = _call(case, run, g, x)
        tag = (case.name, run)
        assert pl == C.launches(case, run), tag          # the table's instantiations are the ones that ran
        segs = _segments(case, run)
        if out is not None:
            written = torch.zeros(out.shape[1], dtype=torch.bool, device=DEV)
            for d, j, c in segs:
                got = out[:, c:c + D]
                assert torch.equal(_bits(got), _bits(y[d][:, j].contiguous())), tag
                assert ((got.to(F64) - want[d][:, j]).abs() <= bound[d][:, j]).all(), tag
                written[c:c + D] = True
            assert (out[:, ~written] == SENT).all(), tag
        if bf is not None:
            written = torch.zeros(bf.shape[1], dtype=torch.bool, device=DEV)
            for d, j, c in segs:
                assert torch.equal(_bits(bf[:, c:c + D]), _bits(hi_want[d][:, j].contiguous())), tag
                written[c:c + D] = True
            assert (bf[:, ~written] == PSENT).all(), tag
        if planes is not None:
            hi, lo = planes
            Dw = C.pad_cols(D, run.seg(D))
            written = torch.zeros(hi.shape[1], dtype=torch.bool, device=DEV)
            for d, j, c in segs:
                assert torch.equal(_bits(hi[:, c:c + D]), _bits(hi_want[d][:, j].contiguous())), tag
                assert torch.equal(_bits(lo[:, c:c + D]), _bits(lo_want[d][:, j].contiguous())), tag
                pv = hi[:, c:c + D].to(F64) + lo[:, c:c + D].to(F64)
                wj = want[d][:, j]
                assert ((pv - wj).abs() <= bound[d][:, j] + 2.0 ** -17 * wj.abs()).all(), tag
                assert (hi[:, c + D:c + Dw] == 0).all() and (lo[:, c + D:c + Dw] == 0).all(), tag
                written[c:c + Dw] = True
            assert (hi[:, ~written] == PSENT).all() and (lo[:, ~written] == PSENT).all(), tag
        if possible is not None:
            assert torch.equal(possible.to(F64), poss_want), tag
