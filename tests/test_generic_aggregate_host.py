"""CPU: the launch restatement of tests/agg_cases.py on hand-worked examples of csrc/aggregate.cu, and the reach of
the case table tests/test_generic_aggregate_gpu.py runs: every instantiation and runtime branch of the generic
aggregation kernel is taken by at least one case, so removing a case or a run that is the only one to reach a
variant fails here."""
import numpy as np

import agg_cases as C
from agg_cases import Launch


def _l(vec, ch, passes, ni=1, j0=0, dt=0, segp=0, use_tma=False, planes=False, out_bf16=False):
    return Launch(vec, ch, passes, ni, j0, dt, segp, use_tma, planes, out_bf16)


def test_plan_on_worked_examples():
    # D = 50 (the reference's ReaRev width): float2 lanes, one 64-column chunk
    assert C.plan(50, 1, 1, out=0, out_row_stride=50, seg_stride_j=50) == [_l(2, 1, 1)]
    # D = 200 dual at pitch 208 without TMA: the DT-specialised instance, fp32 then planes, per group of 4
    got = C.plan(200, 5, 2, out=0, out_hi=0, out_lo=0, out_row_stride=2080, ld_planes=2080, seg_stride_j=416,
                 seg_stride_dir=208, tables=(0, 0))
    assert got == [_l(4, 2, 1, 4, 0, 200, 208), _l(4, 2, 1, 4, 0, 200, 208, planes=True),
                   _l(4, 2, 1, 1, 4, 200, 208), _l(4, 2, 1, 1, 4, 200, 208, planes=True)]
    # ... at pitch 200 as well; with agg_tma the runtime-D kernel stages with bulk copies instead
    assert C.plan(200, 2, 2, out=0, out_row_stride=800, seg_stride_j=400, seg_stride_dir=200,
                  tables=(0, 0))[0].segp == 200
    assert C.plan(200, 2, 2, out=0, out_row_stride=800, seg_stride_j=400, seg_stride_dir=200, tables=(0, 0),
                  agg_tma=1) == [_l(4, 2, 1, 2, use_tma=True)]
    # a pitch that is neither 200 nor 208 stays generic; so does a single direction
    assert C.plan(200, 1, 2, out=0, out_row_stride=440, seg_stride_j=440, seg_stride_dir=220,
                  tables=(0, 0))[0].dt == 0
    assert C.plan(200, 1, 1, out=0, out_row_stride=200, seg_stride_j=200)[0].dt == 0
    # D = 400: two column passes of 256; D = 129 at VEC 1: three passes of 64
    assert C.plan(400, 1, 1, out=0, out_row_stride=400, seg_stride_j=400) == [_l(4, 2, 2)]
    assert C.plan(129, 1, 1, out=0, out_row_stride=129, seg_stride_j=129) == [_l(1, 2, 3)]
    # alignment alone lowers VEC at D % 4 == 0: an odd out_col0, a column offset of 2, a table one float off
    assert C.plan(64, 1, 1, out=0, out_col0=1, out_row_stride=65, seg_stride_j=64) == [_l(1, 2, 1)]
    assert C.plan(64, 1, 1, out=0, out_col0=2, out_row_stride=66, seg_stride_j=64) == [_l(2, 1, 1)]
    assert C.plan(64, 1, 1, out=0, out_row_stride=64, seg_stride_j=64, tables=(4,)) == [_l(1, 2, 1)]
    # I = 6: NI 4 at j0 = 0, NI 2 at j0 = 4
    assert [(x.ni, x.j0) for x in C.plan(33, 6, 1, out=0, out_row_stride=198, seg_stride_j=33)] == [(4, 0), (2, 4)]
    # bf16 output never stages through TMA; TMA needs 16-byte aligned src and rel
    assert C.plan(64, 1, 1, out_bf=0, out_row_stride=64, seg_stride_j=64, agg_tma=1) == [_l(4, 1, 1, out_bf16=True)]
    assert C.plan(64, 1, 1, out=0, out_row_stride=64, seg_stride_j=64, agg_tma=1, srcs=(4,))[0].use_tma is False
    # planes only need 2-byte alignment per lane element: an 8-byte plane base keeps VEC 4
    assert C.plan(64, 1, 2, out_hi=8, out_lo=8, ld_planes=128, seg_stride_j=128, seg_stride_dir=64,
                  tables=(0, 0))[0].vec == 4


def test_pad_columns():
    assert C.pad_cols(50, 50) == 50 and C.pad_cols(50, 56) == 56 and C.pad_cols(50, 64) == 64
    assert C.pad_cols(50, 80) == 64 and C.pad_cols(200, 208) == 208 and C.pad_cols(200, 200) == 200
    assert C.pad_cols(1, 1) == 1 and C.pad_cols(1, 16) == 16


def _all():
    for case in C.CASES:
        for run in case.runs:
            yield case, run, C.launches(case, run)


def test_case_table_reaches_every_instantiation():
    ls = [(case, run, x) for case, run, xs in _all() for x in xs]
    assert {(x.vec, x.ch) for _, _, x in ls} == {(v, c) for v in (4, 2, 1) for c in (1, 2)}
    assert {1, 2, 3} <= {x.passes for _, _, x in ls}
    # VEC lowered by alignment alone, at D % 4 == 0
    assert {x.vec for c, _, x in ls if c.D % 4 == 0} >= {1, 2, 4}
    # every NI as the first group and as a tail group
    assert {(x.ni, x.j0 > 0) for _, _, x in ls} == {(n, t) for n in (1, 2, 3, 4) for t in (False, True)}
    assert {c.I for c in C.CASES} >= set(range(1, 9))
    assert {(x.use_tma, x.planes) for _, _, x in ls} == {(a, b) for a in (False, True) for b in (False, True)}
    assert any(x.out_bf16 for _, _, x in ls)
    # the DT-specialised instance: both pitches, fp32 and planes, I in {1, 4, 5, 8}, N < 64, j0 > 0
    dt = [(c, x) for c, _, x in ls if x.dt]
    assert {(x.segp, x.planes) for _, x in dt} == {(p, q) for p in (200, 208) for q in (False, True)}
    assert {c.I for c, _ in dt} >= {1, 4, 5, 8}
    assert any(c.N < 64 for c, _ in dt) and any(x.j0 > 0 for _, x in dt)
    # ... and the same inputs with agg_tma, where the runtime-D kernel runs instead
    for case in {c.name: c for c, _ in dt}.values():
        assert any(r.tma and all(x.dt == 0 and x.use_tma for x in C.launches(case, r)) for r in case.runs)
    # TMA requested with misaligned src / rel: plain staging
    assert any(r.tma and r.csr_off and not any(x.use_tma for x in xs) for _, r, xs in _all())


def test_case_table_reaches_every_output_kind():
    runs = [(c, r) for c in C.CASES for r in c.runs]
    kinds = {r.kind for _, r in runs}
    assert kinds == set(C.SINGLE_KINDS) | set(C.DUAL_KINDS)
    poss = [(c, r) for c, r in runs if r.kind == "possible"]
    assert any(c.I > 4 and C.launches(c, r)[0].passes > 1 for c, r in poss)
    dual = [(c, r.seg(c.D)) for c, r in runs if r.kind == "dual"]
    assert any(p == c.D for c, p in dual) and any(p > c.D for c, p in dual)
    planes = [(c, r.seg(c.D)) for c, r in runs if r.kind in ("planes", "both")]
    assert any(p == c.D and p != C.r16(c.D) for c, p in planes)
    assert any(p == C.r16(c.D) != c.D for c, p in planes)
    assert any(p > C.r16(c.D) for c, p in planes)
    assert any(c.D < p < C.r16(c.D) for c, p in planes)          # a pad that stops at the pitch


def _rows_of_tiles(case):
    return [(r0, min(r0 + C.K_ROWS, case.Nt)) for r0 in range(0, case.Nt, C.K_ROWS)]


def test_case_table_reaches_every_tile_geometry():
    Ns = {c.N for c in C.CASES}
    assert {1, 5, 31, 63, 64, 65, 200} <= Ns
    assert any(c.N * 3 <= C.K_ROWS and c.B >= 3 for c in C.CASES)          # more than two questions in one tile
    assert any(c.N % C.K_ROWS and c.N > C.K_ROWS for c in C.CASES)          # a tile straddling a question boundary
    assert any(c.Nt % C.K_ROWS and c.Nt > C.K_ROWS for c in C.CASES)
    assert any(c.Nt < C.K_ROWS for c in C.CASES)


def test_case_inputs_reach_every_edge_branch():
    hub_seen = tma_f_seen = 0
    for case in C.CASES:
        x = C.make_inputs(case)
        h, r, t, Nt = x["heads"], x["rels"], x["tails"], case.Nt
        F = len(h)
        assert F > 0 and h.max() < Nt and t.max() < Nt
        assert (h // case.N == t // case.N).all()                            # facts stay inside their question
        deg_t, deg_h = np.bincount(t, minlength=Nt), np.bincount(h, minlength=Nt)
        assert ((deg_t == 0) & (deg_h == 0)).any()                           # rows with no in-edges at all
        assert r.min() == 0 and r.max() == case.R1 - 1
        assert (x["ins"] == 0).any() and (x["ins"] > 0).any() and (x["ins"] < 0).any()
        assert (x["table_fwd"][1] >= 0).all()
        if case.weights:
            assert (x["w"] == 0).any()
        if case.prior == "onehot":
            assert ((x["prior"] > 0).sum(1) == 1).all()
        if F % 4 and any(run.tma for run in case.runs):
            tma_f_seen += 1
        if case.hub:
            for dst in (t, h):
                rp = C.csr_rowptr(dst, Nt)
                r0, r1 = _rows_of_tiles(case)[0]
                assert rp[r1] - rp[r0] > 2 * C.EDGE_CAP
                pos = rp[r0:r1 + 1] - rp[r0]
                straddle = np.flatnonzero((pos[:-1] < C.EDGE_CAP) & (pos[1:] > C.EDGE_CAP))
                assert len(straddle) == 1 and straddle[0] > 0                # a non-first row straddles the stage
                assert (pos[:-1] > C.EDGE_CAP).sum() > 5                      # later rows lie wholly past it
                slot = C.csr_order(dst, Nt)[rp[r0] + C.EDGE_CAP]
                assert x["w"][slot] == C.BIG
            hub_seen += 1
    assert hub_seen >= 2 and tma_f_seen >= 5
    assert any(c.prior == "onehot" for c in C.CASES) and any(not c.weights for c in C.CASES)
    # in-degrees that are not a multiple of 4 (the branch-free blocks of 4 pad the row's last block)
    x = C.make_inputs(C.CASES[0])
    assert (np.bincount(x["tails"]) % 4 != 0).any()
