"""The generic aggregation kernel (csrc/aggregate.cu, ``agg_kernel``) restated as the launches it makes, and the case
table its float64 test runs (tests/test_generic_aggregate_gpu.py).

``plan`` restates how ``launch_agg`` / ``launch_agg2`` / ``launch_agg3`` pick instantiations from the shape, the
strides, the pointer alignments and ``agg_tma``: one :class:`Launch` per kernel launch, in launch order.  It does not
import ``gnn_rag_b200``; the host test checks it on hand-worked examples and checks that the case table reaches every
instantiation and runtime branch the kernel has, so an edit to the table cannot silently drop one.

A :class:`Case` is one set of logical inputs (graph, tables, instructions, prior, weights), built by ``make_inputs``
in numpy from a seed.  Its :class:`Run` list says how the kernel is called on them: which entry point, which output
layout, which options.  Every run of a case computes the same values, so the test holds them bit for bit to each other
as well as to float64.
"""
from collections import namedtuple
from dataclasses import dataclass, field

import numpy as np

K_ROWS = 64          # destination rows per CTA tile (kRows)
EDGE_CAP = 1024      # staged edges per direction per tile (kEdgeCap)
BIG = 30.0           # weight of the planted edge at tile slice position EDGE_CAP (hub cases)

Launch = namedtuple("Launch", "vec ch passes ni j0 dt segp use_tma planes out_bf16")


def r16(n):
    return (n + 15) // 16 * 16


def plan(D, I, ndir, out=None, out_bf=None, out_hi=None, out_lo=None, out_row_stride=0, out_col0=0,
         seg_stride_j=0, seg_stride_dir=0, ld_planes=0, ins=0, tables=(0,), srcs=(0,), rels=(0,), agg_tma=0):
    """Launches of one message-mode call.  Pointer arguments are addresses (only their alignment matters; None = a
    null pointer, which is aligned); ``tables`` / ``srcs`` / ``rels`` hold one address per direction."""
    def al(p, nbytes):
        return p is None or p % nbytes == 0

    def aligned(v):
        a = 4 * v
        ok = (D % v == 0 and out_row_stride % v == 0 and out_col0 % v == 0 and seg_stride_j % v == 0
              and seg_stride_dir % v == 0 and al(out, a) and al(ins, a) and ld_planes % v == 0
              and al(out_hi, a // 2) and al(out_lo, a // 2) and al(out_bf, a // 2))
        return ok and all(al(t, a) for t in tables[:ndir])

    vec = 4 if aligned(4) else 2 if aligned(2) else 1
    ch = 2 if D > 32 * vec else 1
    passes = -(-D // (32 * vec * ch))
    tma = bool(agg_tma) and all(al(s, 16) and al(r, 16) for s, r in zip(srcs[:ndir], rels[:ndir]))
    launches = []
    for j0 in range(0, I, 4):
        ni = min(4, I - j0)
        dt = segp = 0
        if vec == 4 and ch == 2 and D == 200 and ndir == 2 and not tma:
            if (seg_stride_dir, seg_stride_j) in ((200, 400), (208, 416)):
                dt, segp = 200, seg_stride_dir
        base = dict(vec=vec, ch=ch, passes=passes, ni=ni, j0=j0, dt=dt, segp=segp)
        if out is not None:
            launches.append(Launch(**base, use_tma=tma and dt == 0, planes=False, out_bf16=False))
        if dt == 0 and out_bf is not None:
            launches.append(Launch(**base, use_tma=False, planes=False, out_bf16=True))
        if out_hi is not None:
            launches.append(Launch(**base, use_tma=tma and dt == 0, planes=True, out_bf16=False))
    return launches


# ------------------------------------------------------------------ the case table --------------------------------
SINGLE_KINDS = ("fwd", "inv", "bf16", "possible")     # gr_aggregate(_ex): one direction ("bf16" / "possible": fwd)
DUAL_KINDS = ("dual", "planes", "both")              # gr_aggregate_dual: fp32, planes, or both in one call


@dataclass(frozen=True)
class Run:
    """One call on a case's inputs.  ``pitch``: seg_stride of a single call / seg_pitch of a dual one (None = D);
    ``col0``: out_col0; ``extra``: columns past the last segment in each output row; ``table_off``: the tables start
    one float past a 16-byte boundary; ``csr_off``: src / rel start one entry past it (no bulk-TMA staging)."""
    kind: str
    pitch: int = None
    col0: int = 0
    extra: int = 0
    tma: int = 0
    table_off: int = 0
    csr_off: int = 0

    def seg(self, D):
        return D if self.pitch is None else self.pitch

    def width(self, D, I):
        """Columns of the output row (and of the planes' row, ld_planes)."""
        nseg = I if self.kind in SINGLE_KINDS else 2 * I
        return self.col0 + nseg * self.seg(D) + self.extra


@dataclass(frozen=True)
class Case:
    name: str
    D: int
    I: int
    B: int
    N: int
    runs: tuple
    R1: int = 23
    deg: float = 3.0            # mean random in-edges per node and direction
    prior: str = "dense"        # "dense": softmax per question; "onehot": one seed per question
    weights: bool = True        # per-fact weights (with exact zeros) or None
    hub: int = 0                # > 0: every row of the first tile gets `hub` more in-edges per direction
    seed: int = 0
    empty: float = 0.15         # share of rows with no fact at all
    tags: tuple = field(default=())

    @property
    def Nt(self):
        return self.B * self.N


def _std(D, extra=()):
    """The runs most cases share: both singles, dual fp32 at pitch D, planes at round16(D), possible."""
    return (Run("fwd", extra=3), Run("inv", col0=4, extra=4), Run("dual"), Run("planes", pitch=r16(D)),
            Run("possible")) + tuple(extra)


def _dt(I, N, B, seed):
    return Case("d200_dt_i%d_n%d" % (I, N), 200, I, B, N, seed=seed, runs=(
        Run("dual", pitch=200), Run("dual", pitch=208, col0=8), Run("planes", pitch=200),
        Run("planes", pitch=208, extra=16), Run("both", pitch=208),
        Run("dual", pitch=200, tma=1), Run("planes", pitch=208, tma=1), Run("both", pitch=208, tma=1),
        Run("fwd", pitch=208)))


CASES = (
    Case("d1_n1", 1, 3, 13, 1, seed=1, runs=(
        Run("fwd"), Run("inv"), Run("dual"), Run("planes"), Run("planes", pitch=16), Run("bf16"),
        Run("possible"), Run("dual", tma=1))),
    Case("d2_n5", 2, 2, 20, 5, seed=2, prior="onehot", runs=(
        Run("fwd", col0=2), Run("possible"), Run("dual"), Run("dual", pitch=3), Run("planes", pitch=16),
        Run("planes", pitch=20), Run("fwd", tma=1), Run("bf16"))),
    Case("d3_n31", 3, 4, 4, 31, seed=3, runs=(
        Run("fwd"), Run("inv"), Run("dual", pitch=3), Run("planes", pitch=16), Run("both", pitch=8),
        Run("dual", tma=1), Run("possible"))),
    Case("d33_n63", 33, 6, 3, 63, seed=4, prior="onehot", runs=_std(33, (
        Run("planes", pitch=64), Run("dual", tma=1), Run("bf16")))),
    Case("d50_n64", 50, 2, 3, 64, seed=5, runs=_std(50, (
        Run("fwd", col0=1), Run("planes", pitch=56), Run("bf16"), Run("fwd", tma=1), Run("dual", tma=1),
        Run("both", pitch=50)))),
    Case("d64_n65", 64, 7, 3, 65, seed=6, runs=_std(64, (
        Run("inv", col0=2), Run("fwd", table_off=1), Run("planes", pitch=80), Run("both", pitch=64),
        Run("dual", tma=1), Run("dual", tma=1, csr_off=1), Run("dual", pitch=66)))),
    Case("d65_n200", 65, 1, 2, 200, seed=7, runs=_std(65, (
        Run("planes", pitch=96), Run("bf16"), Run("dual", tma=1), Run("fwd", tma=1)))),
    Case("d66_n64", 66, 2, 2, 64, seed=8, weights=False, runs=_std(66, (Run("planes", pitch=72),))),
    Case("d128_n200", 128, 8, 2, 200, seed=9, prior="onehot", runs=_std(128, (
        Run("fwd", col0=1), Run("dual", tma=1), Run("planes", pitch=128, tma=1)))),
    Case("d129_n65", 129, 5, 2, 65, seed=10, runs=_std(129, (
        Run("planes", pitch=160), Run("bf16"), Run("dual", tma=1), Run("possible", tma=1)))),
    Case("d130_n200", 130, 3, 1, 200, seed=11, runs=_std(130, (Run("dual", table_off=1),))),
    Case("d132_n64", 132, 2, 3, 64, seed=12, runs=_std(132, (Run("fwd", col0=2), Run("dual", tma=1)))),
    Case("d256_n65", 256, 4, 2, 65, seed=13, runs=_std(256, (Run("bf16"), Run("dual", tma=1)))),
    Case("d260_n200", 260, 2, 1, 200, seed=14, runs=_std(260, (Run("planes", pitch=288), Run("dual", tma=1)))),
    Case("d400_n64", 400, 2, 2, 64, seed=15, runs=_std(400, (
        Run("bf16"), Run("fwd", col0=1), Run("dual", tma=1), Run("planes", pitch=400)))),
    _dt(1, 63, 3, 16),
    _dt(4, 200, 2, 17),
    _dt(5, 31, 4, 18),
    _dt(8, 5, 12, 19),
    # the first tile's slice runs past the stage through 40 extra in-edges on each of its rows: a middle row straddles
    # slice position EDGE_CAP, later rows lie wholly past it, and the edge at position EDGE_CAP weighs BIG
    Case("hub_d50", 50, 5, 2, 200, seed=20, hub=40, runs=_std(50, (
        Run("dual", tma=1), Run("planes", pitch=64, tma=1), Run("possible", tma=1), Run("bf16")))),
    Case("hub_d200", 200, 2, 2, 200, seed=21, hub=40, runs=(
        Run("fwd"), Run("inv"), Run("dual", pitch=208), Run("planes", pitch=208), Run("planes", pitch=208, tma=1),
        Run("dual", tma=1), Run("possible"))),
)


def launches(case, run):
    """``plan`` of one run with the addresses the test allocates: fresh tensors start on a 256-byte boundary, the
    offsets ``table_off`` / ``csr_off`` move the tables / src and rel by 4 bytes."""
    D, I = case.D, case.I
    seg, w = run.seg(D), run.width(D, I)
    tab = 4 * run.table_off
    csr = 4 * run.csr_off
    common = dict(out_col0=run.col0, ins=0, srcs=(csr, csr), rels=(csr, csr), agg_tma=run.tma)
    if run.kind in SINGLE_KINDS:
        kw = dict(out_bf=0) if run.kind == "bf16" else dict(out=0)
        return plan(D, I, 1, out_row_stride=w, seg_stride_j=seg, tables=(tab,), **kw, **common)
    kw = {}
    if run.kind in ("dual", "both"):
        kw.update(out=0, out_row_stride=w)
    if run.kind in ("planes", "both"):
        kw.update(out_hi=0, out_lo=0, ld_planes=w)
    return plan(D, I, 2, seg_stride_j=2 * seg, seg_stride_dir=seg, tables=(tab, tab), **kw, **common)


def pad_cols(D, pitch):
    """Dw: the plane columns written per segment.  Columns D .. Dw - 1 are zero, Dw .. pitch - 1 are not written."""
    return min(r16(D), max(pitch, D))


# ------------------------------------------------------------------ inputs ----------------------------------------
def make_inputs(case):
    """numpy inputs of a case: facts (heads, rels, tails: global rows), per-fact weights (or None), the two tables
    [R1, D], ins [B, I, D] and the prior [B, N].  Rows are global (b * N + local)."""
    rs = np.random.RandomState(1000 + case.seed)
    B, N, D, I, R1, Nt = case.B, case.N, case.D, case.I, case.R1, case.Nt
    live = rs.rand(Nt) >= case.empty
    live[0] = True                                       # row 0 has facts (hub tile, prior seed)
    heads, tails = [], []
    for b in range(B):
        nodes = b * N + np.flatnonzero(live[b * N:(b + 1) * N])
        if len(nodes) == 0:
            continue
        E = rs.poisson(case.deg * len(nodes))
        heads.append(rs.choice(nodes, E))
        tails.append(rs.choice(nodes, E))
        if case.hub and b == 0:                          # extra in-edges (and out-edges) for the first tile's rows
            rows = nodes[nodes < K_ROWS]
            rows_rep = np.repeat(rows, case.hub)
            other = rs.choice(nodes, len(rows_rep))
            heads += [other, rows_rep]
            tails += [rows_rep, other]
    h = np.concatenate(heads).astype(np.int64)
    t = np.concatenate(tails).astype(np.int64)
    if len(h) % 4 == 0:                                  # F % 4 != 0: the last tile's slice ends off a 4-entry boundary
        h, t = h[:-1], t[:-1]
    F = len(h)
    r = rs.randint(0, R1, size=F).astype(np.int64)
    r[:2] = [0, R1 - 1]
    w = None
    if case.weights or case.hub:
        w = rs.uniform(0.2, 1.5, size=F).astype(np.float32)
        w[rs.rand(F) < 0.1] = 0.0
        if case.hub:
            for dst in (t, h):                           # both directions: the edge at slice position EDGE_CAP
                slot = csr_order(dst, Nt)[csr_rowptr(dst, Nt)[0] + EDGE_CAP]
                w[slot] = BIG
    tables = []
    for _ in range(2):
        tab = rs.randn(R1, D).astype(np.float32)
        tab[1] = np.abs(tab[1])                          # all-non-negative rows
        tab[R1 // 2] = np.abs(tab[R1 // 2])
        tables.append(tab)
    ins = rs.randn(B, I, D).astype(np.float32)
    ins[rs.rand(B, I, D) < 0.1] = 0.0                    # exact zeros among both signs
    if case.prior == "onehot":
        prior = np.zeros((B, N), dtype=np.float32)
        prior[np.arange(B), rs.randint(0, N, size=B)] = 1.0
    else:
        x = rs.randn(B, N)
        prior = (np.exp(x) / np.exp(x).sum(1, keepdims=True)).astype(np.float32)
    return dict(heads=h, rels=r, tails=t, w=w, table_fwd=tables[0], table_inv=tables[1], ins=ins, prior=prior)


def csr_order(dst, Nt):
    """Fact ids in destination-CSR slot order: by destination row, facts of one row in fact order."""
    return np.argsort(dst, kind="stable")


def csr_rowptr(dst, Nt):
    return np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=Nt))])
