"""GPU: edges of the aggregation kernel family (csrc/aggregate.cu) against the float64 references of tests/fp64_ref.py:
the TypeLayer mode (gr_type_layer) and the generic message kernel's slow path for tiles whose edge slice overflows
the 1024-entry shared-memory stage, with the NSM ``possible`` output.

Bounds (u = 2^-24): a type-layer element sums n_t + n_h weighted table values in two fp32 chains and adds them:
(n_t + n_h + 1) u of fp64_ref.type_layer_abs.  A message element sums n edges into two chains A, S and forms A - S
with c = w*(w*p): (2n + 8) u of fp64_ref.aggregate_abs.  bf16 planes add 2^-17 of the value (the lo plane's
rounding).  At a hub the bound grows with n, so the edge at slice position 1024 -- the first one the slow path
reads -- carries a dominant coefficient: dropping or repeating it misses by far more than the bound."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import ops

import fp64_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64
HUB = 64               # first row of the second 64-row tile
BIG = 30.0             # weight of the hub's edge at slice position 1024


def _r16(n):
    return (n + 15) // 16 * 16


def _build(rs, B, N, E, R1, hub_edges=0):
    """Random facts inside every question plus a self-loop per node; ``hub_edges`` more facts with tail HUB and as
    many with head HUB (question 0).  Returns numpy facts, the graph and the fact ids at the hub's in-edge position
    1024 in each CSR (tail, head)."""
    h = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
    t = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
    loops = np.arange(B * N)
    h, t = np.concatenate([h, loops]), np.concatenate([t, loops])
    if hub_edges:
        src = rs.randint(0, N, size=hub_edges)
        h = np.concatenate([h, src, np.full(hub_edges, HUB)])
        t = np.concatenate([t, np.full(hub_edges, HUB), src])
    r = rs.randint(0, R1, size=len(h))
    r[:2] = [0, R1 - 1]
    g = ops.csr_build(*(torch.from_numpy(a.astype(np.int64)).to(DEV) for a in (h, r, t)), B, N, R1)
    g.check_status()
    big = None
    if hub_edges:
        big = (np.flatnonzero(t == HUB)[1024], np.flatnonzero(h == HUB)[1024])
        assert int(g.rowptr_t[HUB + 1] - g.rowptr_t[HUB]) > 1024 and int(g.rowptr_h[HUB + 1] - g.rowptr_h[HUB]) > 1024
    return h, r, t, g, big


def _weights(rs, g, F, big=None, zeros=True):
    w = rs.uniform(0.2, 1.5, size=F).astype(np.float32)
    if zeros:
        w[rs.rand(F) < 0.1] = 0.0
    if big is not None:
        w[list(big)] = BIG
    wd = torch.from_numpy(w).to(DEV)
    return wd, ops.gather_f32(wd, g.fact_t), ops.gather_f32(wd, g.fact_h)


def _dev(*arrs):
    return tuple(torch.from_numpy(a.astype(np.int64)).to(DEV) for a in arrs)


@pytest.mark.parametrize("D", [1, 3, 33, 64, 200, 256, 400])
@pytest.mark.parametrize("shape,weights", [("tile", False), ("tile", True), ("small_n", False), ("small_n", True),
                                           ("hub", True)])
def test_type_layer_vs_fp64(D, shape, weights):
    """fp32 output and split-bf16 planes of gr_type_layer.  "small_n": N = 13 < 64, several questions per tile;
    "hub": a row with 1500 in-edges per direction (the tile's stage overflows; slow path)."""
    rs = np.random.RandomState(D + 3 * weights)
    B, N, E = {"tile": (3, 150, 400), "small_n": (10, 13, 30), "hub": (2, 200, 300)}[shape]
    R1 = 29
    h, r, t, g, big = _build(rs, B, N, E, R1, hub_edges=1500 if shape == "hub" else 0)
    F = len(h)
    wd = w_t = w_h = None
    if weights:
        wd, w_t, w_h = _weights(rs, g, F, big)
    table = torch.from_numpy(rs.randn(R1, D).astype(np.float32)).to(DEV)
    if shape == "hub":                                            # the planted edge's relation row is not tiny
        rb = int(r[big[0]])
        table[rb] = torch.where(table[rb] < 0, -1.0, 1.0) * table[rb].abs().clamp_min(0.5)
    Nt = B * N
    out = torch.full((Nt, D), -9.0, device=DEV)
    P = _r16(D) + 16
    hi = torch.full((Nt, P), 3.0, dtype=torch.bfloat16, device=DEV)
    lo = torch.full((Nt, P), 3.0, dtype=torch.bfloat16, device=DEV)
    ops.type_layer(g, table, out, w_t, w_h, planes=(hi, lo))
    facts = _dev(h, r, t)
    w64 = None if wd is None else wd.to(F64)
    want = R.type_layer(table.to(F64), *facts, w64, Nt)
    scale = R.type_layer_abs(table.to(F64), *facts, w64, Nt)
    n = torch.from_numpy(np.bincount(t, minlength=Nt) + np.bincount(h, minlength=Nt)).to(DEV, F64)[:, None]
    bound = (n + 1) * U * scale + 1e-35
    err = (out.to(F64) - want).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    assert (want == 0).any() and (want > 0).any()
    if shape == "hub":
        assert (BIG * table[r[big[0]]].abs().to(F64) > 10 * bound[HUB]).any()   # one planted edge is far outside
    hi_want = out.to(torch.bfloat16)
    assert torch.equal(hi[:, :D].view(torch.int16), hi_want.view(torch.int16))
    assert torch.equal(lo[:, :D].view(torch.int16), (out - hi_want.float()).to(torch.bfloat16).view(torch.int16))
    assert (hi[:, D:_r16(D)] == 0).all() and (lo[:, D:_r16(D)] == 0).all()   # padding to 16 columns is zeroed
    assert (hi[:, _r16(D):] == 3.0).all() and (lo[:, _r16(D):] == 3.0).all()


def test_type_layer_without_facts():
    """F = 0: every row is relu(0) = 0 in both outputs."""
    g = ops.csr_build(*(torch.zeros(0, dtype=torch.int64, device=DEV) for _ in range(3)), 3, 70, 5)
    table = torch.randn(5, 33, device=DEV)
    out = torch.full((210, 33), -9.0, device=DEV)
    hi = torch.full((210, 48), 3.0, dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    ops.type_layer(g, table, out, planes=(hi, lo))
    assert (out == 0).all() and (hi == 0).all() and (lo == 0).all()


@pytest.mark.parametrize("tma", [0, 1])
@pytest.mark.parametrize("D,I", [(33, 1), (64, 2), (200, 3), (256, 5)])
def test_generic_aggregate_hub_tile_vs_fp64(tma, D, I):
    """gr_aggregate (each direction) and gr_aggregate_dual (fp32 and planes) at a hub tile beyond the 1024-edge
    stage, with the staged loads (agg_tma 0) and the bulk-TMA loads (agg_tma 1)."""
    rs = np.random.RandomState(D + I + 100 * tma)
    B, N, R1 = 2, 200, 31
    h, r, t, g, big = _build(rs, B, N, 300, R1, hub_edges=1500)
    wd, w_t, w_h = _weights(rs, g, len(h), big)
    f = lambda *s: torch.from_numpy(rs.randn(*s).astype(np.float32)).to(DEV)   # noqa: E731
    tf, ti, ins = f(R1, D), f(R1, D), f(B, I, D)
    prior = torch.softmax(f(B, N), 1)
    facts = _dev(h, r, t)
    Nt = B * N
    ops.set_option("agg_tma", tma)
    try:
        singles = [ops.aggregate(g, d, prior, tab, ins, w=ww) for d, tab, ww in (("fwd", tf, w_t), ("inv", ti, w_h))]
        dual = torch.full((Nt, 2 * I * D), -9.0, device=DEV)
        ops.aggregate_dual(g, prior, tf, ti, ins, dual, 0, w_t, w_h)
        P = _r16(D)
        hi = torch.full((Nt, 2 * I * P), 3.0, dtype=torch.bfloat16, device=DEV)
        lo = hi.clone()
        ops.aggregate_dual(g, prior, tf, ti, ins, None, 0, w_t, w_h, planes=(hi, lo), seg_pitch=P)
    finally:
        ops.set_option("agg_tma", 0)
    w64 = wd.to(F64)
    for d, (tab, got, deg) in enumerate(((tf, singles[0], t), (ti, singles[1], h))):
        direction = ("fwd", "inv")[d]
        want = R.aggregate(tab.to(F64), ins.to(F64), prior.to(F64), *facts, w64, direction)
        scale = R.aggregate_abs(tab.to(F64), ins.to(F64), prior.to(F64), *facts, w64, direction)
        n = torch.from_numpy(np.bincount(deg, minlength=Nt)).to(DEV, F64)[:, None]
        bound = (2 * n + 8) * U * scale + 1e-35
        fb = big[d]
        src = (h, t)[d][fb]
        planted = BIG * BIG * prior.view(-1)[src].to(F64) * torch.relu(tab[r[fb]].to(F64) * ins[0].to(F64)).view(-1)
        assert (planted > 100 * bound[HUB]).any()                 # one slow-path edge is far outside the bound
        for got_k in (got, dual.view(Nt, I, 2, D)[:, :, d].reshape(Nt, I * D)):
            err = (got_k.to(F64) - want).abs()
            assert (err <= bound).all(), (direction, (err / bound).max().item())
        pl = (hi.to(F64) + lo.to(F64)).view(Nt, I, 2, P)[:, :, d, :D].reshape(Nt, I * D)
        assert ((pl - want).abs() <= bound + 2.0 ** -17 * want.abs()).all()
        assert (hi.view(Nt, I, 2, P)[:, :, d, D:] == 0).all()


def test_possible_mask_around_the_threshold_and_beyond_the_stage():
    """The NSM ``possible`` output of gr_aggregate: 1 where the prior mass over a row's in-edges exceeds 1e-10.
    Rows fed by 1.1e-10 / 0.9e-10 sit just above / below; the hub row's only mass arrives on the edge at slice
    position 1024, read by the slow path."""
    rs = np.random.RandomState(7)
    B, N, R1, D = 1, 300, 11, 40
    hub_src = rs.randint(50, 300, size=1500)                  # zero-prior sources
    hub_src[1024] = 3
    h = np.concatenate([[1, 2, 4, 4], hub_src, np.arange(N)])
    t = np.concatenate([[10, 11, 12, 13], np.full(1500, HUB), np.arange(N)])
    r = rs.randint(0, R1, size=len(h))
    g = ops.csr_build(*_dev(h, r, t), B, N, R1)
    p = np.zeros((B, N), dtype=np.float32)
    p[0, 1], p[0, 2], p[0, 3], p[0, 4] = 1.1e-10, 0.9e-10, 2e-10, 0.5
    prior = torch.from_numpy(p).to(DEV)
    table = torch.randn(R1, D, device=DEV)
    ins = torch.randn(B, 1, D, device=DEV)
    possible = torch.full((B * N,), -1.0, device=DEV)
    for tma in (0, 1):
        ops.set_option("agg_tma", tma)
        try:
            out = ops.aggregate(g, "fwd", prior, table, ins, possible=possible)
        finally:
            ops.set_option("agg_tma", 0)
        want, mass = R.possible(prior.to(F64), _dev(h, r, t), None, B * N)
        assert torch.equal(possible.to(F64), want)
        assert possible[10] == 1 and possible[11] == 0 and possible[HUB] == 1 and possible[12] == 1
        agg = R.aggregate(table.to(F64), ins.to(F64), prior.to(F64), *_dev(h, r, t), None, "fwd")
        sc = R.aggregate_abs(table.to(F64), ins.to(F64), prior.to(F64), *_dev(h, r, t), None, "fwd")
        n = torch.from_numpy(np.bincount(t, minlength=B * N)).to(DEV, F64)[:, None]
        assert ((out.to(F64) - agg).abs() <= (2 * n + 8) * U * sc + 1e-45).all()
        assert (agg[HUB] != 0).any()
