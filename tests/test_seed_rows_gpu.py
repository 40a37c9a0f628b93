"""GPU: the row-selected fp32 output of the wgmma GEMM (ops.linear_tc_planes(out_rows=...), gr_linear_tc_planes_rows)
and the ReaRev forward that uses it.

The GEMM with a row predicate must write, on NaN-prefilled outputs, exactly the fp32 rows the predicate flags with the
bits of the launch without it, leave every other fp32 row NaN, and write the planes and the score dots bit for bit as
that launch does.  It runs in the grouped K-order form the D = 200 dense layer uses (staged TMA-store epilogue) and in
the segment-order form at N = 50 (direct stores), with no seed, one, many, a seed in the last partial tile and M not a
multiple of 128.

At model level the ReaRev forward writes fp32 h on the seed rows only in the last layer of every iteration but the
last (where that layer runs as the grouped-order pair), writes no operand planes after the last layer and skips the
last query reform.  pred_dist, loss, pred, the
ranked candidates and ``layer.h_view`` after the forward must equal, bit for bit, a forward whose layers write every
output (the layer without ``h_rows`` / ``next_layer``), eagerly and through GraphedStep."""
import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import ops
from gnn_rag_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
NAN = float("nan")


def _bits(x):
    return x.view(torch.int16 if x.dtype == BF16 else torch.int32)


def _same(a, b):
    """Equal as bit patterns (fp32) or values (integers)."""
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(
        *((_bits(a), _bits(b)) if a.dtype == torch.float32 else (a, b)))


def _gemm_case(layout, M, rs):
    """(planes, W, bias, w_score, launch kwargs) of one GEMM form."""
    if layout == "korder":          # the D = 200 dense layer: grouped K order over the K-order layout, TMA-store epilogue
        D, P, I = 200, 208, 2
        K = (2 * I + 1) * P
        kp = (ops.k_order_nb0(P) + 2 * I * P + 63) // 64 * 64
        kw = dict(k_seg=D, k_seg_pitch=P, k_grouped=True, k_order=True)
    else:                           # N = 50 in segment order: N % 4 != 0 takes the direct-store epilogue
        D, P, I = 50, 64, 2
        K = (2 * I + 1) * P
        kp = K
        kw = dict(k_seg=D, k_seg_pitch=P)
    x = torch.from_numpy(rs.randn(M, kp).astype(np.float32)).to(DEV)
    hi = x.to(BF16)
    lo = (x - hi.float()).to(BF16)
    W = torch.from_numpy((rs.randn(D, (2 * I + 1) * D) / np.sqrt(D)).astype(np.float32)).to(DEV)
    bias = torch.from_numpy((rs.randn(D) * 0.1).astype(np.float32)).to(DEV)
    wsc = torch.from_numpy(rs.randn(D).astype(np.float32)).to(DEV)
    return (hi, lo), K, W, bias, wsc, kw


def _run(planes, K, W, bias, wsc, kw, rows=None):
    M, D = planes[0].shape[0], W.shape[0]
    h = torch.full((M, D), NAN, device=DEV)
    out_planes = tuple(torch.full((M, 256), NAN, dtype=BF16, device=DEV) for _ in range(2))
    dots = torch.full((2 * M,), NAN, device=DEV)
    ops.linear_tc_planes(planes[0], planes[1], K, W, bias, out=h, out_planes=out_planes, w_score=wsc, dots=dots,
                         relu=True, out_rows=rows, **kw)
    return h, out_planes, dots


@pytest.mark.parametrize("layout", ["korder", "segments_n50"])
@pytest.mark.parametrize("M,seeds", [
    (677, "none"),                   # M not a multiple of 128: 5 full tiles and a 37-row one
    (677, "one"),
    (677, "many"),
    (677, "last_tile"),              # seeds in the last, partial tile only (its last row among them)
    (128 * 300 + 64, "many"),        # several tiles per persistent CTA, a half last tile
])
def test_rows_equal_the_unselected_launch_and_nothing_else_is_written(layout, M, seeds):
    rs = np.random.RandomState(M + len(seeds))
    planes, K, W, bias, wsc, kw = _gemm_case(layout, M, rs)
    sel = np.zeros(M, np.float32)
    if seeds == "one":
        sel[rs.randint(M)] = 1.0
    elif seeds == "many":
        idx = rs.choice(M, size=max(3, M // 40), replace=False)
        sel[idx] = rs.choice([1.0, 0.5, 1.0 / 3.0, -2.0], size=idx.size)
        sel[[0, 1, 8, 9, 63, 64, M - 1]] = 1.0       # both rows of a thread, both halves of a tile, the very last row
        sel[2] = -0.0                                # compares equal to zero: not a seed (the reform skips it too)
    elif seeds == "last_tile":
        sel[[M - 1, M - 9, M - 30]] = 1.0
    rows = torch.from_numpy(sel).to(DEV)
    want = _run(planes, K, W, bias, wsc, kw)
    got = _run(planes, K, W, bias, wsc, kw, rows)
    flag = torch.from_numpy(sel != 0).to(DEV)
    assert not torch.isnan(want[0]).any()
    assert torch.equal(_bits(got[0][flag]), _bits(want[0][flag]))
    assert torch.isnan(got[0][~flag]).all()
    for g_, w_ in zip(got[1], want[1]):
        assert torch.equal(_bits(g_), _bits(w_))
    assert torch.equal(_bits(got[2]), _bits(want[2]))


def test_rows_need_an_fp32_output_of_m_rows():
    rs = np.random.RandomState(3)
    planes, K, W, bias, wsc, kw = _gemm_case("korder", 300, rs)
    h = torch.empty(300, 200, device=DEV)
    for rows, out in ((torch.ones(300, device=DEV), None), (torch.ones(299, device=DEV), h),
                      (torch.ones(600, device=DEV)[::2], h), (torch.ones(300, device=DEV, dtype=torch.float64), h)):
        with pytest.raises((ValueError, RuntimeError)):
            ops.linear_tc_planes(planes[0], planes[1], K, W, bias, out=out, w_score=wsc,
                                 out_planes=tuple(torch.empty(300, 256, dtype=BF16, device=DEV) for _ in range(2)),
                                 out_rows=rows, **kw)


# ---- model level -----------------------------------------------------------------------------------------------------

def _full_writes(layer):
    """The layer's forward with every output written: no seed-row h, planes after every layer."""
    forward = layer.forward

    def full(dist, ins, step=0, need_h=True, sparse_prior=False, h_rows=None, next_layer=True):
        return forward(dist, ins, step=step, need_h=need_h, sparse_prior=sparse_prior)
    return full


def _results(model, out, num_entity, eps):
    loss, pred, dist = out[:3]
    db = model.last_batch
    idx, count, total = ops.rank_candidates(dist, db.local_entity, db.query_entities, num_entity, eps)
    ranked = [idx[b, : int(count[b])].tolist() for b in range(idx.shape[0])]
    return dist.clone(), loss.clone(), pred.clone(), ranked, total.clone(), model.reasoning.h_view.clone()


@pytest.mark.parametrize("kind", [
    "pair",          # D = 200: |v|-aggregation + grouped K-order GEMM with the seed rows (the cfg2 path)
    "unfused",       # D = 200 with ops.FUSED_LAYER off: |v|-aggregation + segment-order GEMM, every h row
    "d50",           # D = 50: generic aggregation + segment-order GEMM, every h row
    "fused",         # D = 200 with ops.DENSE_WIDE_AS_PAIR off: the fused layer kernel writes every h row
    "one_layer",     # num_gnn = 1: the last layer of each iteration is the sparse-prior path, which writes everything
])
def test_forward_equals_the_forward_that_writes_every_output(kind, monkeypatch):
    D = 50 if kind == "d50" else 200
    num_gnn = 1 if kind == "one_layer" else 3
    args = S.model_args("ReaRev", entity_dim=D, num_iter=3, num_ins=2, num_gnn=num_gnn, use_cuda=True)
    torch.manual_seed(0)
    model = G.ReaRev(dict(args), 3000, 40, 100).eval()
    with torch.no_grad():
        model.reasoning.score_func.weight.mul_(20.0)
    batch = S.make_batch(11, B=5, N=2000, E=9000, num_entity=3000, num_relation=40, num_word=100, multi_seed=True,
                         test=True)[:7]
    monkeypatch.setattr(ops, "FUSED_MIN_ROWS", 0)
    if kind == "unfused":
        monkeypatch.setattr(ops, "FUSED_LAYER", False)
    if kind == "fused":
        monkeypatch.setattr(ops, "DENSE_WIDE_AS_PAIR", False)
    calls = []
    linear = ops.linear_tc_planes

    def spy(*a, **kw):
        calls.append((kw.get("out_rows") is not None, kw.get("out_planes") is None))
        return linear(*a, **kw)
    monkeypatch.setattr(ops, "linear_tc_planes", spy)
    got = _results(model, model(batch), 3000, args["eps"])
    assert model.reasoning.h32_valid
    # the pair: one seed-row GEMM per iteration but the last
    assert sum(r for r, _ in calls) == (args["num_iter"] - 1 if kind == "pair" else 0)
    if kind in ("pair", "unfused", "d50"):
        assert calls[-1] == (False, True)                                # the last GEMM: full h, no planes
    gs = G.GraphedStep(model, 3000)
    g_out = gs(batch)
    graphed = (g_out.pred_dist.clone(), g_out.loss.clone(), g_out.pred.clone())
    monkeypatch.setattr(model.reasoning, "forward", _full_writes(model.reasoning))
    want = _results(model, model(batch), 3000, args["eps"])
    for a, b in zip(got[:3] + got[4:], want[:3] + want[4:]):
        assert _same(a, b)
    assert got[3] == want[3]                                             # ranked candidates: same ids, same order
    for a, b in zip(graphed, want[:3]):
        assert _same(a, b)
