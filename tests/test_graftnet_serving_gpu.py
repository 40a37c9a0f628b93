"""GraftNet served like ReaRev: ``gr_graft_stage`` with live counts over fixed-capacity lists, ``GraphedStep`` on the
graft tuple (bit-equal to eager ``model(batch)`` + ``evaluate.retrieve``: goldens, synthetic D = 50 / 200, capacity
buckets with stale tails, alternating shapes, the submit/collect pipeline, refusal of malformed graft lists) and the
question shards of ``parallel.shard_graft_batch``."""
import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import batching, evaluate, graphed, ops, parallel, synthetic as S
from test_graftnet_host import CASES, NUM_ENTITY, load_model

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
NE, NR, NW = 5000, 60, 200
REJECTED_MSG = "graft fact lists rejected"


# ---- gr_graft_stage with live counts -------------------------------------------------------------------------------

def _lists(rs, B, N, maxF, per_q):
    """Paired graft lists (loader layout: tail list permuted within each question)."""
    hb, hf, he, tb, te, tf = ([] for _ in range(6))
    for b in range(B):
        slots = rs.permutation(maxF)[:per_q[b]]
        heads, tails = rs.randint(0, N, len(slots)), rs.randint(0, N, len(slots))
        perm = rs.permutation(len(slots))
        hb += [b] * len(slots); hf += list(slots); he += list(heads)
        tb += [b] * len(slots); te += list(tails[perm]); tf += list(slots[perm])
    return [np.asarray(x, dtype=np.int64) for x in (hb, hf, he)], [np.asarray(x, dtype=np.int64) for x in (tb, te, tf)]


def _stage(e2f, f2e, kfr, B, N, R1, live=None):
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.int64), device=dev)  # noqa: E731
    lv = None if live is None else torch.tensor(live, dtype=torch.int32, device=dev)
    gg = ops.graft_stage([t(a) for a in e2f], [t(a) for a in f2e], t(kfr), B, N, R1, live=lv)
    torch.cuda.synchronize()
    n = int(gg.nfacts.item())
    return dict(n=n, status=int(gg.status.item()), csr=int(gg.graph.status.item()),
                **{k: getattr(gg, k)[:n].cpu().numpy() for k in ("heads", "rels", "tails", "slot_of")})


def _with_tail(live_lists, stale_lists, bad, cap):
    """live prefix + a stale tail (entries of another batch that look valid, then out-of-range ids) up to ``cap``."""
    out = []
    for a, s, x in zip(live_lists, stale_lists, bad):
        buf = np.concatenate([a, s, np.full(cap, x, dtype=np.int64)])[:cap]
        assert len(buf) == cap
        out.append(buf)
    return out


@pytest.mark.parametrize("case", ["some", "zero", "full", "tail_longer", "unpaired"])
def test_graft_stage_live_counts_ignore_stale_tail(case):
    rs = np.random.RandomState(7)
    B, N, maxF, R1 = 3, 17, 40, 9
    kfr = rs.randint(0, R1, size=(B, maxF))
    e2f, f2e = _lists(rs, B, N, maxF, [25, 0, 14])
    st_e2f, st_f2e = _lists(np.random.RandomState(8), B, N, maxF, [30, 20, 30])     # an earlier batch
    n0 = n1 = len(e2f[0])
    if case == "zero":
        n0 = n1 = 0
    elif case == "tail_longer":
        # the tail list has one more live entry than the head list: its slot's head sits in the head list's stale
        # tail, so pairing it there would hide the unpaired slot
        n0 = len(e2f[0]) - 1
    elif case == "unpaired":
        f2e = [a[:-1] for a in f2e]
        n1 = len(f2e[0])
    cap = graphed.fact_capacity(max(n0, n1) + 1) if case != "full" else max(n0, n1)
    bad_e2f, bad_f2e = (B + 3, maxF + 5, -4), (-1, N + 9, maxF * 2)
    E = _with_tail([a[:n0] for a in e2f], st_e2f, bad_e2f, cap)
    F = _with_tail([a[:n1] for a in f2e], st_f2e, bad_f2e, cap)
    if case == "tail_longer":
        E[0][n0], E[1][n0], E[2][n0] = e2f[0][n0], e2f[1][n0], e2f[2][n0]          # the missing head, in the stale tail
    got = _stage(E, F, kfr, B, N, R1, live=[n0, n1])
    want = _stage([a[:n0] for a in e2f], [a[:n1] for a in f2e], kfr, B, N, R1)
    for k in ("n", "status", "csr", "heads", "rels", "tails", "slot_of"):
        assert np.array_equal(got[k], want[k]), k
    expect_status = 8 if case in ("tail_longer", "unpaired") else 0
    assert got["status"] == expect_status and got["csr"] == 0
    if case == "zero":
        assert got["n"] == 0
    if case in ("some", "full"):
        assert got["n"] == n0


# ---- GraphedStep on the graft tuple --------------------------------------------------------------------------------

def _eager(m, batch, eps):
    loss, pred, dist, _ = m(batch)
    ret, _ = evaluate.retrieve(dist, m.last_batch, m.num_entity, eps)
    return dist.clone(), float(loss), pred.clone(), [(r.ent.tolist(), r.prob.tolist()) for r in ret]


def _graphed(gs, batch):
    out = gs(batch)
    ret, _ = gs.retrieve(out)
    return out.pred_dist.clone(), float(out.loss), out.pred.clone(), [(r.ent.tolist(), r.prob.tolist()) for r in ret]


def _assert_same(a, b):
    assert torch.equal(a[0], b[0])
    assert a[1] == b[1] or (np.isnan(a[1]) and np.isnan(b[1]))
    assert torch.equal(a[2], b[2])
    assert a[3] == b[3]


@pytest.mark.parametrize("name", CASES)
def test_graphed_equals_eager_on_goldens(name):
    m, g = load_model(name, "cuda")
    m = m.cuda()
    gs = G.GraphedStep(m, NUM_ENTITY)
    eps = g.args["eps"]
    got = _graphed(gs, g.batch)
    want = _eager(m, g.batch, eps)
    if g.args.get("lm", "lstm") == "lstm":
        _assert_same(got, want)
    else:
        # With the transformer encoder and relation-text pooling (torch ops this case adds to the step), graph replay
        # and eager differ in the last bits of pred_dist; which op makes the difference is not pinned down yet.  The
        # LSTM goldens and the synthetic cases are bit-identical.
        rel = float(((got[0] - want[0]).abs() / want[0].abs().max(dim=1, keepdim=True)[0].clamp_min(1e-30)).max())
        assert rel <= 1e-5, rel                            # measured: up to 2.4e-6
        assert [e for e, _ in got[3]] == [e for e, _ in want[3]]
    _assert_same(_graphed(gs, g.batch), got)               # a second replay of the same graph


def _model(D, layers=3, sharpen=None, **over):
    args = S.model_args("GraftNet", entity_dim=D, num_layer=layers, word_dim=64, use_cuda=True, **over)
    torch.manual_seed(D + layers)
    m = G.GraftNet(dict(args), NE, NR, NW).cuda().eval()
    if sharpen:
        with torch.no_grad():
            m.reasoning.score_func.weight.mul_(sharpen)
    return m, args


def _batch(seed, B, N, E, max_fact=None, **kw):
    b = S.make_graft_batch(seed, B, N, E, num_entity=NE, num_relation=NR, num_word=NW, **kw)
    if max_fact is not None:      # a real loader's max_facts is one constant of the dataset: pad with the pad relation
        kfr = b[5]
        assert kfr.shape[1] <= max_fact
        wide = np.full((kfr.shape[0], max_fact), NR, dtype=np.int64)
        wide[:, :kfr.shape[1]] = kfr
        b = b[:5] + (wide,) + b[6:]
    return b


@pytest.mark.parametrize("D,over,bkw", [
    (50, {}, dict(with_weights=False)),
    (200, {}, dict(with_weights=False, fact_dropout=0.2)),
    (50, dict(norm_rel=True), dict(with_weights=True)),
    (200, dict(use_inverse_relation=True, norm_rel=True), dict(with_weights=True, use_inverse_relation=True)),
])
def test_graphed_equals_eager_synthetic(D, over, bkw):
    m, args = _model(D, **over)
    assert m.encode_type
    gs = G.GraphedStep(m, NE)
    for seed in (3, 4):
        b = _batch(seed, 8, 300, 900, test=True, **bkw)
        _assert_same(_graphed(gs, b), _eager(m, b, args["eps"]))


def test_graphed_buckets_stale_tails_and_lru():
    m, args = _model(50)
    gs = G.GraphedStep(m, NE, max_graphs=2)
    B, N, MF = 6, 250, 3000
    # graft and kb counts of these batches fall into one capacity bucket each: one graph; the smaller batch right after
    # the larger one leaves a stale tail in every fact buffer
    batches = [_batch(s, B, N, E, max_fact=MF, with_weights=False) for s, E in ((51, 700), (52, 760), (53, 720))]
    keys = {(graphed.fact_capacity(len(b[2][0])), graphed.fact_capacity(len(b[3][0][0]))) for b in batches}
    assert len(keys) == 1
    assert len(batches[1][3][0][0]) > len(batches[2][3][0][0]) and len(batches[1][2][0]) > len(batches[2][2][0])
    entries = []
    for b in batches:
        _assert_same(_graphed(gs, b), _eager(m, b, args["eps"]))
        entries.append(next(reversed(gs._cache.values())))
    assert len(gs._cache) == 1 and entries[0] is entries[1] is entries[2]
    # other buckets: the LRU is held to max_graphs and every result still equals eager
    for s, E in ((54, 1000), (55, 1200), (56, 760)):
        b = _batch(s, B, N, E, max_fact=MF, with_weights=False)
        _assert_same(_graphed(gs, b), _eager(m, b, args["eps"]))
        assert len(gs._cache) <= 2


@pytest.mark.parametrize("max_graphs", [8, 1])
def test_graphed_alternating_shapes(max_graphs):
    """(B, N) = (4, 300), (6, 200), (5, 300), then the first two again: every graph's operand planes stay owned by its
    cache entry after the layers' plane cache moved on to another B*N ((4, 300) and (6, 200) share one)."""
    m, args = _model(50)
    gs = G.GraphedStep(m, NE, max_graphs=max_graphs)
    shapes = [(4, 300, 900, 61), (6, 200, 600, 62), (5, 300, 900, 63), (4, 300, 900, 64), (6, 200, 600, 65),
              (4, 300, 900, 61)]
    for B, N, E, seed in shapes:
        b = _batch(seed, B, N, E, max_fact=2500, with_weights=False)
        got = _graphed(gs, b)
        _assert_same(got, _eager(m, b, args["eps"]))
        assert len(gs._cache) <= max_graphs


@pytest.mark.parametrize("pinned", [False, True])
def test_graphed_pipeline_matches_sync(pinned):
    m, args = _model(50)
    gs = G.GraphedStep(m, NE)
    batches = [_batch(s, 8, 300, E, max_fact=2500, with_weights=False) for s, E in
               ((71, 900), (72, 850), (73, 950), (74, 600), (75, 900))]
    if pinned:
        batches = [batching.pin_graft_batch(b) for b in batches]
    want = []
    for b in batches:
        out = gs(b)
        ret, _ = gs.retrieve(out)
        want.append(([r.ent.tolist() for r in ret], [r.prob.tolist() for r in ret], float(out.loss),
                     out.pred.tolist()))
    got, prev = [], None
    for b in batches:
        t = gs.submit(b)
        if prev is not None:
            got.append(gs.collect(prev))       # one step late: two tickets in flight
        prev = t
    got.append(gs.collect(prev))
    for (ents, probs, loss, pred), (ret, nbytes, gl, gp) in zip(want, got):
        assert [r.ent.tolist() for r in ret] == ents
        assert [r.prob.tolist() for r in ret] == probs
        assert gl == loss and gp.tolist() == pred
        assert nbytes > 0


@pytest.mark.parametrize("bad", ["duplicate_slot", "unpaired_slot", "head_outside"])
def test_graphed_refuses_malformed_graft_lists(bad):
    m, args = _model(50, layers=2)
    gs = G.GraphedStep(m, NE)
    B, N = 4, 200
    good = _batch(81, B, N, 600, max_fact=1500, with_weights=False)
    b = list(_batch(81, B, N, 600, max_fact=1500, with_weights=False))
    (hb, hf, he, hv), (tb, te, tf, tv) = b[3]
    hf, he = hf.copy(), he.copy()
    assert hb[0] == hb[1]
    if bad == "duplicate_slot":
        hf[1] = hf[0]
    elif bad == "unpaired_slot":
        tb, te, tf, tv = tb[:-1], te[:-1], tf[:-1], tv[:-1]
    else:
        he[0] = N + 5
    b[3] = ((hb, hf, he, hv), (tb, te, tf, tv))
    b = tuple(b)
    with pytest.raises(RuntimeError, match=REJECTED_MSG):
        gs.retrieve(gs(b))
    with pytest.raises(RuntimeError, match=REJECTED_MSG):
        gs(b, check=True)
    with pytest.raises(RuntimeError, match=REJECTED_MSG):
        gs.collect(gs.submit(b))
    with pytest.raises(RuntimeError, match=REJECTED_MSG):
        m(b)                                   # the eager forward raises the same way
    _assert_same(_graphed(gs, good), _eager(m, good, args["eps"]))     # and the step is usable afterwards


# ---- question shards -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3])
def test_shards_on_one_gpu_match_full_batch(world):
    for sharpen in (None, 20.0):
        m, args = _model(50, sharpen=sharpen)
        b = _batch(91, 7, 300, 900, with_weights=False, fact_dropout=0.1, test=True)
        full, _l, _p, full_lists = _eager(m, b, args["eps"])
        parts, lists = [], []
        for r in range(world):
            sb = parallel.shard_graft_batch(b, r, world)
            d, _l, _p, li = _eager(m, sb, args["eps"])
            parts.append(d)
            lists += li
        got = torch.cat(parts)
        # the torch question-encoder GEMM may pick other kernels at another B: not bit-equal, within 1e-5
        rel = float(((got - full).abs() / full.abs().max(dim=1, keepdim=True)[0].clamp_min(1e-30)).max())
        assert rel <= 1e-5, rel
        if sharpen:
            assert [e for e, _ in lists] == [e for e, _ in full_lists]
