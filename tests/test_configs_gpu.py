"""GPU: the other BASELINE configurations (size-independent properties + kernel-level parity at full size) and the
`.info` wire format the LLM stage consumes."""
import json
import os

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import batching, evaluate, graphed, ops, synthetic as S
from oracle import kgqa_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))


def _model(c, model="ReaRev", **kw):
    args = S.model_args(model, entity_dim=c["D"], num_iter=c["T"], num_ins=c["I"], num_gnn=c["K"], num_step=c["K"],
                        use_cuda=True, **kw)
    torch.manual_seed(0)
    cls = G.NSM if model == "NSM" else G.ReaRev
    return cls(dict(args), S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_RELATION, S.WEBQSP_NUM_WORD).eval(), args


def test_cfg5_stress_graph_aggregate_parity_and_forward_properties():
    """cfg5: 100k-node / 1M-edge subgraph, 400-dim features (generic runtime-D kernel, two column passes, hub rows
    beyond the smem edge staging, fp32 SIMT linear because D > 256)."""
    c = S.CONFIGS["cfg5"]
    b = S.make_batch(3, B=1, N=c["N"], E=c["E"], powerlaw=True, with_weights=False)
    db = batching.stage_batch(b, torch.device(DEV), S.WEBQSP_NUM_RELATION + 1)
    db.graph.check_status()
    rs = np.random.RandomState(0)
    D = c["D"]
    table = torch.from_numpy(rs.randn(S.WEBQSP_NUM_RELATION + 1, D).astype(np.float32))
    ins = torch.from_numpy(rs.randn(1, 1, D).astype(np.float32))
    prior = torch.softmax(torch.from_numpy(rs.randn(1, c["N"]).astype(np.float32)), 1)
    got = ops.aggregate(db.graph, "fwd", prior.to(DEV), table.to(DEV), ins.to(DEV)).cpu()
    mats = O.FactMats(b[2], 1, c["N"], False)
    want = O.reason_layer(mats, prior, ins[:, 0, :], table, torch.eye(D), None, False)
    assert (got - want).abs().max().item() <= 5e-5 * (want.abs().max().item() + 1e-12)
    m, args = _model(c)
    _, _, d1, _ = m(b)
    _, _, d2, _ = m(b)
    assert torch.equal(d1, d2)                                        # deterministic at stress size
    assert abs(float(d1.sum()) - 1.0) < 1e-4 and (d1 >= 0).all()
    ret, _ = evaluate.retrieve(d1, m.last_batch, S.WEBQSP_NUM_ENTITY, args["eps"])
    assert len(ret) == 1 and len(ret[0]) > 0


def test_cfg3_cwq_shape_forward_properties():
    """cfg3 shape (10k nodes, 40k edges, 4 hops, 3 instructions) at B=8: split-bf16 planes with 7 segments,
    the NI=3 aggregation instance, GEMM K = 7*208."""
    c = dict(S.CONFIGS["cfg3"], B=8)
    m, args = _model(c)
    b = S.make_batch(5, B=c["B"], N=c["N"], E=c["E"], n_real=9000, with_weights=False, multi_seed=True)
    _, _, d1, _ = m(b)
    _, _, d2, _ = m(b)
    assert torch.equal(d1, d2)
    assert torch.allclose(d1.sum(1), torch.ones(c["B"], device=DEV), atol=1e-4)
    assert (d1[:, 9000:] == 0).all()
    # and against the CPU oracle on the first two questions (block-diagonal independence)
    from gnn_rag_b200 import parallel
    small = parallel.shard_batch(b, 0, 4)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    _, _, want = O.forward(sd, args, S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_WORD, small)
    _, _, got, _ = m(small)
    err = ((got.cpu() - want).abs() / want.clamp_min(1e-30)).max().item()
    assert err < 1e-3, err


def test_nsm_webqsp_shape_vs_oracle_and_reason_kb():
    c = dict(S.CONFIGS["cfg2"], B=4)
    m, args = _model(c, "NSM", reason_kb=True)
    b = S.make_batch(9, B=4, N=c["N"], E=c["E"], with_weights=False)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    _, _, want = O.forward(sd, args, S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_WORD, b)
    _, _, got, _ = m(b)
    nz = want > 0
    assert ((got.cpu() > 0) == nz).all()                              # possible_tail mask identical
    assert ((got.cpu() - want).abs()[nz] / want[nz]).max().item() < 1e-3


class _FakeLoader:
    """SingleDataLoader's batching contract (gnn/dataset_load.py:599-629, 130-141): ``get_batch`` slices
    ``self.batches[start:end]`` into ``self.sample_ids``; ``get_quest`` decodes ONLY those and does not exist as a
    usable call before the first ``get_batch`` (no ``sample_ids`` attribute yet)."""

    def __init__(self, B, N, E, num_data):
        self.num_data = num_data
        self.max_local_entity = N
        self.data = S.make_batch(20, B=num_data, N=N, E=E, num_entity=500, num_relation=30, num_word=60,
                                 test=True, with_weights=False)
        self.N = N
        self.batches = np.arange(num_data)

    def reset_batches(self, is_sequential=True):
        self.batches = np.arange(self.num_data)

    def get_quest(self):
        return ["question %d " % i for i in self.sample_ids]      # AttributeError before the first get_batch

    def get_batch(self, iteration, batch_size, fact_dropout, q_type=None, test=False):
        start, end = batch_size * iteration, min(batch_size * (iteration + 1), self.num_data)
        ids = self.batches[start:end]
        self.sample_ids = ids
        le, qe, kb, qi, sd, _, ad, al = self.data
        heads, rels, tails, bids = kb[0], kb[1], kb[2], kb[3]
        sel = np.isin(bids, ids)
        remap = -np.ones(self.num_data, dtype=np.int64)
        remap[ids] = np.arange(len(ids))
        nb = remap[bids[sel]]
        h = heads[sel] - bids[sel] * self.N + nb * self.N
        t = tails[sel] - bids[sel] * self.N + nb * self.N
        kb2 = (h, rels[sel], t, nb, np.arange(len(h)), None, None)
        out = (le[ids], qe[ids], kb2, qi[ids], sd[ids], None, ad[ids])
        return out + (al[ids],) if test else out


def test_info_jsonl_matches_shipped_schema(tmp_path):
    """Rows written by Evaluator.evaluate(write_info=True) parse exactly like the reference's shipped
    llm/results/gnn/*/test.info (first 3 rows kept in tests/golden/test_info_sample.jsonl)."""
    sample = [json.loads(l) for l in open(os.path.join(HERE, "golden", "test_info_sample.jsonl"))]
    args = S.model_args("ReaRev", entity_dim=32, num_iter=3, num_ins=2, num_gnn=2, word_dim=16, use_cuda=True,
                        checkpoint_dir=str(tmp_path) + "/", experiment_name="t")
    torch.manual_seed(0)
    m = G.ReaRev(dict(args), 500, 30, 60).eval()
    with torch.no_grad():
        m.reasoning.score_func.weight.mul_(30.0)
    entity2id = {"m.%04d" % i: i for i in range(500)}
    ev = G.Evaluator(args, m, entity2id, {}, torch.device(DEV))
    loader = _FakeLoader(B=4, N=64, E=200, num_data=10)          # 10 questions, batches of 4: 4 + 4 + 2
    f1, h1, em = ev.evaluate(loader, test_batch_size=4, write_info=True)
    rows = [json.loads(l) for l in open(os.path.join(str(tmp_path), "t_test.info"))]
    assert len(rows) == 10 and 0.0 <= f1 <= 1.0
    assert [r["question"] for r in rows] == ["question %d " % i for i in range(10)]   # per-batch get_quest, in order
    for r in rows:
        assert list(r.keys()) == list(sample[0].keys())               # same keys, same order
        for k, v in sample[0].items():
            assert type(r[k]) is type(v), k
        assert all(isinstance(c[0], str) and isinstance(c[1], float) for c in r["cand"])
        probs = [c[1] for c in r["cand"]]
        assert probs == sorted(probs, reverse=True)
    # metrics agree with the reference's formula (oracle f1_and_hits) on the same retrieved lists
    b = loader.get_batch(0, 4, 0.0, test=True)
    _, _, dist, _ = m(b[:-1])
    ret, _ = evaluate.retrieve(dist, m.last_batch, 500, args["eps"])
    for q in range(4):
        ids = ret[q].ent.tolist()
        p, r_, f, h, e, _ = evaluate.f1_and_hits(list(b[-1][q]), ids)
        assert (p, r_, f, h) == O.f1_and_hits(list(b[-1][q]), ids, ids[0] if ids else -1)


def test_graphed_step_matches_eager():
    """CUDA-graph replay of (CSR batching + forward + ranking) == eager path, bit for bit, across batches."""
    c = dict(S.CONFIGS["cfg2"], B=8, N=500, E=1500)
    m, args = _model(c)
    gs = G.GraphedStep(m, S.WEBQSP_NUM_ENTITY)
    for seed in (11, 12, 13):
        b = S.make_batch(seed, B=c["B"], N=c["N"], E=c["E"], with_weights=False)
        out = gs(b)
        ret_g, _ = gs.retrieve(out)
        dist_g = out.pred_dist.clone()
        loss, pred, dist, _ = m(b)
        ret_e, _ = evaluate.retrieve(dist, m.last_batch, S.WEBQSP_NUM_ENTITY, args["eps"])
        assert torch.equal(dist_g, dist)
        assert float(out.loss) == float(loss)
        assert [r.ent.tolist() for r in ret_g] == [r.ent.tolist() for r in ret_e]


def test_graphed_step_buckets_fact_counts_and_evicts():
    """Real ``get_batch`` output has a different fact count almost every batch: batches whose counts fall into one
    capacity bucket replay ONE captured graph (facts in front, device-side live count) and still equal the eager
    path bit for bit; the cache is an LRU of ``max_graphs`` entries; ids outside the batch are reported."""
    c = dict(S.CONFIGS["cfg2"], B=6, N=400, E=1300)
    m, args = _model(c)
    gs = G.GraphedStep(m, S.WEBQSP_NUM_ENTITY, max_graphs=2)
    caps = set()
    for seed, E in ((31, 1300), (32, 1250), (33, 1350), (34, 700), (35, 2600), (36, 1300)):
        b = S.make_batch(seed, B=c["B"], N=c["N"], E=E, with_weights=False)
        F = len(b[2][0])
        caps.add(graphed.fact_capacity(F))
        assert graphed.fact_capacity(F) >= F and graphed.fact_capacity(F) <= 1.13 * F + 1024
        out = gs(b)
        dist_g = out.pred_dist.clone()
        ret_g, _ = gs.retrieve(out)
        _, _, dist, _ = m(b)
        ret_e, _ = evaluate.retrieve(dist, m.last_batch, S.WEBQSP_NUM_ENTITY, args["eps"])
        assert torch.equal(dist_g, dist)
        assert [r.ent.tolist() for r in ret_g] == [r.ent.tolist() for r in ret_e]
        assert len(gs._cache) <= 2
    assert len(caps) >= 3                                         # several buckets were exercised -> evictions
    bad = S.make_batch(37, B=c["B"], N=c["N"], E=1300, with_weights=False)
    bad[2][0][5] = c["B"] * c["N"] + 3                           # a head id outside the batch
    with pytest.raises(RuntimeError, match="outside the batch"):
        gs.retrieve(gs(bad))


def test_graphed_step_with_edge_weights():
    """normalized_gnn / norm_rel weight lists ride along in the captured step (fixed-capacity buffers)."""
    args = S.model_args("ReaRev", entity_dim=200, num_iter=2, num_ins=2, num_gnn=2, use_cuda=True,
                        normalized_gnn=True, norm_rel=True)
    torch.manual_seed(0)
    m = G.ReaRev(dict(args), 3000, 40, 100).eval()
    gs = G.GraphedStep(m, 3000)
    for seed in (41, 42):
        b = S.make_batch(seed, B=4, N=128, E=500 + 10 * seed, num_entity=3000, num_relation=40, num_word=100)
        out = gs(b)
        dist_g = out.pred_dist.clone()
        _, _, dist, _ = m(b)
        assert torch.equal(dist_g, dist)


def test_graphed_pipeline_submit_collect_matches_sync():
    """Two-deep submit/collect pipeline (copy-stream H2D/D2H overlapped with the graph) returns exactly what the
    synchronous graphed call returns, batch by batch, also when tickets are collected one step late."""
    c = dict(S.CONFIGS["cfg2"], B=8, N=500, E=1500)
    m, args = _model(c)
    gs = G.GraphedStep(m, S.WEBQSP_NUM_ENTITY)
    batches = [S.make_batch(seed, B=c["B"], N=c["N"], E=c["E"], with_weights=False) for seed in (21, 22, 23, 24, 25)]
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
            got.append(gs.collect(prev))
        prev = t
    got.append(gs.collect(prev))
    for (ents, probs, loss, pred), (ret, nbytes, gl, gp) in zip(want, got):
        assert [r.ent.tolist() for r in ret] == ents
        assert [r.prob.tolist() for r in ret] == probs
        assert gl == loss and gp.tolist() == pred
        assert nbytes > 0


@pytest.mark.parametrize("kw", [dict(), dict(multi_seed=True, powerlaw=True), dict(n_real="ragged")])
def test_sparse_prior_fastpath_matches_dense_path(kw):
    """First layer of every iteration: K=1-segment GEMM + frontier fix-up == full aggregation + full GEMM."""
    c = dict(S.CONFIGS["cfg2"], B=6, N=700, E=2400)
    m, args = _model(c)
    with torch.no_grad():
        m.reasoning.score_func.weight.mul_(20.0)
    b = S.make_batch(31, B=c["B"], N=c["N"], E=c["E"], with_weights=False, **kw)
    outs = {}
    for flag in (True, False):
        ops.SPARSE_PRIOR_FASTPATH = flag
        try:
            _, _, d, _ = m(b)
            outs[flag] = (d.clone(), torch.stack(m.dist_history[1:]).clone(), m.reasoning.h_view.clone(),
                          int(m.reasoning.fr_count.item()))
        finally:
            ops.SPARSE_PRIOR_FASTPATH = True
    rel = ((outs[True][0] - outs[False][0]).abs() / outs[False][0].clamp_min(1e-30)).max().item()
    assert rel < 1e-4, rel
    assert (outs[True][2] - outs[False][2]).abs().max().item() <= 1e-4 * outs[False][2].abs().max().item()
    assert 0 < outs[True][3] < c["B"] * c["N"] // 4 and outs[False][3] == 0
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    _, _, want = O.forward(sd, args, S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_WORD, b)
    assert ((outs[True][0].cpu() - want).abs() / want.clamp_min(1e-30)).max().item() < 1e-3


def test_bf16_activation_storage_tracks_fp32():
    """BASELINE configs[2] ("bf16"): activations stored as ONE bf16 plane (aggregation writes no lo plane, the e2e GEMM
    runs one bf16 product), fp32 tables / accumulation / scores.  Stated tolerance: answer probabilities within 5 %
    relative of the fp32 path on entries above 1e-6 (bf16 inputs, K = 1000, 6 layers), argmax and row sums intact."""
    c = dict(S.CONFIGS["cfg2"], B=4, N=256, E=900, T=2)
    m, args = _model(c)
    b = S.make_batch(51, B=c["B"], N=c["N"], E=c["E"], with_weights=False, n_real="ragged")
    _, pred32, d32, _ = m(b)
    d32 = d32.clone()
    ops.ACT_BF16 = True
    try:
        _, pred16, d16, _ = m(b)
        d16 = d16.clone()
        gs = G.GraphedStep(m, S.WEBQSP_NUM_ENTITY)
        assert torch.equal(gs(b).pred_dist, d16)                  # graph replay == eager in this mode too
    finally:
        ops.ACT_BF16 = False
    big = d32 > 1e-6
    rel = ((d16 - d32).abs()[big] / d32[big]).max().item()
    print("bf16 activation storage: max relative deviation from the fp32 path %.2e" % rel)
    assert 0 < rel < 5e-2
    assert torch.allclose(d16.sum(1), torch.ones_like(d16.sum(1)), atol=1e-4)
    assert ((d16 == 0) == (d32 == 0)).all()                       # pads stay exactly zero


def test_entity_dim_400_runs_on_the_tensor_core_path():
    """cfg5's feature width (D = 400 > 256 accumulator columns per GEMM launch): the GEMM is tiled over the output columns (two
    launches per layer); same numbers as the exact-fp32 SIMT path within the split-bf16 bound."""
    c = dict(S.CONFIGS["cfg5"], B=2, N=300, E=1200, T=2)
    m, args = _model(c)
    b = S.make_batch(52, B=2, N=300, E=1200, with_weights=False, powerlaw=True)
    assert m.reasoning.__class__._alloc is not None
    _, _, d_tc, _ = m(b)
    assert m.reasoning.use_planes                                  # the plane / tensor-core data flow was taken
    d_tc = d_tc.clone()
    ops.TC_LINEAR = False
    try:
        _, _, d_ref, _ = m(b)
        assert not m.reasoning.use_planes
    finally:
        ops.TC_LINEAR = True
    big = d_ref > 1e-12
    rel = ((d_tc - d_ref).abs()[big] / d_ref[big]).max().item()
    print("D=400 wgmma (N-tiled) vs fp32 SIMT: max relative deviation %.2e" % rel)
    assert rel < 1e-3
