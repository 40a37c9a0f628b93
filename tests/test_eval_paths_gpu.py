"""The shortest-path node sets of an evaluation epoch (GraphedStep.start_eval(..., path_targets=T), EvalRun.paths) on
the GPU.

Question by question they equal the per-batch path -- ``split.get_batch`` -> model -> ``evaluate.retrieve`` ->
``evaluate.path_node_sets(db, retrieved, T)`` -- for ReaRev, NSM and GraftNet, int32 and int64 indices, short last
batches, T = 1, 32 and above every candidate count, questions with several seeds and with none, candidates a seed
cannot reach, and a shuffled split.  Turning the paths on changes nothing else a run returns, and a sweep member with
paths matches its solo run.  gr_eval_step_paths is held to the restatement in tests/eval_paths_ref.py at its edges."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import evaluate, graphed, loader, ops

import eval_paths_ref as R
from test_device_split_host import NE
from test_eval_epoch_gpu import _evaluator, _loader, _model

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def _paths_loader(name, **kw):
    """test_eval_epoch_gpu's stand-in split with seeds changed: questions 7 and 8 have three and two seeds, 9 and 10
    none, and the seed of question 12 (local 0) is in no fact, so no candidate of it is reachable."""
    L = _loader(name, **kw)
    L.query_entities[7, [3, 5]] = 1.0
    L.query_entities[8, 4] = 1.0
    L.query_entities[[9, 10]] = 0.0
    h, r, t = (np.asarray(a) for a in L.kb_adj_mats[12])
    keep = (h != 0) & (t != 0)
    L.kb_adj_mats[12] = (h[keep], r[keep], t[keep])
    if name == "GraftNet":
        L.kb_fact_rels[12] = L.create_kb_adj_mats_facts(12)[1]
    return L


def _per_batch_paths(m, split, B, eps, T, seeds=None):
    """The per-batch path: (node lists, pair blocks [n_seeds, n_targets]) of every question in batch order; the
    blocks' fill past the counts is checked here."""
    split.reset_batches(is_sequential=True)
    sets, blocks = [], []
    for it in range(-(-split.num_data // B)):
        kw = {} if seeds is None else dict(seed=seeds[it:it + 1])
        batch = split.get_batch(it, B, 0.0, test=True, **kw)
        with torch.no_grad():
            _loss, _pred, dist, _tp = m(batch[:-1])
        ret, _ = evaluate.retrieve(dist, m.last_batch, NE, eps)
        nodes, pair = evaluate.path_node_sets(m.last_batch, ret, T)
        qe = batch[1].cpu().numpy()
        for b, r in enumerate(ret):
            ns, nt = int(np.count_nonzero(qe[b])), min(len(r), T)
            assert (pair[b, ns:] == -1).all() and (pair[b, :, nt:] == -1).all()
            sets.append(nodes[b])
            blocks.append(pair[b, :ns, :nt])
    return sets, blocks


def _assert_paths(got, want):
    sets, blocks = got
    assert len(sets) == len(want[0]) == len(blocks)
    for q, (s, w) in enumerate(zip(sets, want[0])):
        assert s == w, q
    for q, (b, w) in enumerate(zip(blocks, want[1])):
        assert b.dtype == np.int32 and b.shape == w.shape and np.array_equal(b, w), q


@pytest.mark.parametrize("name,index_dtype,B,T,eps", [
    ("ReaRev", torch.int32, 4, 32, 1.0), ("ReaRev", torch.int64, 5, 1, 0.95), ("NSM", torch.int32, 4, 1000, 1.0),
    ("NSM", torch.int64, 3, 32, 0.95), ("GraftNet", torch.int32, 4, 32, 1.0), ("GraftNet", torch.int64, 6, 2, 0.95)])
def test_equal_to_the_per_batch_path(name, index_dtype, B, T, eps):
    """eps = 1 keeps every candidate (question 12's among them), eps = 0.95 the ranking's cut."""
    L = _paths_loader(name)
    m = _model(name, L)
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype)
    step = graphed.GraphedStep(m, NE, eps=eps)
    run = step.start_eval(split, B, path_targets=T)
    got = run.paths()
    want = _per_batch_paths(m, split, B, eps, T)
    _assert_paths(got, want)
    seeds = split.seed_counts()
    assert split.max_seeds() == 3 and seeds[9] == seeds[10] == 0
    assert got[0][9] == [] and got[1][9].shape[0] == 0
    assert any(b.shape[0] > 1 and b.shape[1] > 0 for b in got[1])            # several seeds
    assert got[0][12] == [] and (got[1][12] == -1).all()                        # unreachable candidates
    assert got[1][12].size or eps < 1
    assert [b.shape for b in got[1]] == [(int(seeds[q]), min(len(r), T)) for q, r in enumerate(run.result()[6])]


def test_shuffled_split_replays_from_the_recorded_seeds():
    L = _paths_loader("ReaRev")
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    torch.manual_seed(5)
    run = step.start_eval(split, 4, path_targets=32)
    got = run.paths()
    _assert_paths(got, _per_batch_paths(m, split, 4, 0.95, 32, seeds=run.seeds))


def test_nothing_else_moves(tmp_path):
    """result(), records() and the .info bytes are those of a run without paths; a run without paths captures one
    graph per step shape, as before, and one with paths as many more."""
    L = _paths_loader("GraftNet")
    m = _model("GraftNet", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    tables = _evaluator("GraftNet", m, L, tmp_path, "x", 0.95, step=step).info_tables(split)
    plain = step.start_eval(split, 4)
    want = plain.result(), plain.records(), bytes(plain.info(tables))
    shapes = len(step._cache)
    plan = graphed.epoch_plan(np.arange(L.num_data), split._stored, split._ents, 4, 0.0, split._graft_count)
    assert shapes == len(set(step._layout.epoch_shapes(plan)))
    with_paths = step.start_eval(split, 4, path_targets=32)
    got = with_paths.result(), with_paths.records(), bytes(with_paths.info(tables))
    assert len(step._cache) == 2 * shapes
    for a, b in zip(got[0][:6], want[0][:6]):
        np.testing.assert_array_equal(a, b)
    assert [(r.idx.tolist(), r.ent.tolist(), r.prob.tolist()) for r in got[0][6]] == \
        [(r.idx.tolist(), r.ent.tolist(), r.prob.tolist()) for r in want[0][6]]
    for a, b in zip(got[1], want[1]):
        np.testing.assert_array_equal(a, b)
    assert got[2] == want[2]
    again = step.start_eval(split, 4)
    assert len(step._cache) == 2 * shapes and bytes(again.info(tables)) == want[2]
    with pytest.raises(ValueError, match="started without path_targets"):
        again.paths()


def test_a_sweep_member_with_paths_matches_its_solo_run():
    L = _paths_loader("ReaRev")
    split = loader.DeviceSplit(L, dev)
    m1, m2 = _model("ReaRev", L), _model("NSM", L)
    s1, s2 = graphed.GraphedStep(m1, NE, eps=0.95), graphed.GraphedStep(m2, NE, eps=0.95)
    solo_paths = s1.start_eval(split, 4, path_targets=32).paths()
    solo_plain = s2.start_eval(split, 5).result()
    sweep = graphed.Sweep([s1, s2])
    r1, r2 = sweep.start_evals([(split, 4, 32), (split, 5)])
    _assert_paths(r1.paths(), solo_paths)
    for a, b in zip(r2.result()[:6], solo_plain[:6]):
        np.testing.assert_array_equal(a, b)
    with pytest.raises(ValueError, match="started without path_targets"):
        r2.paths()
    with pytest.raises(ValueError, match="start_eval: path_targets must be a positive int"):
        sweep.start_evals([(split, 4, 0), None])


# ---- gr_eval_step_paths against the restatement -------------------------------------------------------------------

def _t(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dev, dtype)


def _graph(rs, N, n_edges, hub=None):
    h, t = rs.randint(0, N, n_edges), rs.randint(0, N, n_edges)
    if hub is not None:
        h = np.concatenate([h, np.full(3000, hub)])
        t = np.concatenate([t, rs.randint(0, N, 3000)])
    return h, t


def _run_steps(rs, N, num_data, bs, S, T, capacity=None, cursors=None, hub=False):
    """gr_eval_step_paths over ceil(num_data / bs) steps (or at ``cursors``) of random questions -> (device records,
    the restated (nodes, block) of every recorded position)."""
    steps = -(-num_data // bs)
    i32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.int64, device=dev)
    cap = num_data * N if capacity is None else capacity
    node_off, node_count = torch.full((num_data,), -5, **i64), torch.full((num_data,), -5, **i32)
    pair = torch.full((num_data, S, T), -5, **i32)
    nodes, total, status = torch.full((max(cap, 1),), -7, **i32), torch.zeros(1, **i64), torch.zeros(1, **i32)
    cursor = torch.zeros(1, **i64)
    want = {}
    for c in (range(steps) if cursors is None else cursors):
        B = max(min(bs, num_data - c * bs), 1)
        graphs = [_graph(rs, N, N // 2 + rs.randint(0, N), hub=(7 if hub and b == 0 else None)) for b in range(B)]
        qe = np.zeros((B, N), np.float32)
        for b in range(B):
            k = rs.randint(0, S + 1)
            qe[b, rs.choice(N, k, replace=False)] = rs.choice([1.0, 0.5, -2.0], k)
        cand = np.stack([rs.permutation(N) for _ in range(B)]).astype(np.int32)
        cnt = rs.randint(0, min(N, T + 3) + 1, B).astype(np.int32)
        for b in range(B):                                   # a source equal to a target
            src = np.nonzero(qe[b])[0]
            if len(src) and cnt[b]:
                cand[b, 0] = src[0]
        heads = np.concatenate([h + b * N for b, (h, _) in enumerate(graphs)])
        tails = np.concatenate([t + b * N for b, (_, t) in enumerate(graphs)])
        g = ops.csr_build(_t(heads, torch.int64), _t(np.zeros_like(heads), torch.int64), _t(tails, torch.int64),
                          B, N, 1)
        cursor.fill_(c)
        ops.eval_step_paths(cursor, bs, steps, num_data, g, _t(qe, torch.float32), _t(cand, torch.int32),
                            _t(cnt, torch.int32), S, T, node_off, node_count, pair, nodes[:cap], total, status)
        if 0 <= c < steps:
            for b, rec in enumerate(R.eval_step_paths(graphs, N, qe, cand, cnt, S, T)):
                if c * bs + b < num_data:
                    want[c * bs + b] = rec
    out = dict(node_off=node_off.cpu().numpy(), node_count=node_count.cpu().numpy(), pair=pair.cpu().numpy(),
               nodes=nodes.cpu().numpy(), total=int(total.item()), status=int(status.item()))
    return out, want, steps


def _check(out, want, bs, capacity=None):
    run = 0
    written = {}
    for c in sorted({p // bs for p in want}):
        ps = [p for p in sorted(want) if p // bs == c]
        end = run + sum(len(want[p][0]) for p in ps)
        for p in ps:
            nodes, block = want[p]
            assert out["node_off"][p] == run and out["node_count"][p] == len(nodes), p
            assert np.array_equal(out["pair"][p], block), p
            written[p] = capacity is None or end <= capacity
            if written[p]:
                assert out["nodes"][run:run + len(nodes)].tolist() == nodes, p
            run += len(nodes)
    assert out["total"] == run
    return run, written


@pytest.mark.parametrize("N,S,T", [(40, 3, 4), (513, 2, 5), (13_000, 1, 3)])
def test_step_kernel_against_the_restatement(N, S, T):
    """N below one block, N = 513 (not a multiple of the 512-thread block) and N = 13 000 (past the shared-memory
    distance rows); several steps, the last one short; S above most questions' seed counts; a hub row."""
    out, want, steps = _run_steps(np.random.RandomState(N), N, num_data=7, bs=3, S=S, T=T, hub=True)
    assert len(want) == 7 and out["status"] == 0
    run, _ = _check(out, want, 3)
    assert run > 0
    assert (out["nodes"][run:] == -7).all()


def test_step_kernel_overflow_and_cursors_past_the_steps():
    full, want, _ = _run_steps(np.random.RandomState(3), 60, num_data=8, bs=3, S=2, T=6)
    total = full["total"]
    cap = total // 2
    out, want2, _ = _run_steps(np.random.RandomState(3), 60, num_data=8, bs=3, S=2, T=6, capacity=cap)
    assert out["status"] == 2 and out["total"] == total
    _run, written = _check(out, want2, 3, capacity=cap)
    assert not all(written.values())
    last = max((out["node_off"][p] + out["node_count"][p] for p, w in written.items() if w), default=0)
    assert (out["nodes"][last:cap] == -7).all()                       # nothing of a step that does not fit
    for k in ("node_off", "node_count", "pair"):
        assert np.array_equal(out[k], full[k]), k
    # a cursor outside [0, steps) writes nothing
    out, want3, _ = _run_steps(np.random.RandomState(4), 30, num_data=6, bs=3, S=2, T=3, cursors=[0, 5, -1])
    assert sorted(want3) == [0, 1, 2]
    _check(out, want3, 3)
    assert (out["node_off"][3:] == -5).all() and (out["pair"][3:] == -5).all()
