"""A whole evaluation replayed as CUDA graphs (GraphedStep.start_eval, Evaluator(step=...)) on the GPU.

Over a ``loader.DeviceSplit`` the evaluation epoch returns what the per-batch ``Evaluator`` returns -- equal means,
equal ``case_ct`` and a byte-identical ``.info`` file -- for ReaRev, NSM and GraftNet, int32 and int64 indices, fact
weights, short last batches, one batch larger than the split, batches of one, every candidate kept and almost none,
and questions without answers, with answers outside the subgraph, with repeated answers and without facts.  A shuffled
split replays from the recorded seeds.  The graphs survive in-place parameter updates without a new capture, a warm
evaluation does not synchronise with the host, and malformed orders reach ``EvalRun.check``.  gr_eval_step_record is
held to an exact restatement on ``evaluate.f1_and_hits`` at its edges."""
import os

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import evaluate, graphed, loader, ops, synthetic as S

from test_device_split_host import NE, NW, GraftSplitLoader, SplitLoader

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
ENT = {"e%d" % i: i for i in range(NE)}          # the pad id is len(ENT) = NE, the stand-ins' pad


def _loader(name, num_questions=13, seed=21, **kw):
    """A stand-in split whose answers cover the evaluator's cases: question 0 has neither answers nor candidates (its
    entities are its seed and pads), 1 one answer outside its subgraph, 2 a repeated one, 3 a repeat and an outsider,
    5 answers but no candidates, 6 candidates but no answers; question 4 has no facts."""
    cls = GraftSplitLoader if name == "GraftNet" else SplitLoader
    L = cls(seed=seed, num_questions=num_questions, max_local_entity=50, facts_lo=20, facts_hi=300, **kw)
    row = lambda q: L.candidate_entities[q]                  # noqa: E731
    outsider = lambda q: int(next(e for e in range(NE) if e not in set(row(q).tolist())))   # noqa: E731
    L.candidate_entities[[0, 5], 1:] = NE
    L.answer_lists[0] = L.answer_lists[6] = []
    L.answer_lists[1] = [outsider(1)]
    L.answer_lists[2] = [int(row(2)[1])] * 2 + list(L.answer_lists[2])
    L.answer_lists[3] = [outsider(3), int(row(3)[2]), int(row(3)[2])]
    empty = np.zeros(0, dtype=int)
    L.kb_adj_mats[4] = (empty, empty, empty)
    if name == "GraftNet":
        L.kb_fact_rels[4] = L.create_kb_adj_mats_facts(4)[1]
    return L


def _model(name, L, **over):
    torch.manual_seed(0)
    args = S.model_args(name, entity_dim=50, use_cuda=True, word_dim=64, linear_dropout=0.0, lm_dropout=0.0, **over)
    if name == "ReaRev":
        args.update(num_ins=2, num_iter=2, num_gnn=2)
    elif name == "NSM":
        args.update(num_step=2)
    else:
        args.update(num_layer=2)
    cls = {"ReaRev": G.ReaRev, "NSM": G.NSM, "GraftNet": G.GraftNet}[name]
    m = cls(dict(args), NE, L.num_kb_relation, NW).cuda().eval()
    with torch.no_grad():                  # a sharper distribution: fewer candidates survive the eps cut
        for p in m.parameters():
            if p.dim() == 2:
                p.mul_(3.0)
    return m


def _evaluator(name, m, L, tmp_path, tag, eps, step=None):
    args = dict(S.model_args(name), checkpoint_dir=str(tmp_path), experiment_name=tag, eps=eps)
    rel = {"r%d" % i: i for i in range(L.num_kb_relation)}
    return evaluate.Evaluator(args, m, ENT, rel, dev, step=step)


def _run(ev, split, B, tmp_path, tag):
    out = ev.evaluate(split, test_batch_size=B)
    with open(os.path.join(str(tmp_path), tag + "_test.info"), "rb") as f:
        return out, dict(ev.case_ct), f.read()


def _assert_same_as_per_batch(name, m, L, split, B, eps, tmp_path, step):
    want = _run(_evaluator(name, m, L, tmp_path, "batch", eps), split, B, tmp_path, "batch")
    ids_batch = list(L.sample_ids)
    got = _run(_evaluator(name, m, L, tmp_path, "epoch", eps, step=step), split, B, tmp_path, "epoch")
    assert list(L.sample_ids) == ids_batch
    assert got[0] == want[0] and all(type(x) is float for x in got[0])
    assert got[1] == want[1]
    assert got[2] == want[2] and len(want[2].splitlines()) == L.num_data
    return want


@pytest.mark.parametrize("name,index_dtype,over", [
    ("ReaRev", torch.int32, {}), ("ReaRev", torch.int64, dict(normalized_gnn=True, norm_rel=True)),
    ("NSM", torch.int32, {}), ("NSM", torch.int64, dict(normalized_gnn=True)),
    ("GraftNet", torch.int32, {}), ("GraftNet", torch.int64, dict(norm_rel=True))])
def test_equal_to_the_per_batch_evaluator(name, index_dtype, over, tmp_path):
    L = _loader(name)
    m = _model(name, L, **over)
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    want = _assert_same_as_per_batch(name, m, L, split, 4, 0.95, tmp_path, step)
    assert set(want[1]) == {0, 1, 2, 3}


@pytest.mark.parametrize("B,eps", [(1, 0.95), (64, 0.95), (5, 1.0), (5, 1e-6)])
def test_batch_sizes_and_eps(B, eps, tmp_path):
    """B = 1, one batch larger than the split, every candidate (eps >= 1) and only the first ones (tiny eps)."""
    L = _loader("ReaRev")
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=eps)
    want = _assert_same_as_per_batch("ReaRev", m, L, split, B, eps, tmp_path, step)
    if eps >= 1:
        assert 1 in want[1]                           # candidates without answers


def _per_batch(m, split, B, eps, seeds=None):
    """The per-batch evaluation loop on the records' terms: (metrics [n, 5], cases, [(idx, ent, prob)])."""
    split.reset_batches(is_sequential=True)
    rows, cases, cands = [], [], []
    for it in range(-(-split.num_data // B)):
        kw = {} if seeds is None else dict(seed=seeds[it:it + 1])
        batch = split.get_batch(it, B, 0.0, test=True, **kw)
        with torch.no_grad():
            _loss, _pred, dist, _tp = m(batch[:-1])
        ret, _ = evaluate.retrieve(dist, m.last_batch, NE, eps)
        for r, answers in zip(ret, batch[-1]):
            p, rc, f1, hit, em, case = evaluate.f1_and_hits(list(answers), r.ent.tolist())
            rows.append((p, rc, f1, hit, float(em)))
            cases.append(case)
            cands.append((r.idx.tolist(), r.ent.tolist(), r.prob.tolist()))
    return np.array(rows, dtype=np.float64).reshape(-1, 5), cases, cands


def _assert_result(res, want):
    metrics, cases, cands = want
    for k in range(5):
        np.testing.assert_array_equal(res[k], metrics[:, k])
        assert res[k].dtype == np.float64
    assert res[5].tolist() == cases
    assert [(r.idx.tolist(), r.ent.tolist(), r.prob.tolist()) for r in res[6]] == cands


def test_shuffled_split_replays_from_the_recorded_seeds():
    L = _loader("GraftNet")
    m = _model("GraftNet", L)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    torch.manual_seed(7)
    run = step.start_eval(split, 4)
    res = run.result()
    run.check()
    assert run.seeds is not None and run.seeds.numel() == 4
    _assert_result(res, _per_batch(m, split, 4, 0.95, seeds=run.seeds))


def test_graphs_survive_in_place_updates(tmp_path):
    """optimizer.step() and load_state_dict write the parameters in place: no new capture, and the next evaluation
    is the per-batch evaluator's at the new weights."""
    L = _loader("ReaRev")
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    first = _assert_same_as_per_batch("ReaRev", m, L, split, 4, 0.95, tmp_path, step)
    graphs = len(step._cache)
    params = [p for p in m.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=2e-2)
    g = torch.Generator(device=dev).manual_seed(3)
    for p in params:
        p.grad = torch.randn(p.shape, device=dev, generator=g)
    opt.step()
    second = _assert_same_as_per_batch("ReaRev", m, L, split, 4, 0.95, tmp_path, step)
    assert len(step._cache) == graphs
    assert second[2] != first[2]                      # the update changed what is retrieved
    m.load_state_dict({k: v * 0.5 if v.is_floating_point() else v for k, v in m.state_dict().items()})
    third = _assert_same_as_per_batch("ReaRev", m, L, split, 4, 0.95, tmp_path, step)
    assert len(step._cache) == graphs
    assert third[2] != second[2]


def test_warm_evaluation_does_not_synchronise():
    L = _loader("NSM")
    m = _model("NSM", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    want = step.evaluate_split(split, 4)
    graphs = len(step._cache)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        run = step.start_eval(split, 4)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(step._cache) == graphs
    got = run.result()
    run.check()
    for a, b in zip(got[:6], want[:6]):
        np.testing.assert_array_equal(a, b)


def test_out_of_range_question_id_reaches_check():
    L = _loader("ReaRev")
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)

    def bad_order(is_sequential=True):
        L.batches = np.arange(L.num_data)
        L.batches[5] = L.num_data + 7
    L.reset_batches = bad_order
    run = step.start_eval(split, 4)
    run.result()
    with pytest.raises(RuntimeError, match=r"DeviceSplit: batch assembly status 1 \(1: question id out of range"):
        run.check()
    with pytest.raises(RuntimeError, match="batch assembly status 1"):
        step.evaluate_split(split, 4)


def test_refusals(tmp_path):
    L = _loader("ReaRev")
    m = _model("ReaRev", L, normalized_gnn=True)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    Lg = _loader("GraftNet")
    mg = _model("GraftNet", Lg)
    gsplit = loader.DeviceSplit(Lg, dev)
    for st, data, B, msg in [
            (step, L, 4, "the split must be a loader.DeviceSplit"),
            (step, gsplit, 4, "a ReaRev / NSM model evaluates a kb split"),
            (graphed.GraphedStep(mg, NE), split, 4, "GraftNet evaluates a GraftNet split"),
            (step, split, 0, "batch_size must be a positive int"), (step, split, -2, "batch_size must be a positive"),
            (step, split, True, "batch_size must be a positive int"), (step, split, 2.0, "batch_size must be"),
            (step, loader.DeviceSplit(L, dev, weights="none"), 4, "normalized_gnn / norm_rel need fact weights")]:
        with pytest.raises(ValueError, match="start_eval: " + msg):
            st.start_eval(data, B)
    L.q_type = "con"
    with pytest.raises(ValueError, match="start_eval: q_type must be 'seq'"):
        step.start_eval(split, 4)
    L.q_type = "seq"
    bad = _loader("ReaRev")
    bad.answer_lists[6] = [3, 4.5]
    with pytest.raises(ValueError, match="question 6 has an answer that is not an int64 entity id"):
        step.start_eval(loader.DeviceSplit(bad, dev), 4)
    assert len(step._cache) == 0
    for st, eps, msg in [(graphed.GraphedStep(m, NE + 1, eps=0.95), 0.95, "pad id %d" % (NE + 1)),
                         (graphed.GraphedStep(m, NE, eps=0.5), 0.95, "eps 0.5"),
                         (graphed.GraphedStep(mg, NE, eps=0.95), 0.95, "a graphed.GraphedStep of this model")]:
        with pytest.raises(ValueError, match="Evaluator: .*" + msg):
            _evaluator("ReaRev", m, L, tmp_path, "x", eps, step=st)


# ---- gr_eval_step_record against f1_and_hits ---------------------------------------------------------------------

def _record_case(rs, B, N, num_data, num_q, answers, capacity=None, steps=None, cursors=None):
    """Run gr_eval_step_record at ``cursors`` (default: every step) over the order 0, 1, .. num_q - 1, 0, .. of
    ``num_data`` ids on random ranked lists -> (order, device buffers, the host inputs of every call)."""
    bs = B
    steps = -(-num_data // bs) if steps is None else steps
    order = np.arange(num_data) % num_q
    off, ids = loader.pack_answers(answers)
    a_off, a_ids = (torch.from_numpy(a).to(dev) for a in (off, ids))
    cap = B * N * max(steps, 1) if capacity is None else capacity
    i64, i32 = dict(dtype=torch.int64, device=dev), dict(dtype=torch.int32, device=dev)
    cursor = torch.zeros(1, **i64)
    metrics = torch.full((num_data, 5), -7.0, dtype=torch.float64, device=dev)
    cases = torch.full((num_data,), -1, dtype=torch.int8, device=dev)
    counts, cand_off = torch.full((num_data,), -1, **i32), torch.full((num_data,), -1, **i64)
    cand, total = torch.zeros(max(cap, 1), 2, **i64), torch.zeros(1, **i64)
    seeds, status = torch.zeros(max(steps, 1), **i64), torch.zeros(3, **i32)
    inputs = []
    for c in (range(steps) if cursors is None else cursors):
        cursor.fill_(c)
        pos = [c * bs + j for j in range(B)]
        step_ids = np.array([order[p] if 0 <= p < num_data else -1 for p in pos], dtype=np.int64)
        le = rs.randint(0, 12, (B, N)).astype(np.int64)               # few distinct ids: repeats among candidates
        le[:, :3] = -1 if c % 2 else le[:, :3]                          # -1 entities (matched by a -1 answer)
        dist = rs.rand(B, N).astype(np.float32)
        cidx = np.stack([rs.permutation(N) for _ in range(B)]).astype(np.int32)
        cnt = rs.randint(0, N + 1, B).astype(np.int32)
        cnt[0] = 0 if c % 3 == 0 else N
        seed = torch.tensor([1000 + c], **i64)
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
        ops.eval_step_record(cursor, bs, steps, T(step_ids), T(le), T(dist), T(cidx), T(cnt), a_off, a_ids, seed,
                             torch.tensor([c % 2], **i32), torch.tensor([4 if c == 1 else 0], **i32), metrics,
                             cases, counts, cand_off, cand, total, seeds, status)
        inputs.append((c, step_ids, le, dist, cidx, cnt))
    return order, dict(metrics=metrics, cases=cases, counts=counts, cand_off=cand_off, cand=cand, total=total,
                       seeds=seeds, status=status, cursor=cursor), inputs


def _expected(answers, inputs, bs, num_data):
    want = {}
    for c, step_ids, le, dist, cidx, cnt in inputs:
        for j in range(len(step_ids)):
            p = c * bs + j
            if p >= num_data or step_ids[j] < 0:
                continue
            k = cidx[j, :cnt[j]]
            ents = le[j, k].tolist()
            q = int(step_ids[j])
            want[p] = (evaluate.f1_and_hits(list(answers[q]) if q < len(answers) else [], ents), k, le[j, k],
                       dist[j, k])
    return want


def _check_records(out, want, capacity):
    m, cases, counts = out["metrics"].cpu().numpy(), out["cases"].cpu().tolist(), out["counts"].cpu().tolist()
    offs, cand = out["cand_off"].cpu().tolist(), out["cand"].cpu().numpy()
    run = 0
    for p in sorted(want):
        (pr, rc, f1, hit, em, case), k, ents, probs = want[p]
        assert m[p].tolist() == [pr, rc, f1, hit, float(em)], p
        assert type(pr) is float and type(f1) is float
        assert cases[p] == case and counts[p] == len(k)
        assert offs[p] == run
        if run + len(k) <= capacity:
            rec = cand[run:run + len(k)]
            assert rec[:, 0].tolist() == ents.tolist()
            pair = rec[:, 1:].copy().view(np.int32)
            assert pair[:, 0].tolist() == k.tolist()
            assert pair[:, 1].view(np.float32).tobytes() == probs.tobytes()
        run += len(k)
    return run


def test_record_kernel_against_f1_and_hits():
    """Short last batch (positions past num_data), C = 0 with and without answers, C = N, repeated candidate ids, -1
    among the answers (hit with no candidate), repeated answers and a question of 1 000 answers."""
    rs = np.random.RandomState(0)
    num_q = 9
    answers = [[] for _ in range(num_q)]
    answers[1] = [3, 3, 5]
    answers[2] = [-1]
    answers[3] = [-1, 7, 7, 2]
    answers[4] = list(range(2, 2002, 2))                     # A = 1 000
    answers[5] = [100, 200]                                  # never among the candidates
    for q in (6, 7, 8):
        answers[q] = rs.randint(0, 12, rs.randint(1, 6)).tolist()
    B, N, num_data = 7, 40, 30                               # 5 steps, the last one of 2
    order, out, inputs = _record_case(rs, B, N, num_data, num_q, answers)
    want = _expected(answers, inputs, B, num_data)
    assert len(want) == num_data
    assert {w[0][5] for w in want.values()} == {0, 1, 2, 3}
    run = _check_records(out, want, out["cand"].shape[0])
    assert out["total"].item() == run
    assert out["seeds"].cpu().tolist() == [1000 + c for c in range(5)]
    assert out["status"].cpu().tolist() == [1, 4, 0] and out["cursor"].item() == 5


def test_record_kernel_past_the_steps_and_cut_short():
    rs = np.random.RandomState(1)
    num_q, B, N, num_data = 6, 5, 30, 12
    answers = [rs.randint(0, 12, 3).tolist() for _ in range(num_q)]
    # a cursor past the steps records nothing and flags bit 2
    order, out, inputs = _record_case(rs, B, N, num_data, num_q, answers, steps=3, cursors=[0, 1, 2, 3, 7])
    want = _expected(answers, [i for i in inputs if i[0] < 3], B, num_data)
    _check_records(out, want, out["cand"].shape[0])
    assert out["status"].cpu().tolist()[0] & 2 and out["cursor"].item() == 8
    assert out["seeds"].cpu().tolist() == [1000, 1001, 1002]
    # records cut short: the question that does not fit is not written, and nothing after it
    order, full, inputs = _record_case(np.random.RandomState(2), B, N, num_data, num_q, answers)
    want = _expected(answers, inputs, B, num_data)
    total = full["total"].item()
    cap = total // 2
    order, out, _ = _record_case(np.random.RandomState(2), B, N, num_data, num_q, answers, capacity=cap)
    assert out["status"].cpu().tolist()[2] == 1 and out["total"].item() == total
    _check_records(out, want, cap)
    for k in ("metrics", "cases", "counts", "cand_off"):
        assert torch.equal(out[k], full[k]), k
    fits = [p for p in sorted(want) if full["cand_off"][p].item() + len(want[p][1]) <= cap]
    last = max((full["cand_off"][p].item() + len(want[p][1]) for p in fits), default=0)
    assert not out["cand"][last:].any()
