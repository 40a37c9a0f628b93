"""Rule-guided reasoning paths on the GPU (csrc/rule_paths.cu through gnn_rag_b200.paths) against the reference's
stored results and its networkx restatement (tests/rule_paths_ref.py): same paths, same ORDER."""
import numpy as np
import pytest
import torch

import rule_paths_ref as R
from gnn_rag_b200 import _lib, ops, paths

pytestmark = pytest.mark.gpu

GOLDEN = R.load_golden()


@pytest.mark.parametrize("q", GOLDEN, ids=[q["id"] for q in GOLDEN])
def test_golden_cases_equal_in_content_and_order(q):
    g = paths.build_graph(q["graph"])
    for e, r, want in q["bfs_with_rule"]:
        assert paths.bfs_with_rule(g, e, r) == want
    assert paths.apply_rules(g, q["predicted_paths"], q["q_entity"]) == q["apply_rules"]
    assert paths.direct_answer(q) == [p[-1][-1] for p in q["apply_rules"] if p]     # build_qa_input.py:66-81


def test_batch_equals_golden():
    got = paths.reasoning_paths(GOLDEN)
    for q, r in zip(GOLDEN, got):
        assert r.rule_paths == q["apply_rules"], q["id"]
        assert r.with_rules == q["lists_with_rules"], q["id"]
        assert r.without_rules == q["lists_without_rules"], q["id"]


def random_case(seed, n_ent, n_tri, n_rel, hub_deg=0):
    rs = np.random.RandomState(seed)
    tri = [("m.%03d" % a, " rel.%d " % r, "m.%03d" % b)
           for a, b, r in zip(rs.randint(n_ent, size=n_tri), rs.randint(n_ent, size=n_tri), rs.randint(n_rel, size=n_tri))]
    tri += [tri[0], (tri[1][2], "rel.0", tri[1][0]), (tri[2][0], "rel.1", tri[2][0])]   # duplicate, relabel, self-loop
    src = ["m.%03d" % i for i in rs.randint(n_ent, size=2)] + ["m.absent"]
    if hub_deg:                 # hub rows: merged row longer than the shared-memory sort, duplicates and relabels
        for i in range(hub_deg):
            t = "m.%03d" % rs.randint(n_ent)
            tri.append(("m.hub", "rel.%d" % rs.randint(3), t) if i % 4 else (t, "rel.%d" % rs.randint(3), "m.hub"))
        src.append("m.hub")
    rules = [["rel.%d" % x for x in rs.randint(n_rel, size=rs.randint(1, 4))] for _ in range(3)]
    rules += [[], [" rel.0"], ["rel.%d" % n_rel]]
    names = sorted({h for h, _, _ in tri})
    cand = [names[i] for i in rs.randint(len(names), size=3)] + [src[0]]
    return dict(graph=tri, q_entity=src, predicted_paths=rules, cand=cand)


CASES = [(1, 30, 60, 4, 0), (2, 200, 500, 7, 0), (3, 12, 80, 3, 0), (4, 400, 800, 5, 600), (5, 400, 600, 5, 2600),
         (6, 2000, 6000, 9, 0)]


@pytest.mark.parametrize("seed,n_ent,n_tri,n_rel,hub", CASES)
def test_random_graphs_equal_networkx(seed, n_ent, n_tri, n_rel, hub):
    q = random_case(seed, n_ent, n_tri, n_rel, hub)
    want = R.apply_rules(R.build_graph(q["graph"]), q["predicted_paths"], q["q_entity"])
    got = paths.apply_rules(paths.build_graph(q["graph"]), q["predicted_paths"], q["q_entity"])
    assert got == want
    assert len(want) > 3


def test_batch_with_ragged_questions_equals_the_drop_ins():
    qs = [random_case(s, n, t, r, h) for s, n, t, r, h in CASES[:5]] + GOLDEN[-4:] + [random_case(9, 5, 6, 2)]
    qs[1] = dict(qs[1], cand=None)
    got = paths.reasoning_paths(qs)
    for q, r in zip(qs, got):
        g = paths.build_graph(q["graph"])
        assert r.rule_paths == paths.apply_rules(g, q["predicted_paths"], q["q_entity"])
        strings = [paths.path_to_string(p) for p in r.rule_paths]
        truth = None if q["cand"] is None else [paths.path_to_string(p)
                                                for p in paths.get_truth_paths(q["q_entity"], q["cand"], g)]
        assert r.with_rules == paths.prompt_path_list(strings, truth) == R.lists_of_paths(q, True)
        assert r.without_rules == paths.prompt_path_list([], truth) == R.lists_of_paths(q, False)


def star_walks(k, steps):
    g = paths.build_graph([("c", "r", "l%d" % i) for i in range(k)])
    one = lambda v: np.array([v], dtype=np.int32)  # noqa: E731
    return g.rule_walks(one(0), one(0), one(steps), np.zeros(steps, dtype=np.int32))


@pytest.mark.parametrize("k", [2000, 2500])     # 2500: the hub row is sorted in global memory
def test_star_fan_out_in_closed_form(k):
    nodes, counts, elem_off = star_walks(k, 4)
    assert counts.tolist() == [k * k] and elem_off.tolist() == [0]
    i = np.arange(k * k)
    want = np.stack([np.zeros_like(i), 1 + i // k, np.zeros_like(i), 1 + i % k, np.zeros_like(i)], 1)
    assert np.array_equal(nodes.reshape(k * k, 5), want)


def test_level_beyond_int32_is_refused_with_its_count():
    k = 46341                                     # k * k = 2 147 488 281 > INT32_MAX paths at the third level
    with pytest.raises(_lib.GrError, match="2147488281"):
        star_walks(k, 3)


def test_two_runs_are_bit_identical():
    q = random_case(5, 400, 600, 5, 2600)
    g = paths.build_graph(q["graph"])
    jobs = [(e, r) for e in q["q_entity"] for r in q["predicted_paths"]]
    start, off, ln, lab = paths._encode_jobs(g.lab2id, [g.ent2id.get(e, -1) for e, _ in jobs], [r for _, r in jobs])
    runs = []
    for _ in range(2):
        adj = ops.rule_adjacency(g.csr)
        out, counts, eoff = ops.rule_walks(adj, start, off, ln, lab)
        runs.append((out.clone(), counts, eoff, adj.len.clone(), adj.nbr.clone(), adj.lab.clone()))
    torch.cuda.synchronize()
    a, b = runs
    assert torch.equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert torch.equal(a[3], b[3])
    rp, ln_ = adj.rowptr.cpu().numpy(), a[3].cpu().numpy()
    used = np.concatenate([np.arange(s, s + n) for s, n in zip(rp[:-1], ln_)])     # the rest of a row is capacity
    assert torch.equal(a[4][used], b[4][used]) and torch.equal(a[5][used], b[5][used])
