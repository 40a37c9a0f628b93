"""The restatements of tests/rule_adj_ref.py pinned without a GPU: the label-grouped adjacency against networkx's
neighbour lists (tests/rule_paths_ref.build_graph), and the level expansion against the networkx restatement of
bfs_with_rule / apply_rules, on graphs with duplicate, reversed and relabelled triples, self-loops and isolated nodes,
and on the golden questions."""
import numpy as np
import pytest

pytest.importorskip("networkx")

import rule_adj_ref as A  # noqa: E402
import rule_paths_ref as R  # noqa: E402

GOLDEN = R.load_golden()


def messy_triples(seed, n_ent, n_tri, n_rel, extra):
    """n_tri random triples, then ``extra`` of each kind inserted at a random later place than the triple they copy:
    a duplicate, the reversed pair with the same label, the pair (either direction) with another label, and a
    self-loop.  Relation strings carry surrounding whitespace now and then (the label is the stripped string)."""
    rs = np.random.RandomState(seed)
    rel = lambda: ("r%d" % rs.randint(n_rel)) if rs.rand() < 0.8 else (" r%d " % rs.randint(n_rel))  # noqa: E731
    tri = [("e%d" % rs.randint(n_ent), rel(), "e%d" % rs.randint(n_ent)) for _ in range(n_tri)]
    for kind in range(4):
        for _ in range(extra):
            k = rs.randint(len(tri))
            h, r, t = tri[k]
            new = [(h, r, t), (t, r, h), ((h, rel(), t) if rs.rand() < 0.5 else (t, rel(), h)), (h, rel(), h)][kind]
            tri.insert(rs.randint(k + 1, len(tri) + 1), new)
    return tri


GRAPHS = [messy_triples(1, 6, 10, 2, 3), messy_triples(2, 30, 80, 4, 10), messy_triples(3, 200, 600, 6, 60),
          messy_triples(4, 12, 300, 3, 40), [("a", "r", "a")], [("a", "r", "a"), ("a", "s", "a"), ("a", "r", "b")]]


def nx_rows(tri):
    """Per entity id, networkx's neighbour list with label ids, after a stable sort by label."""
    names, lab2id, _, _, _ = A.intern(tri)
    ids = {e: i for i, e in enumerate(names)}
    G = R.build_graph(tri)
    rows = []
    for e in names:
        row = [(ids[v], lab2id[G[e][v]["relation"]]) for v in G.neighbors(e)]
        rows.append(sorted(row, key=lambda x: x[1]))
    return rows


@pytest.mark.parametrize("tri", GRAPHS, ids=range(len(GRAPHS)))
def test_adjacency_rows_are_networkx_neighbours_stably_by_label(tri):
    names, _, h, l, t = A.intern(tri)
    pad = 3                                                   # isolated rows, as in a padded batch
    adj = A.adjacency(h, l, t, 1, len(names) + pad)
    for u, want in enumerate(nx_rows(tri)):
        assert A.row(adj, u) == want, u
    for u in range(len(names), len(names) + pad):
        assert A.row(adj, u) == []
    deg = np.array([(h == u).sum() + (t == u).sum() for u in range(len(names) + pad)])   # a self-loop counts twice
    assert np.array_equal(np.diff(adj["rowptr"]), deg) and adj["rowptr"][0] == 0
    assert (adj["len"] <= deg).all()
    assert np.array_equal(adj["key"], np.sort(adj["key"]))
    used = A.used_slots(adj)
    assert len(np.unique(used)) == len(used) and (used < adj["rowptr"][-1]).all()


def test_adjacency_of_a_batch_is_each_question_shifted():
    N = 250
    qs = GRAPHS[:4]
    parts = [A.intern(tri) for tri in qs]
    adj = A.adjacency(np.concatenate([p[2] + b * N for b, p in enumerate(parts)]), np.concatenate([p[3] for p in parts]),
                      np.concatenate([p[4] + b * N for b, p in enumerate(parts)]), len(qs), N)
    for b, (tri, p) in enumerate(zip(qs, parts)):
        for u, want in enumerate(nx_rows(tri)):
            assert A.row(adj, b * N + u) == [(v + b * N, x) for v, x in want]
        assert all(A.row(adj, b * N + u) == [] for u in range(len(p[0]), N))


def rules_for(tri, seed):
    """Rules over the graph's labels (lengths 1-4), an empty rule, an unstripped label, a label the graph does not
    have at the first and at a middle position."""
    rs = np.random.RandomState(seed)
    labs = sorted({r.strip() for _, r, _ in tri})
    rules = [[labs[i] for i in rs.randint(len(labs), size=rs.randint(1, 5))] for _ in range(5)]
    return rules + [[], [" " + labs[0]], ["absent", labs[0]], [labs[0], "absent", labs[0]]]


@pytest.mark.parametrize("tri", GRAPHS, ids=range(len(GRAPHS)))
def test_expand_equals_networkx_apply_rules(tri):
    names = A.intern(tri)[0]
    rs = np.random.RandomState(len(tri))
    sources = [names[i] for i in rs.randint(len(names), size=3)] + ["absent"]
    rules = rules_for(tri, len(tri))
    got = A.apply_rules(tri, rules, sources)
    assert got == R.apply_rules(R.build_graph(tri), rules, sources)
    assert len(got) > len(sources)                      # at least the empty rule's path per source, and more


@pytest.mark.parametrize("q", GOLDEN, ids=[q["id"] for q in GOLDEN])
def test_expand_reproduces_the_golden_questions(q):
    assert A.apply_rules(q["graph"], q["predicted_paths"], q["q_entity"]) == q["apply_rules"]


def test_empty_graph_empty_rule_and_absent_start():
    assert A.apply_rules([], [[], ["r"]], ["a"]) == [[]]
    tri = [("a", "r", "b")]
    assert A.apply_rules(tri, [[], ["r"], ["r", "r"]], ["zz", "a"]) == \
        [[], [], [("a", "r", "b")], [("a", "r", "b"), ("b", "r", "a")]]


def test_expand_levels_are_job_major_and_finish_where_the_rule_ends():
    tri = GRAPHS[2]
    names, lab2id, h, l, t = A.intern(tri)
    rules = rules_for(tri, 7)
    jobs = [(s, r) for s in [-1, 0, 5, 17] for r in rules]
    start, off, ln, lab = A.encode_jobs(lab2id, [s for s, _ in jobs], [r for _, r in jobs])
    x = A.expand(A.adjacency(h, l, t, 1, len(names)), start, off, ln, lab)
    for lv, level in enumerate(x["levels"]):
        assert (np.diff(level["job"]) >= 0).all()
        assert level["off"][-1] == (len(x["levels"][lv + 1]["node"]) if lv + 1 < len(x["levels"]) else level["off"][-1])
        fin = np.flatnonzero(ln == lv)
        assert np.array_equal(level["fin"], fin)
        for j, b, c in zip(fin, level["res_begin"], level["res_count"]):
            assert (level["job"][b: b + c] == j).all() and c == (level["job"] == j).sum()
    dropped = [j for j, (s, r) in enumerate(jobs) if s < 0 and len(r)]
    assert all(x["counts"][j] == 0 for j in dropped)
    assert all(x["counts"][j] == 1 for j, (_, r) in enumerate(jobs) if not r)
