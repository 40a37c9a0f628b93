"""Generate tests/golden/rule_paths/cases.json: rule-guided reasoning paths of the UNMODIFIED reference
(``llm/src/utils/graph_utils.py`` and ``llm/src/utils/utils.py`` of cmavro/GNN-RAG, loaded by file path) on seeded
synthetic question graphs.  Needs a checkout of the reference:

    python tests/golden/make_rule_paths_golden.py [REFERENCE_LLM_DIR]

``graph_utils`` opens ``entities_names.json`` from the working directory at import time, so the script changes into
the reference's ``llm/`` directory before loading it.  The relation strings and rules come from the shipped
``results/gen_rule_path/RoG-*/RoG/test/predictions_3_False.jsonl``; chains that follow the rules are planted in the
graphs so that the rules match.  Stored per question: the inputs, every ``bfs_with_rule`` call that
``PromptBuilder.apply_rules`` makes (build_qa_input.py:58-64) in its order -- their concatenation is the ``apply_rules``
result --, and the ``lists_of_paths`` of ``process_input`` (:92-124) with ``add_rule`` on and off.
"""
import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(HERE, "rule_paths", "cases.json")


def load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def apply_rules(gu, graph, rules, sources):                  # build_qa_input.py:58-64
    results = []
    for entity in sources:
        for rule in rules:
            results.extend(gu.bfs_with_rule(graph, entity, rule))
    return results


def lists_of_paths(gu, ut, q, add_rule):                      # build_qa_input.py:92-124, before check_prompt_length
    lists = []
    graph = None
    if add_rule:
        graph = gu.build_graph(q["graph"], [], False)
        rules = q["predicted_paths"]
        if len(rules) > 0:
            lists = [ut.path_to_string(p) for p in apply_rules(gu, graph, rules, q["q_entity"])]
        else:
            lists = []
    if q["cand"] is not None:
        if not add_rule:
            graph = gu.build_graph(q["graph"], [], False)
        for p in gu.get_truth_paths(q["q_entity"], q["cand"], graph):
            if ut.path_to_string(p) not in lists:
                lists.append(ut.path_to_string(p))
    return lists


def plant(rs, tri, ents, start, rule, branches):
    """Add chains from ``start`` whose i-th edge carries rule[i] (random direction, some steps to existing nodes)."""
    frontier = [start]
    for rel in rule:
        nxt = []
        for u in frontier:
            for _ in range(branches):
                v = ents[rs.randint(len(ents))] if rs.rand() < 0.3 else "m.p%d" % len(tri)
                tri.append((u, rel, v) if rs.rand() < 0.5 else (v, rel, u))
                nxt.append(v)
        frontier = nxt[:2]
    return tri


def planted_case(rs, name, rules, pool, n_ent, n_tri, n_src=1):
    ents = ["m.%d" % i for i in range(n_ent)]
    tri = [(ents[rs.randint(n_ent)], pool[rs.randint(len(pool))], ents[rs.randint(n_ent)]) for _ in range(n_tri)]
    src = [ents[i] for i in rs.choice(n_ent, size=n_src, replace=False)]
    for s in src:
        for r in rules:
            plant(rs, tri, ents, s, r, 2 if len(r) < 3 else 1)
    names = sorted({h for h, _, _ in tri} | {t for _, _, t in tri})
    cand = [names[i] for i in rs.choice(len(names), size=4, replace=False)] + ["m.absent"]
    return dict(id=name, graph=tri, q_entity=src, predicted_paths=rules, cand=cand)


def main():
    llm = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(ref_harness.REFERENCE_GNN), "llm")
    os.chdir(llm)
    gu = load("ref_graph_utils", os.path.join(llm, "src", "utils", "graph_utils.py"))
    ut = load("ref_utils", os.path.join(llm, "src", "utils", "utils.py"))
    preds = []
    for ds in ("RoG-webqsp", "RoG-cwq"):
        with open(os.path.join(llm, "results", "gen_rule_path", ds, "RoG", "test", "predictions_3_False.jsonl")) as f:
            preds.append([json.loads(line)["prediction"] for line in f])
    rs = np.random.RandomState(2024)
    pool = sorted({rel for p in preds for rules in p for rule in rules for rel in rule})
    qs = []
    # shipped rules (WebQSP and CWQ, incl. questions with an empty rule), planted on random graphs
    web_empty = [i for i, r in enumerate(preds[0]) if any(len(x) == 0 for x in r)][:1]
    cwq_long = [i for i, r in enumerate(preds[1]) if any(len(x) >= 4 for x in r)][:1]
    picks = [(0, i) for i in list(rs.choice(len(preds[0]), 1)) + web_empty] + \
            [(1, i) for i in list(rs.choice(len(preds[1]), 1)) + cwq_long]
    for k, (d, i) in enumerate(picks):
        rules = preds[d][i]
        local = sorted({rel for r in rules for rel in r}) + [pool[j] for j in rs.choice(len(pool), 2)]
        qs.append(planted_case(rs, "shipped_%d_%d" % (d, i), rules, local, 10 + 4 * k, 12 + 4 * k, 1 + k % 2))
    r1, r2, r3 = sorted(pool, key=lambda x: (len(x), x))[:3]             # short labels keep the fixture readable
    # duplicate triples, a reversed duplicate that relabels the pair, labels with whitespace around them
    qs.append(dict(id="duplicates_relabel", q_entity=["a"], cand=["c", "b"],
                   graph=[("a", r1, "b"), ("a", r1, "b"), ("b", r1, "c"), ("c", r2, "b"), ("a", " %s " % r3, "d"),
                          ("d", r1, "a"), ("a", r1, "e"), ("e", r2, "a"), ("a", r1, "e")],
                   predicted_paths=[[r1], [r2], [r1, r1], [r1, r2], [r3], [r1, r3]]))
    # self-loops: u is once in its own neighbour list
    qs.append(dict(id="self_loop", q_entity=["a", "b"], cand=["a"],
                   graph=[("a", r1, "a"), ("a", r1, "b"), ("b", r2, "b"), ("b", r1, "c")],
                   predicted_paths=[[r1], [r1, r1], [r1, r1, r1], [r2, r2, r1]]))
    # a cycle: walks revisit nodes and step straight back
    qs.append(dict(id="cycle", q_entity=["x"], cand=["z"],
                   graph=[("x", r1, "y"), ("y", r1, "z"), ("z", r1, "x"), ("z", r2, "w")],
                   predicted_paths=[[r1, r1, r1, r1], [r1, r1, r2], [r1, r2, r2, r1]]))
    # a hub: out through the hub and back, two labels interleaved in insertion order
    hub = [("hub", r1 if i % 3 else r2, "leaf%d" % i) for i in range(24)] + [("src", r1, "hub")]
    hub += [("leaf%d" % i, r3, "hub") for i in range(0, 24, 7)]             # relabels some hub-leaf pairs
    qs.append(dict(id="hub", q_entity=["src"], cand=["leaf5", "leaf9"], graph=hub,
                   predicted_paths=[[r1, r1], [r1, r2, r2], [r1, r3, r3]]))
    # labels absent from the graph, rule elements with whitespace, empty rules, starts not in the graph
    qs.append(dict(id="absent_whitespace_empty_missing", q_entity=["a", "not.in.graph", "b"], cand=None,
                   graph=[("a", r1, "b"), ("b", " %s" % r2, "c"), ("c", r1, "a")],
                   predicted_paths=[["no.such.relation"], [" %s" % r2], [r1, " %s " % r2], [], [r1, r2], [r1, "x"]]))
    # duplicate sources and duplicate rules
    qs.append(dict(id="duplicate_sources_rules", q_entity=["a", "b", "a"], cand=["c", "c"],
                   graph=[("a", r1, "b"), ("b", r1, "c"), ("a", r2, "c")],
                   predicted_paths=[[r1], [r1], [r2, r1], []]))
    # no rules at all, no triples at all
    qs.append(dict(id="no_rules", q_entity=["a"], cand=["b"], graph=[("a", r1, "b")], predicted_paths=[]))
    qs.append(dict(id="no_triples", q_entity=["a"], cand=["a"], graph=[], predicted_paths=[[], [r1]]))

    for q in qs:
        graph = gu.build_graph(q["graph"], [], False)
        q["bfs_with_rule"] = [[e, r, gu.bfs_with_rule(graph, e, r)] for e in q["q_entity"] for r in q["predicted_paths"]]
        # apply_rules is stored as the concatenation of these calls; check that this is what it returns
        assert apply_rules(gu, graph, q["predicted_paths"], q["q_entity"]) == [p for _, _, ps in q["bfs_with_rule"]
                                                                               for p in ps]
        q["lists_with_rules"] = lists_of_paths(gu, ut, q, True)
        q["lists_without_rules"] = lists_of_paths(gu, ut, q, False)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:                             # one question per line
        f.write("[\n" + ",\n".join(json.dumps(q, separators=(",", ":")) for q in qs) + "\n]\n")
    print("wrote %s: %d questions, %d bytes, %d rule paths" % (OUT, len(qs), os.path.getsize(OUT),
                                                               sum(len(ps) for q in qs for _, _, ps in q["bfs_with_rule"])))


if __name__ == "__main__":
    main()
