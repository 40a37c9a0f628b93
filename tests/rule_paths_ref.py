"""networkx restatement of the reference's rule-path functions, used by tests/test_rule_paths_*.py as the yardstick
(pinned against the unmodified reference by tests/golden/rule_paths/cases.json, tests/golden/make_rule_paths_golden.py):
``build_graph`` / ``bfs_with_rule`` / ``get_truth_paths`` (llm/src/utils/graph_utils.py:10-75), ``path_to_string``
(llm/src/utils/utils.py:34-44), ``PromptBuilder.apply_rules`` and the path list of ``process_input``
(llm/src/qa_prediction/build_qa_input.py:58-64,92-124)."""
import collections
import json
import os

import networkx as nx

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rule_paths", "cases.json")


def build_graph(triples):                                      # graph_utils.py:10-21 (encrypt=False)
    G = nx.Graph()
    for h, r, t in triples:
        G.add_edge(h, t, relation=r.strip())
    return G


def bfs_with_rule(graph, start_node, target_rule):             # graph_utils.py:24-47 (max_p unused there too)
    result_paths = []
    queue = collections.deque([(start_node, [])])
    while queue:
        current_node, current_path = queue.popleft()
        if len(current_path) == len(target_rule):
            result_paths.append(current_path)
        if len(current_path) < len(target_rule):
            if current_node not in graph:
                continue
            for neighbor in graph.neighbors(current_node):
                rel = graph[current_node][neighbor]["relation"]
                if rel != target_rule[len(current_path)]:
                    continue
                queue.append((neighbor, current_path + [(current_node, rel, neighbor)]))
    return result_paths


def apply_rules(graph, rules, sources):                        # build_qa_input.py:58-64
    out = []
    for e in sources:
        for r in rules:
            out.extend(bfs_with_rule(graph, e, r))
    return out


def path_to_string(path):                                      # utils.py:34-44
    result = ""
    for i, p in enumerate(path):
        if i == 0:
            h, r, t = p
            result += f"{h} -> {r} -> {t}"
        else:
            _, r, t = p
            result += f" -> {r} -> {t}"
    return result.strip()


def get_truth_paths(q_entity, a_entity, graph):                # graph_utils.py:49-75
    out = []
    for h in q_entity:
        if h not in graph:
            continue
        for t in a_entity:
            if t not in graph:
                continue
            try:
                out.extend(nx.all_shortest_paths(graph, h, t))
            except Exception:                                   # noqa: BLE001 -- NetworkXNoPath is swallowed at :64-65
                pass
    return [[(p[i], graph[p[i]][p[i + 1]]["relation"], p[i + 1]) for i in range(len(p) - 1)] for p in out]


def lists_of_paths(q, add_rule, rules_key="predicted_paths"):  # build_qa_input.py:92-124, before check_prompt_length
    lists = []
    graph = build_graph(q["graph"])
    if add_rule and len(q[rules_key]) > 0:
        lists = [path_to_string(p) for p in apply_rules(graph, q[rules_key], q["q_entity"])]
    if q["cand"] is not None:
        for p in get_truth_paths(q["q_entity"], q["cand"], graph):
            if path_to_string(p) not in lists:
                lists.append(path_to_string(p))
    return lists


def _paths(ps):
    return [[tuple(s) for s in p] for p in ps]


def load_golden():
    """The stored questions, with triples and path steps as tuples (JSON keeps them as lists).  ``apply_rules`` is the
    concatenation of the stored ``bfs_with_rule`` calls, which are in apply_rules' order."""
    with open(GOLDEN) as f:
        qs = json.load(f)
    for q in qs:
        q["graph"] = [tuple(t) for t in q["graph"]]
        q["bfs_with_rule"] = [(e, r, _paths(ps)) for e, r, ps in q["bfs_with_rule"]]
        q["apply_rules"] = [p for _, _, ps in q["bfs_with_rule"] for p in ps]
    return qs
