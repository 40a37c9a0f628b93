"""CPU: the rule-path restatement (tests/rule_paths_ref.py) reproduces the reference's stored results, and the host half
of gnn_rag_b200.paths -- job order, the empty-rule and missing-start rules, id -> entity mapping, path_to_string and
the prompt path lists -- matches it.  The walks the product takes from the device (tests/test_rule_paths_gpu.py) are
supplied here by a host walk over the same label ids."""
import collections

import numpy as np
import pytest

pytest.importorskip("networkx")

import rule_paths_ref as R  # noqa: E402
from gnn_rag_b200 import paths  # noqa: E402

GOLDEN = R.load_golden()
IDS = [q["id"] for q in GOLDEN]


class HostRuleGraph(paths.PathGraph):
    """PathGraph whose rule walks run on the host (no CUDA): same interning, same job arrays in and out."""

    def __init__(self, triples):
        paths._intern(self, triples, {})
        self.csr = object() if len(triples) else None
        self.nb = collections.defaultdict(dict)            # node -> {neighbour: label id}, nx.Graph order
        for h, t, lab in zip(self.heads.tolist(), self.tails.tolist(), self.labs.tolist()):
            self.nb[h][t] = lab
            self.nb[t][h] = lab
        self.calls = 0

    def rule_walks(self, start, rule_off, rule_len, rule_lab):
        self.calls += 1
        blocks, counts = [], []
        for s, o, L in zip(start.tolist(), rule_off.tolist(), rule_len.tolist()):
            rule = rule_lab[o: o + L].tolist()
            level = [[s]] if (L == 0 or s >= 0) else []
            for lab in rule:
                level = [p + [v] for p in level for v, lv in self.nb[p[-1]].items() if lv == lab]
            blocks.append(np.array(level, dtype=np.int32).reshape(-1))
            counts.append(len(level))
        counts = np.array(counts, dtype=np.int64)
        elem_off = np.concatenate([[0], np.cumsum(counts * (rule_len + 1))[:-1]]).astype(np.int64)
        return (np.concatenate(blocks) if blocks else np.zeros(0, np.int32)), counts, elem_off


@pytest.mark.parametrize("q", GOLDEN, ids=IDS)
def test_restatement_reproduces_the_reference(q):
    g = R.build_graph(q["graph"])
    for e, r, want in q["bfs_with_rule"]:
        assert R.bfs_with_rule(g, e, r) == want
    assert R.apply_rules(g, q["predicted_paths"], q["q_entity"]) == q["apply_rules"]
    assert R.lists_of_paths(q, True) == q["lists_with_rules"]
    assert R.lists_of_paths(q, False) == q["lists_without_rules"]


@pytest.mark.parametrize("q", GOLDEN, ids=IDS)
def test_host_half_matches_the_reference(q):
    g = HostRuleGraph(q["graph"])
    for e, r, want in q["bfs_with_rule"]:
        assert paths.bfs_with_rule(g, e, r) == want
    assert paths.apply_rules(g, q["predicted_paths"], q["q_entity"]) == q["apply_rules"]
    strings = [paths.path_to_string(p) for p in q["apply_rules"]] if len(q["predicted_paths"]) else []
    assert strings == q["lists_with_rules"][: len(strings)]          # the rule-path strings open the prompt list
    truth = None if q["cand"] is None else [R.path_to_string(p) for p in
                                            R.get_truth_paths(q["q_entity"], q["cand"], R.build_graph(q["graph"]))]
    assert paths.prompt_path_list(strings, truth) == q["lists_with_rules"]
    assert paths.prompt_path_list([], truth) == q["lists_without_rules"]


def test_apply_rules_is_one_walk_call_in_source_major_rule_minor_order():
    tri = [("a", "r", "b"), ("b", "s", "c"), ("a", "s", "c")]
    g = HostRuleGraph(tri)
    got = paths.apply_rules(g, [["s"], ["r"]], ["a", "b", "a"])
    assert g.calls == 1
    assert got == R.apply_rules(R.build_graph(tri), [["s"], ["r"]], ["a", "b", "a"])
    assert got == [[("a", "s", "c")], [("a", "r", "b")], [("b", "s", "c")], [("b", "r", "a")],
                   [("a", "s", "c")], [("a", "r", "b")]]


def test_empty_rule_and_missing_start():
    g = HostRuleGraph([("a", "r", "b")])
    assert paths.bfs_with_rule(g, "zz", []) == [[]]
    assert paths.bfs_with_rule(g, "zz", ["r"]) == []
    assert paths.bfs_with_rule(g, "a", []) == [[]]
    assert paths.bfs_with_rule(g, "a", [" r"]) == []          # rule elements are not stripped
    empty = HostRuleGraph([])
    assert paths.apply_rules(empty, [[], ["r"]], ["a"]) == [[]]


def test_path_to_string_and_direct_answer_shape():
    assert paths.path_to_string([]) == ""
    p = [(" a", "r", "b"), ("b", "s", "c ")]
    assert paths.path_to_string(p) == R.path_to_string(p) == "a -> r -> b -> s -> c"
    with pytest.raises(NotImplementedError):
        paths.direct_answer(dict(graph=[], q_entity=[], predicted_paths=[]), encrypt=True)


def test_prompt_path_list_dedups_truth_only():
    assert paths.prompt_path_list(["x", "x", "y"], ["y", "z", "z"]) == ["x", "x", "y", "z"]
    assert paths.prompt_path_list(["x"], None) == ["x"]
    assert paths.prompt_path_list([], ["z", "z"]) == ["z"]
