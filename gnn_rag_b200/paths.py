"""Relation-labelled shortest paths between question entities and retrieved candidates -- the hand-over of the GNN
stage to the LLM stage (``llm/src/utils/graph_utils.py:10-21,49-75`` consumed by
``llm/src/qa_prediction/build_qa_input.py:114-127``).

    from gnn_rag_b200.paths import build_graph, get_truth_paths          # same names / arguments as utils.*
    graph = build_graph(question_dict["graph"])
    reasoning_paths = get_truth_paths(question_dict["q_entity"], question_dict["cand"], graph)

Same result as the reference, INCLUDING the order of the paths (the prompt text lists them in that order): the
reference builds an undirected ``networkx.Graph`` (a later triple between the same two entities overwrites the
relation label, either direction) and concatenates ``nx.all_shortest_paths(graph, h, t)`` over all (h, t) pairs.
Here the breadth-first distances from every question entity and every candidate come from the device kernel
(csrc/paths.cu, level-synchronous BFS over both CSRs); a node lies on a shortest h-t path iff d(h,v) + d(v,t) = d(h,t).
Only that sub-graph (a handful of nodes) is then walked on the host, in networkx's order: its BFS predecessor lists
depend only on the insertion order of the on-path nodes' edges -- every predecessor of an on-path node is itself
on-path -- so pruning does not change the order in which paths come out.

Rule paths (the "+RA" retrieval augmentation): ``bfs_with_rule`` / ``apply_rules`` / ``direct_answer`` /
``path_to_string`` are drop-ins for ``graph_utils.py:24-47``, ``build_qa_input.py:58-81`` and ``utils.py:34-44``.  The
walks run on the device (csrc/rule_paths.cu) over a label-grouped adjacency built once per graph; only the mapping of
node ids back to entity strings is host work.  ``reasoning_paths`` does a whole split in one device pass and returns
the path lists ``process_input`` (``build_qa_input.py:93-124``) builds, with and without ``add_rule``.
"""
import collections

import numpy as np
import torch

from . import ops


def _intern(g, triples, lab2id):
    """Host maps of one triple list, in nx.Graph.add_edge insertion order: entity ids, per-triple head / tail / label id
    (stripped relation strings interned into the shared ``lab2id``), and the pair -> label map (last triple wins)."""
    ent = {}
    heads = np.empty(len(triples), dtype=np.int64)
    tails = np.empty(len(triples), dtype=np.int64)
    labs = np.empty(len(triples), dtype=np.int64)
    label = {}
    for k, (h, r, t) in enumerate(triples):                # node / edge insertion order of nx.Graph.add_edge
        hi = ent.setdefault(h, len(ent))
        ti = ent.setdefault(t, len(ent))
        r = r.strip()
        heads[k], tails[k], labs[k] = hi, ti, lab2id.setdefault(r, len(lab2id))
        label[(hi, ti) if hi <= ti else (ti, hi)] = r      # graph_utils.py:20 -- the last triple wins
    g.ent2id, g.id2ent = ent, list(ent)
    g.heads, g.tails, g.labs, g.label = heads, tails, labs, label
    g.lab2id = lab2id
    g.N = max(len(ent), 1)


class PathGraph:
    """Device-resident undirected adjacency of one question's triple list + the host-side label maps."""

    def __init__(self, triples, device=None):
        device = torch.device("cuda") if device is None else torch.device(device)
        _intern(self, triples, {})
        self.device = device
        self._adj = None
        if len(triples):
            self.csr = ops.csr_build(torch.from_numpy(self.heads).to(device), torch.from_numpy(self.labs).to(device),
                                     torch.from_numpy(self.tails).to(device), 1, self.N, max(len(self.lab2id), 1))
        else:
            self.csr = None

    def __contains__(self, entity):
        return entity in self.ent2id

    def rule_walks(self, start, rule_off, rule_len, rule_lab):
        """Device walks of the jobs (see ops.rule_walks); the label-grouped adjacency is built on first use."""
        if self._adj is None:
            self._adj = ops.rule_adjacency(self.csr)
        paths, counts, elem_off = ops.rule_walks(self._adj, start, rule_off, rule_len, rule_lab)
        return paths.cpu().numpy(), counts, elem_off

    def distances(self, nodes):
        """BFS hop distances from each of ``nodes`` (ids) to every node: int32 [len(nodes), N], -1 = unreachable."""
        k = len(nodes)
        src = torch.tensor([nodes], dtype=torch.int32, device=self.device)
        cnt = torch.tensor([k], dtype=torch.int32, device=self.device)
        one = torch.zeros(1, 1, dtype=torch.int32, device=self.device)
        _on, _pd, dist = ops.shortest_path_nodes(self.csr, src, cnt, one, torch.zeros(1, dtype=torch.int32, device=self.device),
                                                 return_distances=True)
        return dist[0, :k].cpu().numpy()


def build_graph(graph, entities=None, encrypt=False, device=None):
    """Drop-in for ``utils.build_graph`` (graph_utils.py:10-21); ``encrypt`` re-labels entities through the reference's
    ``entities_names.json`` and is not supported here."""
    if encrypt:
        raise NotImplementedError("encrypt=True needs the reference's entities_names.json (graph_utils.py:6-8)")
    return PathGraph(graph, device)


def _ordered_adjacency(g, on):
    """Neighbour lists of the on-path nodes in networkx's insertion order, restricted to on-path nodes."""
    sel = np.nonzero(on[g.heads] & on[g.tails])[0]
    adj = {}
    for k in sel.tolist():
        u, v = int(g.heads[k]), int(g.tails[k])
        adj.setdefault(u, {}).setdefault(v, None)
        adj.setdefault(v, {}).setdefault(u, None)
    return adj


def _all_shortest_paths(adj, source, target):
    """networkx.all_shortest_paths on an unweighted graph: ``predecessor`` (unweighted.py) + the stack walk of
    ``_build_paths_from_predecessors`` (generic.py), order preserved."""
    seen, pred, nextlevel, level = {source: 0}, {source: []}, [source], 0
    while nextlevel:
        level += 1
        thislevel, nextlevel = nextlevel, []
        for v in thislevel:
            for w in adj.get(v, ()):
                if w not in seen:
                    pred[w] = [v]
                    seen[w] = level
                    nextlevel.append(w)
                elif seen[w] == level:
                    pred[w].append(v)
    if target not in pred:
        return
    on_stack = {target}
    stack, top = [[target, 0]], 0
    while top >= 0:
        node, i = stack[top]
        if node == source:
            yield [p for p, _ in reversed(stack[: top + 1])]
        if len(pred[node]) > i:
            stack[top][1] = i + 1
            nxt = pred[node][i]
            if nxt in on_stack:
                continue
            on_stack.add(nxt)
            top += 1
            if top == len(stack):
                stack.append([nxt, 0])
            else:
                stack[top][:] = [nxt, 0]
        else:
            on_stack.discard(node)
            top -= 1


def get_truth_paths(q_entity, a_entity, graph):
    """Drop-in for ``utils.get_truth_paths`` (graph_utils.py:49-75): every shortest path between every question entity
    and every candidate, as ``[(u, relation, v), ...]`` triples, in the reference's order."""
    g = graph
    hs = [h for h in q_entity if h in g]
    ts = [t for t in a_entity if t in g]
    if not hs or not ts or g.csr is None:
        return []
    uniq = list(dict.fromkeys(hs + ts))
    return _truth_walk(g, hs, ts, uniq, g.distances([g.ent2id[e] for e in uniq]))


def _truth_walk(g, hs, ts, uniq, dist):
    """get_truth_paths' host walk, given the BFS distances ``dist[i]`` from ``uniq[i]`` (rows may be padded)."""
    row = {e: i for i, e in enumerate(uniq)}
    out = []
    for h in hs:
        dh = dist[row[h]]
        hi = g.ent2id[h]
        for t in ts:
            ti = g.ent2id[t]
            d = int(dh[ti])
            if d < 0:
                continue                                       # nx.NetworkXNoPath, swallowed at :64-65
            dt = dist[row[t]]
            on = (dh >= 0) & (dt >= 0) & (dh + dt == d)
            adj = _ordered_adjacency(g, on)
            for p in _all_shortest_paths(adj, hi, ti):
                out.append([(g.id2ent[p[i]],
                             g.label[(p[i], p[i + 1]) if p[i] <= p[i + 1] else (p[i + 1], p[i])],
                             g.id2ent[p[i + 1]]) for i in range(len(p) - 1)])
    return out


# ---- rule paths (graph_utils.py:24-47, build_qa_input.py:58-124) ---------------------------------------------------

def _encode_jobs(lab2id, start, rules):
    """Jobs -> the arrays of ops.rule_walks: start ids, rule offsets / lengths, flat label ids.  A rule element that
    is not a (stripped) label of the graph -- e.g. one with surrounding whitespace -- gets -1 and matches nothing, as
    the reference's ``rel != target_rule[i]`` never matches it."""
    ln = np.array([len(r) for r in rules], dtype=np.int32)
    off = np.zeros(len(rules), dtype=np.int32)
    np.cumsum(ln[:-1], out=off[1:])
    lab = np.array([lab2id.get(x, -1) for r in rules for x in r], dtype=np.int32)
    return np.asarray(start, dtype=np.int32).reshape(-1), off, ln, lab


def _names(g):
    ents = getattr(g, "_ent_arr", None)
    if ents is None:
        ents = np.empty(len(g.id2ent), dtype=object)
        ents[:] = g.id2ent
        g._ent_arr = ents
    return ents


def _job_paths(g, nodes, count, eoff, rule, base=0):
    """One job's node block [count, len(rule) + 1] -> bfs_with_rule's ``[(u, rel, v), ...]`` lists; the relation of
    step i is rule[i] itself (it matched the edge label)."""
    L = len(rule)
    if L == 0:
        return [[] for _ in range(count)]
    blk = _names(g)[nodes[eoff: eoff + count * (L + 1)] - base].reshape(count, L + 1)
    return [list(zip(row[:-1], rule, row[1:])) for row in blk.tolist()]


def _rule_results(g, jobs):
    """jobs: [(start entity, rule), ...] on one graph -> per job the paths bfs_with_rule returns."""
    if g.csr is None:                                  # no triples: only empty rules give a (single, empty) path
        return [[[]] if len(rule) == 0 else [] for _, rule in jobs]
    rules = [rule for _, rule in jobs]
    start, off, ln, lab = _encode_jobs(g.lab2id, [g.ent2id.get(e, -1) for e, _ in jobs], rules)
    nodes, counts, elem_off = g.rule_walks(start, off, ln, lab)
    return [_job_paths(g, nodes, int(counts[j]), int(elem_off[j]), rule) for j, rule in enumerate(rules)]


def bfs_with_rule(graph, start_node, target_rule, max_p=10):
    """Drop-in for ``utils.bfs_with_rule`` (graph_utils.py:24-47): every walk from ``start_node`` whose i-th edge has
    the relation ``target_rule[i]``, as ``[(u, rel, v), ...]`` in the reference's FIFO order.  Nodes may repeat; an
    empty rule gives ``[[]]`` even for a start outside the graph.  ``max_p`` is not applied, as in the reference."""
    return _rule_results(graph, [(start_node, target_rule)])[0]


def apply_rules(graph, rules, source_entities):
    """Drop-in for ``PromptBuilder.apply_rules`` (build_qa_input.py:58-64): all jobs of one graph in one device pass,
    concatenated ``for entity in source_entities: for rule in rules``."""
    out = []
    for res in _rule_results(graph, [(e, r) for e in source_entities for r in rules]):
        out.extend(res)
    return out


def path_to_string(path):
    """Drop-in for ``utils.path_to_string`` (utils.py:34-44)."""
    result = ""
    for i, p in enumerate(path):
        if i == 0:
            h, r, t = p
            result += f"{h} -> {r} -> {t}"
        else:
            _, r, t = p
            result += f" -> {r} -> {t}"
    return result.strip()


def direct_answer(question_dict, encrypt=False):
    """``PromptBuilder.direct_answer`` (build_qa_input.py:66-81): the end entity of every non-empty rule path."""
    graph = build_graph(question_dict["graph"], [], encrypt)
    rules = question_dict["predicted_paths"]
    prediction = []
    if len(rules) > 0:
        for p in apply_rules(graph, rules, question_dict["q_entity"]):
            if len(p) > 0:
                prediction.append(p[-1][-1])
    return prediction


def prompt_path_list(rule_strings, truth_strings):
    """``lists_of_paths`` of ``process_input`` (build_qa_input.py:92-124) before ``check_prompt_length``: the rule-path
    strings as they come (``[]`` without ``add_rule``), then every truth-path string not already in the list
    (``truth_strings`` is None when the question has no ``cand``)."""
    out = list(rule_strings)
    seen = set(out)
    for s in truth_strings or ():
        if s not in seen:
            out.append(s)
            seen.add(s)
    return out


ReasoningPaths = collections.namedtuple("ReasoningPaths", "rule_paths with_rules without_rules")
ReasoningPaths.__doc__ = """One question's result of :func:`reasoning_paths`: ``rule_paths`` = apply_rules' paths;
``with_rules`` / ``without_rules`` = process_input's ``lists_of_paths`` with ``add_rule`` on / off."""


class _HostGraph:
    """Host maps of one question of a batch (the device arrays are the batch's)."""

    def __init__(self, triples, lab2id):
        _intern(self, triples, lab2id)


def reasoning_paths(questions, rules_key="predicted_paths", device=None):
    """Rule paths and prompt path lists for a whole split in one device pass.

    ``questions``: dicts with ``graph`` (triples), ``q_entity``, ``cand`` (None = no truth paths) and ``rules_key``
    (``predicted_paths``; ``ground_paths`` for ``use_true``).  All graphs go into one batched CSR (question b owns node
    rows b*N ..), every (question, source, rule) job into one level expansion, and the truth-path BFS of every
    question into one ``gr_shortest_path_nodes`` launch.  Returns one :class:`ReasoningPaths` per question."""
    device = torch.device("cuda") if device is None else torch.device(device)
    if not questions:
        return []
    lab2id = {}
    gs = [_HostGraph(q["graph"], lab2id) for q in questions]
    B, N = len(gs), max(g.N for g in gs)
    heads = np.concatenate([g.heads + b * N for b, g in enumerate(gs)])
    tails = np.concatenate([g.tails + b * N for b, g in enumerate(gs)])
    labs = np.concatenate([g.labs for g in gs])
    csr = ops.csr_build(torch.from_numpy(heads).to(device), torch.from_numpy(labs).to(device),
                        torch.from_numpy(tails).to(device), B, N, max(len(lab2id), 1))
    csr.check_status()

    # rule half: apply_rules' job order, question by question
    starts, rules, owner = [], [], []
    for b, (q, g) in enumerate(zip(questions, gs)):
        q_rules = q[rules_key]
        if len(q_rules) > 0:
            for e in q["q_entity"]:
                s = b * N + g.ent2id[e] if e in g.ent2id else -1
                for r in q_rules:
                    starts.append(s)
                    rules.append(r)
                    owner.append(b)
    start, off, ln, lab = _encode_jobs(lab2id, starts, rules)
    nodes_d, counts, elem_off = ops.rule_walks(ops.rule_adjacency(csr), start, off, ln, lab)

    # truth half: BFS from every question's (question entity | candidate) set in one launch
    sel = [None] * B
    for b, (q, g) in enumerate(zip(questions, gs)):
        if q.get("cand") is not None:
            hs = [h for h in q["q_entity"] if h in g.ent2id]
            ts = [t for t in q["cand"] if t in g.ent2id]
            if hs and ts:
                sel[b] = (hs, ts, list(dict.fromkeys(hs + ts)))
    S = max([len(s[2]) for s in sel if s is not None] + [1])
    src = np.zeros((B, S), dtype=np.int32)
    cnt = np.zeros(B, dtype=np.int32)
    for b, s in enumerate(sel):
        if s is not None:
            cnt[b] = len(s[2])
            src[b, : cnt[b]] = [gs[b].ent2id[e] for e in s[2]]
    dist = None
    if cnt.any():
        zero = torch.zeros(B, 1, dtype=torch.int32, device=device)
        _on, _pd, d = ops.shortest_path_nodes(csr, torch.from_numpy(src).to(device), torch.from_numpy(cnt).to(device),
                                              zero, zero[:, 0].contiguous(), return_distances=True)
        dist = d[:, :S].cpu().numpy()
    nodes = nodes_d.cpu().numpy()

    per_q = [[] for _ in range(B)]
    for j, (b, r) in enumerate(zip(owner, rules)):
        per_q[b].extend(_job_paths(gs[b], nodes, int(counts[j]), int(elem_off[j]), r, b * N))
    out = []
    for b, (q, g) in enumerate(zip(questions, gs)):
        truth = None
        if q.get("cand") is not None:
            truth = [] if sel[b] is None else [path_to_string(p) for p in _truth_walk(g, *sel[b], dist[b])]
        rule_strings = [path_to_string(p) for p in per_q[b]]
        out.append(ReasoningPaths(per_q[b], prompt_path_list(rule_strings, truth), prompt_path_list([], truth)))
    return out
