"""Rule-path probe: the prompt path lists of a whole test split (PromptBuilder.apply_rules + process_input,
llm/src/qa_prediction/build_qa_input.py:58-124), networkx restatement of the reference loop vs the batched GPU call.

    python scripts/rule_paths_probe.py --dataset webqsp --nodes 500 --out probe.json

The split is synthetic and seeded: its question count, rules per question and rule lengths follow the shipped
``llm/results/gen_rule_path/RoG-*/RoG/test/predictions_3_False.jsonl`` (histograms below).  The RoG subgraphs are not
shipped, so the graph size is a flag (``--nodes``, ``--degree``); each question's rules are planted as chains from its
question entity so that they match.  Times, in one run: the restatement (one networkx graph per question, then
bfs_with_rule / get_truth_paths / the list assembly), ``paths.reasoning_paths`` end to end (host interning, uploads,
kernels, read-back, string work), and the device section of that call by CUDA events (rule adjacency + level expansion,
incl. the per-level read-back of the level size, and the one BFS launch).  Checks that both give identical lists.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rule_paths_ref as R  # noqa: E402
from gnn_rag_b200 import ops, paths  # noqa: E402

# test split of predictions_3_False.jsonl: questions; {rules per question: count}; {rule length: count}
SPLITS = {
    "webqsp": (1628, {1: 7, 2: 12, 3: 1609}, {0: 4, 1: 3012, 2: 1823, 3: 18, 4: 1}),
    "cwq": (3531, {2: 10, 3: 3521}, {0: 35, 1: 3210, 2: 6778, 3: 453, 4: 96, 5: 11}),
}


def draw(rs, hist, size):
    keys = np.array(sorted(hist))
    p = np.array([hist[k] for k in keys], dtype=np.float64)
    return keys[rs.choice(len(keys), size=size, p=p / p.sum())]


def make_split(dataset, n_nodes, degree, n_rel, seed, questions=None):
    nq, rules_hist, len_hist = SPLITS[dataset]
    nq = questions or nq
    rs = np.random.RandomState(seed)
    out = []
    for qi in range(nq):
        ents = ["m.%d.%d" % (qi, i) for i in range(n_nodes)]
        m = n_nodes * degree // 2
        labs = rs.randint(n_rel, size=m)
        a, b = rs.randint(n_nodes, size=m), rs.randint(n_nodes, size=m)
        tri = [(ents[x], "rel.%d" % r, ents[y]) for x, r, y in zip(a, labs, b)]
        src = ents[rs.randint(n_nodes)]
        rules = [["rel.%d" % r for r in rs.randint(n_rel, size=L)]
                 for L in draw(rs, len_hist, int(draw(rs, rules_hist, 1)[0]))]
        for rule in rules:                                    # plant one chain per rule so that it matches
            u = src
            for rel in rule:
                v = ents[rs.randint(n_nodes)]
                tri.insert(rs.randint(len(tri) + 1), (u, rel, v) if rs.rand() < 0.5 else (v, rel, u))
                u = v
        cand = [ents[i] for i in rs.randint(n_nodes, size=5)]
        out.append(dict(graph=tri, q_entity=[src], predicted_paths=rules, cand=cand))
    return out


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", choices=sorted(SPLITS), default="webqsp")
    ap.add_argument("--questions", type=int, default=None, help="default: the split's size")
    ap.add_argument("--nodes", type=int, default=500, help="entities per question graph (not shipped: a guess)")
    ap.add_argument("--degree", type=int, default=4, help="mean undirected degree")
    ap.add_argument("--relations", type=int, default=40, help="distinct relation labels")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU: no CUDA device visible"
    qs = make_split(a.dataset, a.nodes, a.degree, a.relations, a.seed, a.questions)
    name, pl = card()

    t0 = time.perf_counter()
    want = []
    for q in qs:
        g = R.build_graph(q["graph"])
        rp = R.apply_rules(g, q["predicted_paths"], q["q_entity"])
        want.append((rp, R.lists_of_paths(q, True), R.lists_of_paths(q, False)))
    t_ref = time.perf_counter() - t0

    paths.reasoning_paths(qs[:8])                              # warm-up: module load, allocator
    torch.cuda.synchronize()
    e2e, dev = [], []
    for _ in range(a.repeats):
        ops.STATS.reset()
        ops.STATS.time_ops = True
        t0 = time.perf_counter()
        got = paths.reasoning_paths(qs)
        torch.cuda.synchronize()
        e2e.append(time.perf_counter() - t0)
        ops.STATS.time_ops = False
        dev.append(sum(s.elapsed_time(e) for s, e, c, _ in ops.STATS.op_events
                       if c in ("rule_paths", "paths", "csr_build")) / 1e3)
    equal = all(r.rule_paths == w[0] and r.with_rules == w[1] and r.without_rules == w[2] for r, w in zip(got, want))
    res = dict(card=name, power_limit=pl, dataset=a.dataset, questions=len(qs), nodes=a.nodes, degree=a.degree,
               relations=a.relations, rules=sum(len(q["predicted_paths"]) for q in qs),
               rule_paths=sum(len(w[0]) for w in want), equal=equal,
               reference_loop_s=t_ref, batched_e2e_s=min(e2e), batched_e2e_all_s=e2e, device_s=min(dev),
               device_all_s=dev, speedup_e2e=t_ref / min(e2e))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    if not equal:
        sys.exit("outputs differ")


if __name__ == "__main__":
    main()
