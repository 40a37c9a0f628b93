"""Host-side timing of GraftNet's extra batch assembly at the probe's scale (64 questions x 6000 subgraph tuples,
2000 local entities, 6106 relations): the unmodified reference ``GraftBasicDataLoader._build_fact_mat_maxfacts``
(gnn/dataset_load_graft.py:70-102) vs gnn_rag_b200.loader.build_fact_mat_maxfacts on a seeded stand-in loader state,
same RNG state, outputs compared bit for bit.  The drop-in's first call on a sample also runs the loader's own
``create_kb_adj_mats_facts`` (then cached): reported separately.  CPU only; needs the reference checkout."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gnn_rag_b200 import loader  # noqa: E402
from graft_loader_fixture import GraftStandIn  # noqa: E402
from oracle import ref_harness  # noqa: E402


def timed(fn, seed):
    np.random.seed(seed)
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def flat(out):
    ((a, b, c, d), (e, f, g, h)), r = out
    return [a, b, c, d, e, f, g, h, r]


if __name__ == "__main__":
    B, N, T, R = 64, 2000, 6000, 6106
    ref_harness._import_reference()
    import dataset_load_graft  # noqa: E402  (reference module, imported read-only)
    G = dataset_load_graft.GraftBasicDataLoader

    class RefLoader(GraftStandIn):
        create_kb_adj_mats_facts = G.create_kb_adj_mats_facts

    kw = dict(seed=0, num_questions=B, max_local_entity=N, num_relations=R, form="str", facts_hi=T)
    ld_ref, ld_new = RefLoader(**kw), RefLoader(**kw)
    for ld in (ld_ref, ld_new):          # every question at T tuples
        rs = np.random.RandomState(1)
        for q in range(B):
            ents = list(ld.global2local_entity_maps[q])
            tup = ld.data[q]["subgraph"]["tuples"]
            while len(tup) < T:
                h, t = rs.choice(len(ents), 2)
                tup.append(["ent.%d" % ents[h], "rel.%d" % rs.randint(R), "ent.%d" % ents[t]])
        ld.max_facts = 2 * T + N
    ids = list(range(B))
    res = {"config": dict(B=B, N=N, tuples_per_question=T, relations=R, max_facts=2 * T + N)}
    for dropout in (0.0, 0.3):
        t_ref = min(timed(lambda: G._build_fact_mat_maxfacts(ld_ref, ids, dropout), s)[0] for s in range(3))
        t_first, _ = timed(lambda: loader.build_fact_mat_maxfacts(ld_new, ids, dropout), 0)
        t_new = min(timed(lambda: loader.build_fact_mat_maxfacts(ld_new, ids, dropout), s)[0] for s in range(5))
        _, a = timed(lambda: G._build_fact_mat_maxfacts(ld_ref, ids, dropout), 9)
        _, b = timed(lambda: loader.build_fact_mat_maxfacts(ld_new, ids, dropout), 9)
        same = all(x.dtype == y.dtype and np.array_equal(x, y) for x, y in zip(flat(a), flat(b)))
        ld_new.__dict__.pop("_gr_graft", None)
        res["fact_dropout_%g" % dropout] = dict(reference_ms=t_ref * 1e3, drop_in_first_call_ms=t_first * 1e3,
                                                drop_in_cached_ms=t_new * 1e3, speedup_cached=t_ref / t_new,
                                                bit_identical=bool(same))
    res["host"] = {"cpus": os.cpu_count(), "threads_used": 1}
    print(json.dumps(res, indent=1))
