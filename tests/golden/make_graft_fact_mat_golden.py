"""Golden outputs of the UNMODIFIED reference ``GraftBasicDataLoader.create_kb_adj_mats_facts`` and
``_build_fact_mat_maxfacts`` (gnn/dataset_load_graft.py:27-102) on the stand-in loader states of
tests/graft_loader_fixture.py.  Run where the reference checkout exists:
    python tests/golden/make_graft_fact_mat_golden.py
writes tests/golden/loader/graft_fact_mat_<case>.npz: the per-question ``create_kb_adj_mats_facts`` results
(``q<sid>_*``), the outputs of ``_build_fact_mat_maxfacts`` after ``np.random.seed(seed)``, and for the
``SEQUENCE`` case the outputs of one ``get_batch``'s ``_build_fact_mat`` -> ``_build_fact_mat_maxfacts`` under one
seed (``seq_fm_*`` / ``seq_*``)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from graft_loader_fixture import CASES, PER_Q_KEYS, SEQUENCE, GraftStandIn, flatten_output  # noqa: E402
from oracle import ref_harness  # noqa: E402

FM_KEYS = ("heads", "rels", "tails", "batch_ids", "fact_ids", "weight_list", "weight_rel_list")


def reference_methods():
    ref_harness._import_reference()
    import dataset_load  # noqa: E402  (reference modules, imported read-only)
    import dataset_load_graft  # noqa: E402
    G = dataset_load_graft.GraftBasicDataLoader
    return dataset_load.BasicDataLoader._build_fact_mat, G.create_kb_adj_mats_facts, G._build_fact_mat_maxfacts


class RefGraftLoader(GraftStandIn):
    pass


if __name__ == "__main__":
    build_fact_mat, create, maxfacts = reference_methods()
    RefGraftLoader.create_kb_adj_mats_facts = create
    RefGraftLoader._build_fact_mat_maxfacts = maxfacts
    RefGraftLoader._build_fact_mat = build_fact_mat
    os.makedirs(os.path.join(HERE, "loader"), exist_ok=True)
    for name, (kw, ids, dropout, seed) in CASES.items():
        ld = RefGraftLoader(**kw)
        rec = {}
        for sid in sorted(set(ids)):
            ((a, b, c), (d, e, f)), rel = ld.create_kb_adj_mats_facts(sid)
            for k, v in zip(PER_Q_KEYS, (a, b, c, d, e, f, rel)):
                rec["q%d_%s" % (sid, k)] = v
        np.random.seed(seed)
        rec.update(flatten_output(ld._build_fact_mat_maxfacts(ids, dropout)))
        if name == SEQUENCE:
            np.random.seed(seed)
            fm = ld._build_fact_mat(ids, dropout)
            mf = ld._build_fact_mat_maxfacts(ids, dropout)
            for k, v in zip(FM_KEYS, fm):
                rec["seq_fm_" + k] = np.asarray(v)
            rec.update({"seq_" + k: v for k, v in flatten_output(mf).items()})
        np.savez(os.path.join(HERE, "loader", "graft_fact_mat_%s.npz" % name), **rec)
        print(name, len(rec["mats0_0"]), "graft facts")
