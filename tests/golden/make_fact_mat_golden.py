"""Golden outputs of the UNMODIFIED reference ``BasicDataLoader._build_fact_mat`` (gnn/dataset_load.py:473-527) on
the stand-in loader states of tests/loader_fixture.py.  Run in the build container (needs /root/reference):
    python tests/golden/make_fact_mat_golden.py
writes tests/golden/loader/fact_mat_<case>.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from loader_fixture import CASES, FakeLoader, live_cases  # noqa: E402
from oracle import ref_harness  # noqa: E402


def reference_build_fact_mat():
    ref_harness._import_reference()
    import dataset_load  # noqa: E402  (reference module, imported read-only)
    return dataset_load.BasicDataLoader._build_fact_mat


if __name__ == "__main__":
    fn = reference_build_fact_mat()
    for name, (kw, ids, dropout, seed) in CASES.items():
        ld = FakeLoader(**kw)
        np.random.seed(seed)
        h, r, t, b, f, w, wr = fn(ld, ids, dropout)
        np.savez(os.path.join(HERE, "loader", "fact_mat_%s.npz" % name), heads=h, rels=r, tails=t, batch_ids=b, fact_ids=f,
                 weight_list=np.asarray(w, dtype=np.float64), weight_rel_list=np.asarray(wr, dtype=np.float64))
        print(name, len(h), "facts")
    # the larger states: compressed, indices as int32 (the tests compare values and dtype kinds)
    for name, (kw, ids, dropout, seed) in live_cases().items():
        ld = FakeLoader(**kw)
        np.random.seed(seed)
        h, r, t, b, f, w, wr = fn(ld, ids, dropout)
        np.savez_compressed(os.path.join(HERE, "loader", "fact_mat_%s.npz" % name),
                            **{k: np.asarray(v, dtype=np.int32) for k, v in
                               dict(heads=h, rels=r, tails=t, batch_ids=b, fact_ids=f).items()},
                            weight_list=np.asarray(w, dtype=np.float64), weight_rel_list=np.asarray(wr, dtype=np.float64))
        print(name, len(h), "facts")
