"""CPU: the host arithmetic of a graphed GraftNet training epoch (graphed.epoch_plan with graft counts) against the host
loader's batches, and the refusals of gr_epoch_graft_begin before any CUDA call.  The GPU half is
tests/test_graft_train_epoch_gpu.py."""
import ctypes

import numpy as np
import pytest

from gnn_rag_b200 import _lib, graphed, loader

from test_device_split_host import GraftSplitLoader
from test_train_epoch_host import _counts

PTR = 0x1000          # a non-null device pointer: never dereferenced, every call below is refused first


def _graft_counts(L):
    """Stored graft entries per question, read straight from the loader's create_kb_adj_mats_facts."""
    return np.array([len(L.create_kb_adj_mats_facts(q)[0][0][2]) for q in range(L.num_data)], dtype=np.int64)


LOADERS = {   # name -> GraftSplitLoader kwargs
    "spread": dict(seed=5, num_questions=23, max_local_entity=60, facts_lo=20, facts_hi=600),
    "inverse": dict(seed=6, num_questions=13, max_local_entity=30, facts_lo=5, facts_hi=400,
                    use_inverse_relation=True),
    "empty_questions": dict(seed=4, num_questions=9, max_local_entity=6, facts_hi=1),
}


@pytest.mark.parametrize("p", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("batch_size", [1, 4, 5])
@pytest.mark.parametrize("name", sorted(LOADERS))
def test_plan_equals_the_graft_loaders_batches(name, batch_size, p):
    """Per step: the kb counts as without graft counts, and the graft entries G of the host loader's batch (both
    lists of build_fact_mat_maxfacts, GraftSingleDataLoader's graft half of get_batch, with fact dropout p) with their
    capacity bucket."""
    L = GraftSplitLoader(**LOADERS[name])
    np.random.seed(3)
    L.reset_batches(is_sequential=False)
    stored, ents = _counts(L)
    graft = _graft_counts(L)
    plan = graphed.epoch_plan(L.batches, stored, ents, batch_size, p, graft)
    kb_only = graphed.epoch_plan(L.batches, stored, ents, batch_size, p)
    assert kb_only.G is None and kb_only.graft_capacity is None
    for f in ("B", "F", "K", "capacity", "starts"):
        assert np.array_equal(getattr(plan, f), getattr(kb_only, f)), f
    steps = -(-L.num_data // batch_size)
    assert plan.steps == steps and len(plan.G) == len(plan.graft_capacity) == steps
    for it in range(steps):
        ids = L.batches[batch_size * it:min(batch_size * (it + 1), L.num_data)]
        ((hb, _hf, _he, _hv), (tb, _te, _tf, _tv)), _kfr = loader.build_fact_mat_maxfacts(L, ids, p)
        assert len(hb) == len(tb) == plan.G[it]
        assert plan.graft_capacity[it] == graphed.fact_capacity(len(hb))
    if name == "empty_questions":
        assert (graft == 0).any()
    if name == "inverse":
        assert np.array_equal(graft, 2 * stored)


def test_plan_counts_an_out_of_range_id_as_an_empty_question():
    L = GraftSplitLoader(**LOADERS["spread"])
    stored, ents = _counts(L)
    graft = _graft_counts(L)
    plan = graphed.epoch_plan(np.array([0, 1, 99, 2, -1, 3]), stored, ents, 4, 0.0, graft)
    assert plan.G.tolist() == [int(graft[[0, 1, 2]].sum()), int(graft[3])]
    empty = graphed.epoch_plan([], stored, ents, 4, 0.0, graft)
    assert empty.steps == 0 and empty.G.size == empty.graft_capacity.size == 0


# ---- the entry point -------------------------------------------------------------------------------------------------

def test_header_declaration_and_binding():
    P, I64, I = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    assert _lib.SIGNATURES["gr_epoch_graft_begin"] == (I, [P, I, P, P, I64, I64, P, P, P, P])
    assert _lib.load().gr_epoch_graft_begin.argtypes == [P, I, P, P, I64, I64, P, P, P, P]


def _graft_begin(**over):
    a = dict(ids=PTR, B=4, kept_table=None, g_off=PTR, num_q=5, capacity=1024, kept_g=PTR, graft_live=PTR, status=PTR,
             stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_epoch_graft_begin(*a.values()), lib.gr_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(ids=None), "null pointer"), (dict(g_off=None), "null pointer"), (dict(kept_g=None), "null output"),
    (dict(graft_live=None), "null output"), (dict(status=None), "null output"), (dict(B=0), "need B > 0"),
    (dict(B=-3), "need B > 0"), (dict(num_q=-1), "need B > 0 and num_q >= 0"),
    (dict(capacity=-1), "capacity must be in [0, INT_MAX]"), (dict(capacity=2 ** 31), "capacity must be in")])
def test_graft_begin_refusals(over, msg):
    rc, err = _graft_begin(**over)
    assert rc == -1 and err.startswith("gr_epoch_graft_begin: invalid argument: " + msg)
